"""Cost of the adaptive discriminator augmentation (opt.augment_p / opt.ada_target), in one process on one GPU, with the card
name, power limit and maximum SM clock read in the same run:

* throughput: 256x256 default networks, 16 images, CUDA graphs; one trainer built with the augmentation on, run with it off
  (``trainer.augment = None`` and no model hook: the graphs of the plain path, keys without ("ada",)) and on at fixed
  p = 0, 0.2 and 0.6, alternated, three rounds; each window is 32 half-steps (16 D with one lazy R1, 16 G) between CUDA
  events.  Peak memory of the warm-up and capture, off against on;
* the operator on the 40 images of one D step (real, rec, mix of a 16-image batch) at p = 0.6 draws: the forward
  (sae_augment_sample, the downsampling FIR, sae_augment_color) and the adjoint (sae_augment_color_adjoint, the FIR's
  adjoint, sae_augment_sample_adjoint) between CUDA events, and the two resampling kernels alone.

    python scripts/ada_bench.py [--rounds 3] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import swapping_autoencoder_pytorch_b200 as S  # noqa: E402
from swapping_autoencoder_pytorch_b200 import augment, backend  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    return q or torch.cuda.get_device_name()


def emit(rows, row):
    rows.append(row)
    print(json.dumps(row), flush=True)


def timed(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write every row as one JSON list")
    args = ap.parse_args()
    rows = []
    emit(rows, {"card": card(), "precision": backend.kernels().precision})

    opt = S.default_options(num_gpus=1, batch_size=16, crop_size=256, cuda_graphs=True, augment_p=0.2)
    torch.manual_seed(0)
    trainer = S.create_optimizer(opt, S.create_model(opt))
    pipe = trainer.augment
    inner = trainer.model.singlegpu_model
    images = torch.randn(16, 3, 256, 256, device="cuda", generator=torch.Generator("cuda").manual_seed(1)).clamp(-1, 1)

    def window(p, n, with_r1_every_d=False):
        trainer.augment = None if p is None else pipe
        inner.augment_pipe = None if p is None else pipe
        if p is not None:
            pipe.p.fill_(p)
        trainer.train_mode_counter = 0
        # one lazy R1 per window: on the last D half-step (warm-up: on every D half-step)
        trainer.discriminator_iter_counter = opt.R1_once_every - (n + 1) // 2
        kinds = []
        for _ in range(n):
            if with_r1_every_d:
                trainer.discriminator_iter_counter = opt.R1_once_every - 1
            out = trainer.train_one_step({"real_A": images}, 0)
            kinds.append("D+R1" if "D_R1" in out else ("D" if "D_total" in out else "G"))
        return kinds

    peak = {}
    for name, p in (("off", None), ("on", 0.6)):      # warm-up and capture of every body in both settings
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        window(p, 6, with_r1_every_d=True)
        torch.cuda.synchronize()
        peak[name] = torch.cuda.max_memory_allocated()
    assert trainer.graphs.disabled is None, trainer.graphs.disabled
    configs = [("off", None), ("p=0", 0.0), ("p=0.2", 0.2), ("p=0.6", 0.6)]
    per = {name: [] for name, _ in configs}
    for r in range(args.rounds):
        for name, p in configs:
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            kinds = window(p, args.steps)
            b.record()
            torch.cuda.synchronize()
            assert kinds.count("D+R1") == 1, kinds
            ms = a.elapsed_time(b) / args.steps
            per[name].append(ms)
            emit(rows, {"what": "throughput", "round": r, "config": name, "ms_per_half_step": round(ms, 3),
                        "images_per_s": round(16 * 1000.0 / ms, 1)})
    mean = {k: sum(v) / len(v) for k, v in per.items()}
    emit(rows, {"what": "throughput_summary", **{"ms_per_half_step_" + k: [round(x, 3) for x in v] for k, v in per.items()},
                **{"mean_difference_ms_" + k: round(mean[k] - mean["off"], 3) for k in per if k != "off"},
                "peak_memory_GB_off": round(peak["off"] / 1e9, 3), "peak_memory_GB_on": round(peak["on"] / 1e9, 3),
                "graphs": sorted(str(key) for key in trainer.graphs.captured)})

    # the operator alone, on one D step's 40 images
    n = 16 + 8 + 16
    x = torch.randn(n, 3, 256, 256, device="cuda", generator=torch.Generator("cuda").manual_seed(2)).clamp(-1, 1)
    dy = torch.randn_like(x)
    u, z = augment.draw(n, x.device)
    rec = augment.params(u, z, torch.full((1,), 0.6, device="cuda"), 256, 256)
    k = backend.kernels()
    s = k.augment_sample(x, rec)
    gc = k.augment_color_adjoint(dy, rec)
    ds = augment._downsample_adjoint(gc)
    resampled = int((~(rec[:, :6] == torch.tensor([1.0, 0, 0, 0, 1.0, 0], device="cuda")).all(1)).sum())
    with torch.no_grad():
        fwd = timed(lambda: augment.augment(x, rec), args.reps)
        adj = timed(lambda: augment.adjoint(dy, rec), args.reps)
        smp = timed(lambda: k.augment_sample(x, rec), args.reps)
        sadj = timed(lambda: k.augment_sample_adjoint(ds, gc, rec, 256, 256), args.reps)
        down = timed(lambda: augment._downsample(s), args.reps)
        down_adj = timed(lambda: augment._downsample_adjoint(gc), args.reps)
    emit(rows, {"what": "operator", "images": n, "resampled_images": resampled, "forward_ms": round(fwd, 3),
                "adjoint_ms": round(adj, 3), "sae_augment_sample_ms": round(smp, 3),
                "sae_augment_sample_adjoint_ms": round(sadj, 3), "downsample_fir_ms": round(down, 3),
                "downsample_fir_adjoint_ms": round(down_adj, 3)})
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
