"""Cost of the training statistics (opt.training_stats), in one process on one GPU, with the card name, power limit and
maximum SM clock read in the same run:

* throughput: 256x256 default networks, 16 images, CUDA graphs; one trainer built with the statistics on, run with them off
  (``trainer.stats = None`` and no score sink: the graphs of the plain path, keys without ("stats",)) and on, alternated,
  three rounds; each window is 32 half-steps (16 D with one lazy R1, 16 G) between CUDA events;
* the norm launches of one G update alone (sae_sumsq over the gradients, sae_adam_norms over parameters and moments; E and G,
  106 tensors), between CUDA events over many updates: achieved bandwidth against the 16 bytes per element they read
  (gradient, parameter, both moments) and the H100 SXM data sheet's 3.35 TB/s.

    python scripts/training_stats_bench.py [--rounds 3] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import swapping_autoencoder_pytorch_b200 as S  # noqa: E402
from swapping_autoencoder_pytorch_b200 import backend  # noqa: E402

HBM_DATASHEET_GBS = 3350.0


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    return q or torch.cuda.get_device_name()


def emit(rows, row):
    rows.append(row)
    print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--out", default=None, help="also write every row as one JSON list")
    args = ap.parse_args()
    rows = []
    emit(rows, {"card": card(), "precision": backend.kernels().precision})

    opt = S.default_options(num_gpus=1, batch_size=16, crop_size=256, cuda_graphs=True, training_stats=True)
    torch.manual_seed(0)
    trainer = S.create_optimizer(opt, S.create_model(opt))
    stats = trainer.stats
    inner = trainer.model.singlegpu_model
    images = torch.randn(16, 3, 256, 256, device="cuda", generator=torch.Generator("cuda").manual_seed(1)).clamp(-1, 1)

    def window(on, n, with_r1_every_d=False):
        trainer.stats = stats if on else None
        inner.score_sink = stats.score if on else None
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

    for on in (False, True):                          # warm-up and capture of every body in both settings
        window(on, 6, with_r1_every_d=True)
    torch.cuda.synchronize()
    assert trainer.graphs.disabled is None, trainer.graphs.disabled
    per = {False: [], True: []}
    for r in range(args.rounds):
        for on in (False, True):
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            kinds = window(on, args.steps)
            b.record()
            torch.cuda.synchronize()
            assert kinds.count("D+R1") == 1, kinds
            ms = a.elapsed_time(b) / args.steps
            per[on].append(ms)
            emit(rows, {"what": "throughput", "round": r, "stats": on, "ms_per_half_step": round(ms, 3),
                        "images_per_s": round(16 * 1000.0 / ms, 1)})
    emit(rows, {"what": "throughput_summary", "ms_per_half_step_off": [round(v, 3) for v in per[False]],
                "ms_per_half_step_on": [round(v, 3) for v in per[True]],
                "mean_difference_ms": round(sum(per[True]) / len(per[True]) - sum(per[False]) / len(per[False]), 3),
                "graphs": sorted(str(key) for key in trainer.graphs.captured),
                "max_memory_allocated_GB": round(torch.cuda.max_memory_allocated() / 1e9, 2)})
    window(True, 2)                                   # ends on a G half-step: the G gradients below are its own
    got = trainer.training_stats()                    # every half-step run with the statistics on, warm-up included
    emit(rows, {"what": "window", **{k: v for k, v in got.items() if "/" in k and "nonfinite" not in k}})

    adam = trainer.optimizer_G
    elements = sum(p.numel() for p in adam.params)
    grads = [p.grad for p in adam.params]
    assert all(g is not None for g in grads)

    def norms():
        stats.record_update("G", grads, 1.0)

    for _ in range(10):
        norms()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(args.reps):
        norms()
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / args.reps                # the launches queue back to back
    gbs = 16.0 * elements / (ms * 1e-3) / 1e9
    emit(rows, {"what": "sae_sumsq+sae_adam_norms", "tensors": len(adam.params), "elements": elements,
                "ms_per_update": round(ms, 4), "algorithmic_GB_per_s": round(gbs, 1),
                "fraction_of_3.35_TB_per_s_datasheet": round(gbs / HBM_DATASHEET_GBS, 3)})
    stats.read()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
