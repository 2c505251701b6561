"""Cost of gradient accumulation (opt.micro_batches), in one process on one GPU, with the card name, power limit and maximum SM
clock read in the same run:

* throughput: 256x256 default networks with CUDA graphs, (local batch, micro-batches) in (16, 1), (16, 2) and (32, 2),
  alternated, three rounds; each window is 16 half-steps (8 D with one lazy R1, 8 G) between CUDA events.  (32, 1) is not
  run: a 32-image step does not fit an 80 GB H100 with graphs (bench.py);
* the sae_bucket_accumulate launches alone, on the D and G groups' tensors, between CUDA events: achieved GB/s against the
  12 bytes per element the add needs (gradient read, bucket read, bucket write) and the H100 SXM data sheet's 3.35 TB/s;
* peak memory of one eager D + R1 and one G update with micro-batches of 2, 4 and 8 images (k = 2) at 256x256, 512x512 and
  the ffhq1024 option set (torch.cuda.max_memory_allocated).  A size whose predicted peak (twice the previous one) would not
  fit is skipped and reported as such.

    python scripts/grad_accumulation_bench.py [--rounds 3] [--out FILE.json]
"""
import argparse
import gc
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import swapping_autoencoder_pytorch_b200 as S  # noqa: E402
from swapping_autoencoder_pytorch_b200 import backend  # noqa: E402
from swapping_autoencoder_pytorch_b200.parallel import GradientBucket  # noqa: E402

HBM_DATASHEET_GBS = 3350.0
FFHQ1024 = dict(crop_size=1024, netG_scale_capacity=0.8, netE_num_downsampling_sp=5, netE_scale_capacity=0.4,
                global_code_ch=1536, patch_size=256)
MEMORY_CONFIGS = (("256x256 default nets", dict(crop_size=256)), ("512x512 default nets", dict(crop_size=512)),
                  ("ffhq1024 option set", FFHQ1024))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    return q or torch.cuda.get_device_name()


def emit(rows, row):
    rows.append(row)
    print(json.dumps(row), flush=True)


def throughput(rows, rounds, steps=16):
    opt = S.default_options(num_gpus=1, batch_size=16, crop_size=256, cuda_graphs=True)
    torch.manual_seed(0)
    trainer = S.create_optimizer(opt, S.create_model(opt))
    gen = torch.Generator("cuda").manual_seed(1)
    images = {b: torch.randn(b, 3, 256, 256, device="cuda", generator=gen).clamp(-1, 1) for b in (16, 32)}
    configs = ((16, 1), (16, 2), (32, 2))

    def window(batch, k, n, with_r1_every_d=False):
        opt.micro_batches = k
        trainer.train_mode_counter = 0
        # one lazy R1 per window: on the last D half-step (warm-up: on every D half-step)
        trainer.discriminator_iter_counter = opt.R1_once_every - (n + 1) // 2
        kinds = []
        for _ in range(n):
            if with_r1_every_d:
                trainer.discriminator_iter_counter = opt.R1_once_every - 1
            out = trainer.train_one_step({"real_A": images[batch]}, 0)
            kinds.append("D+R1" if "D_R1" in out else ("D" if "D_total" in out else "G"))
        return kinds

    for batch, k in configs:                     # warm-up and capture of every body of every configuration
        window(batch, k, 6, with_r1_every_d=True)
    torch.cuda.synchronize()
    assert trainer.graphs.disabled is None, trainer.graphs.disabled
    for r in range(rounds):
        for batch, k in configs:
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            kinds = window(batch, k, steps)
            b.record()
            torch.cuda.synchronize()
            assert kinds.count("D+R1") == 1, kinds
            ms = a.elapsed_time(b) / steps
            emit(rows, {"what": "throughput", "round": r, "local_batch": batch, "micro_batches": k,
                        "ms_per_update": round(ms, 3), "images_per_s": round(batch * 1000.0 / ms, 1)})
    emit(rows, {"what": "throughput", "local_batch": 32, "micro_batches": 1,
                "not_measured": "a 32-image step with CUDA graphs does not fit an 80 GB H100 (bench.py)"})
    emit(rows, {"what": "graphs", "captured": sorted(str(key) for key in trainer.graphs.captured),
                "max_memory_allocated_GB": round(torch.cuda.max_memory_allocated() / 1e9, 2)})
    groups = {"G": [p.numel() for p in trainer.Gparams], "D": [p.numel() for p in trainer.Dparams]}
    trainer.graphs.release()
    del trainer
    gc.collect()
    torch.cuda.empty_cache()
    return groups


def accumulate_kernel(rows, groups, reps=50):
    for name, sizes in groups.items():
        grads = [torch.randn(n, device="cuda") for n in sizes]
        bucket = GradientBucket(torch.device("cuda"))
        bucket.fill(grads, 0)
        for _ in range(5):
            bucket.fill(grads, 1)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            bucket.fill(grads, 1)
        b.record()
        torch.cuda.synchronize()
        ms = a.elapsed_time(b) / reps            # includes the host's cached pointer-table lookup, not the device's idle time:
        elements = sum(sizes)                    # the launches queue back to back
        gbs = 12.0 * elements / (ms * 1e-3) / 1e9
        emit(rows, {"what": "sae_bucket_accumulate", "group": name, "tensors": len(sizes), "elements": elements,
                    "ms_per_launch": round(ms, 4), "algorithmic_GB_per_s": round(gbs, 1),
                    "fraction_of_3.35_TB_per_s_datasheet": round(gbs / HBM_DATASHEET_GBS, 3)})
        del grads, bucket
        torch.cuda.empty_cache()


def memory(rows):
    total = torch.cuda.get_device_properties(0).total_memory
    for label, over in MEMORY_CONFIGS:
        prev = None
        for mb in (2, 4, 8):
            if prev is not None and 2 * prev > 0.85 * total:
                emit(rows, {"what": "memory", "config": label, "micro_batch": mb, "micro_batches": 2,
                            "not_measured": "predicted peak %.1f GB (twice the previous) would not fit" % (2 * prev / 1e9)})
                continue
            opt = S.default_options(**dict(over, num_gpus=1, batch_size=2 * mb, micro_batches=2, R1_once_every=1))
            torch.manual_seed(0)
            trainer = S.create_optimizer(opt, S.create_model(opt))
            real = torch.randn(2 * mb, 3, opt.crop_size, opt.crop_size, device="cuda").clamp(-1, 1)
            peaks = {}
            for kind in ("D+R1", "G"):
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                out = trainer.train_one_step({"real_A": real}, 0)
                torch.cuda.synchronize()
                peaks[kind] = torch.cuda.max_memory_allocated()
                assert ("D_R1" in out) == (kind == "D+R1")
            prev = max(peaks.values())
            emit(rows, {"what": "memory", "config": label, "micro_batch": mb, "micro_batches": 2, "batch": 2 * mb,
                        "peak_GB": {k: round(v / 1e9, 2) for k, v in peaks.items()}})
            del trainer, real, out
            gc.collect()
            torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write every row as one JSON list")
    args = ap.parse_args()
    rows = []
    emit(rows, {"card": card(), "precision": backend.kernels().precision})
    groups = throughput(rows, args.rounds)
    accumulate_kernel(rows, groups)
    memory(rows)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
