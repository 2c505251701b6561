"""Overhead of the skip-on-non-finite guard (opt.skip_nonfinite_steps): 256x256 default networks, 16 images, CUDA graphs,
32 half-steps (16 D with one lazy R1, 16 G) timed with CUDA events, alternating guard off / on three times in one process
so that both settings see the same card, clocks and neighbours.  Prints the card name and power limit beside the numbers.

    python scripts/nonfinite_guard_bench.py [--rounds 3] [--steps 32] [--batch 16]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import swapping_autoencoder_pytorch_b200 as S  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--batch", type=int, default=16)
    args = ap.parse_args()
    opt = S.default_options(num_gpus=1, batch_size=args.batch, crop_size=256, cuda_graphs=True)
    torch.manual_seed(0)
    trainer = S.create_optimizer(opt, S.create_model(opt))
    real = torch.randn(args.batch, 3, 256, 256, device="cuda", generator=torch.Generator("cuda").manual_seed(1)).clamp(-1, 1)
    for guard in (False, True):                      # warm up and capture the three bodies of both settings
        opt.skip_nonfinite_steps = guard
        trainer.graphs.warm_up(real)
    assert trainer.graphs.disabled is None, trainer.graphs.disabled

    def timed(guard):
        opt.skip_nonfinite_steps = guard
        # one lazy R1 among the 16 D half-steps: it falls on the last D step of the window
        trainer.train_mode_counter = 0
        trainer.discriminator_iter_counter = opt.R1_once_every - (args.steps + 1) // 2
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        kinds = []
        for _ in range(args.steps):
            out = trainer.train_one_step({"real_A": real}, 0)
            kinds.append("D+R1" if "D_R1" in out else ("D" if "D_total" in out else "G"))
        b.record()
        torch.cuda.synchronize()
        assert kinds.count("D+R1") == 1, kinds
        return a.elapsed_time(b) / args.steps

    rows = []           # images/s as bench.py counts them: one batch per half-step
    for r in range(args.rounds):
        for guard in (False, True):
            ms = timed(guard)
            rows.append({"round": r, "guard": guard, "ms_per_half_step": round(ms, 3),
                         "images_per_s": round(args.batch * 1000.0 / ms, 1)})
            print(json.dumps(rows[-1]), flush=True)
    off = [x["ms_per_half_step"] for x in rows if not x["guard"]]
    on = [x["ms_per_half_step"] for x in rows if x["guard"]]
    print(json.dumps({"card": card(), "batch": args.batch, "steps": args.steps, "off_ms": off, "on_ms": on,
                      "off_spread_ms": round(max(off) - min(off), 3), "mean_diff_ms": round(sum(on) / len(on) - sum(off) / len(off), 3),
                      "nonfinite_steps": trainer.nonfinite_steps()}))


if __name__ == "__main__":
    main()
