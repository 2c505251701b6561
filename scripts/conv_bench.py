#!/usr/bin/env python
"""Per-shape throughput of the conv kernels (CUDA-event timed, L2 flushed between iterations).
usage: python scripts/conv_bench.py [--impl 0|1|2] [--dirs fprop,dgrad,wgrad] [--only SUBSTR] [--iters N] [--batch B]
                                   [--precision tf32|fp32]
--precision fp32 times the split-TF32 (3xTF32) kernels; its fprop / dgrad rows include the filter split (sae_split_tf32).
The TFLOP/s column counts the convolution's FLOPs once in both modes.  "L2->smem GB" (fprop / dgrad rows on the wgmma kernel):
the bytes its TMA loads move into shared memory, A boxes plus B tiles over every CTA, computed from the tile plan of
conv_wgmma.cu (tile_box, tc_plan_groups)."""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from swapping_autoencoder_pytorch_b200 import backend  # noqa: E402
from swapping_autoencoder_pytorch_b200.backend import make_geom  # noqa: E402

# (name, H, C, K, R, stride, pad, images-per-32-batch multiplier)  — SURVEY.md Appendix A, the layers carrying the FLOPs
SHAPES = [
    ("D/G 128->128 @256 s1", 256, 128, 128, 3, 1, 1, 1.0),
    ("D/G 256->256 @128 s1", 128, 256, 256, 3, 1, 1, 1.0),
    ("D/G 512->512 @64 s1", 64, 512, 512, 3, 1, 1, 1.0),
    ("D 512->512 @32 s1", 32, 512, 512, 3, 1, 1, 1.0),
    ("D 128->256 @257 s2", 257, 128, 256, 3, 2, 0, 1.0),
    ("D 256->512 @129 s2", 129, 256, 512, 3, 2, 0, 1.0),
    ("D 512->512 @65 s2", 65, 512, 512, 3, 2, 0, 1.0),
    ("(no strips) 128->256 @256 s2", 256, 128, 256, 3, 2, 0, 1.0),
    ("D skip 128->256 @255 1x1 s2", 255, 128, 256, 1, 2, 0, 1.0),
    ("G skip 512->256 @64 1x1", 64, 512, 256, 1, 1, 0, 1.0),
    ("G convT 256->128 @128 (as dgrad of s2)", 257, 128, 256, 3, 2, 0, 1.0),
    ("FromRGB 32->128 @256 1x1", 256, 32, 128, 1, 1, 0, 1.0),
    ("D skip 128->256 @128 1x1 (decimated)", 128, 128, 256, 1, 1, 0, 1.0),
    ("D skip 256->512 @64 1x1 (decimated)", 64, 256, 512, 1, 1, 0, 1.0),
    ("Dpatch skip 32->64 @64 1x1 (decimated)", 64, 32, 64, 1, 1, 0, 8.0),
    ("Dpatch 32->32 @128 s1", 128, 32, 32, 3, 1, 1, 8.0),
    ("Dpatch 64->64 @64 s1", 64, 64, 64, 3, 1, 1, 8.0),
    ("E 32->32 @258 s1 p0", 258, 32, 32, 3, 1, 0, 1.0),
]


def _pow2_ceil(v):
    return 1 << max(v - 1, 0).bit_length()


def _problem_bytes(n, oh, ow, src_c, ncol, taps, stride, split):
    """L2 -> shared-memory bytes of one conv_wg problem: per CTA and 32-channel block, one A box per tap group
    (th + span rows) and one B tile per tap (BLOCK_N rows of 128 bytes, twice in split-TF32)."""
    tw = min(_pow2_ceil(ow), 16)
    th = min(128 // tw, _pow2_ceil(oh))
    tn = 128 // (tw * th)
    max_span = 160 // tw - th if tn == 1 and tw in (8, 16) else 0
    groups = []                                          # [gy, gx, span], taps in (ox, oy mod stride, oy) order
    for oy, ox in sorted(taps, key=lambda t: (t[1], t[0] % stride, t[0])):
        g = groups[-1] if groups else None
        if g is None or ox != g[1] or (oy - g[0]) % stride or (oy - g[0]) // stride > max_span:
            groups.append([oy, ox, 0])
        else:
            g[2] = (oy - g[0]) // stride
    box_rows = th + max(g[2] for g in groups)
    bn = 128 if ncol % 128 == 0 and not split else 64 if ncol % 64 == 0 else 32
    ctas = -(-ow // tw) * -(-oh // th) * -(-n // tn) * (ncol // bn)
    per_cblk = len(groups) * box_rows * tw * tn * 128 + len(taps) * (2 if split else 1) * bn * 128
    return ctas * (src_c // 32) * per_cblk


def l2_smem_bytes(d, n, h, c, kk, r, stride, pad, split):
    """tc_fprop / tc_dgrad (square maps, pad_t == pad_l): the problems they launch, summed"""
    taps = [(a, b) for a in range(r) for b in range(r)]
    if d == "fprop":
        p = (h + 2 * pad - r) // stride + 1
        return _problem_bytes(n, p, p, c, kk, [(a - pad, b - pad) for a, b in taps], stride, split)
    if stride == 1:
        return _problem_bytes(n, h, h, kk, c, [(pad - a, pad - b) for a, b in taps], 1, split)
    total = 0
    for ho in range(2):                                  # the stride-2 data gradient's parity classes
        for wo in range(2):
            cls = [((ho + pad - a) // 2, (wo + pad - b) // 2) for a, b in taps
                   if a % 2 == (ho + pad) % 2 and b % 2 == (wo + pad) % 2]
            if cls:
                total += _problem_bytes(n, (h - ho + 1) // 2, (h - wo + 1) // 2, kk, c, cls, 1, split)
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--impl", type=int, default=0)
    ap.add_argument("--dirs", default="fprop,dgrad,wgrad")
    ap.add_argument("--only", default="")
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--precision", default="tf32", choices=backend.PRECISIONS)
    args = ap.parse_args()
    k = backend.kernels()
    k.conv_impl = args.impl
    k.precision = args.precision
    dev = torch.device("cuda")
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)
    print("precision %s on %s" % (args.precision, torch.cuda.get_device_name()))
    print("%-42s %-6s %5s %9s %9s %8s %12s" % ("shape", "dir", "impl", "ms", "TFLOP/s", "GB/s", "L2->smem GB"))
    for name, h, c, kk, r, stride, pad, mult in SHAPES:
        if args.only and args.only not in name:
            continue
        n = max(int(args.batch * mult), 1)
        g = make_geom(n, h, h, c, kk, r, r, stride, pad, pad)
        x = torch.randn(n, h, h, c, device=dev)
        w = torch.randn(kk, r, r, c, device=dev) / (c * r * r) ** 0.5
        dy = torch.randn(n, g.P, g.Q, kk, device=dev)
        flops = 2.0 * n * g.P * g.Q * kk * r * r * c
        nbytes = 4.0 * (x.numel() + dy.numel() + w.numel())
        for d in args.dirs.split(","):
            fn = {"fprop": lambda: k.conv_fprop(x, w, g), "dgrad": lambda: k.conv_dgrad(dy, w, g),
                  "wgrad": lambda: k.conv_wgrad(dy, x, g)}[d]
            fn()
            torch.cuda.synchronize()
            ts = []
            for _ in range(args.iters):
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1))
            ms = sorted(ts)[len(ts) // 2]
            impl = k.conv_impl_for(g, {"fprop": 0, "dgrad": 1, "wgrad": 2}[d]) if args.impl == 0 else args.impl
            smem = "-"
            if impl == 2 and d != "wgrad":
                smem = "%.2f" % (l2_smem_bytes(d, n, h, c, kk, r, stride, pad, args.precision == "fp32") / 1e9)
            print("%-42s %-6s %5d %9.3f %9.1f %8.0f %12s" % (name, d, impl, ms, flops / ms / 1e9, nbytes / ms / 1e6, smem),
                  flush=True)
        del x, w, dy


if __name__ == "__main__":
    main()
