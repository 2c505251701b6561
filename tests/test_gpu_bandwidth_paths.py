"""GPU (H100): every launch branch of the bandwidth-bound kernels (``csrc/upfirdn2d.cu``, ``csrc/elementwise.cu``,
``csrc/torgb.cu``, ``csrc/train_ops.cu``) against fp64.

``ROWS`` is a path table: (id, C entry point, expected kernel(s), arguments).  Each row runs its call under ``torch.profiler``
and requires that the device kernels it launched are exactly the expected ones, by their demangled names with template
arguments (``bias_act_kernel<4, unsigned int>``, ``fir_tma_kernel<4, 4, 1>``).  Where a branch lives inside one kernel
(Adam's float4 / scalar loop, ``modulate_bwd_kernel``'s narrow / wide loop) the row also names the branch, and a mirror of
the kernel's predicate asserts it.  ``tests/test_bandwidth_path_table.py`` (CPU) parses the four sources and fails when a
kernel or template instantiation has neither a row here nor an entry in ``UNREACHED``.

All rows run with ``round_tf32 = False`` (the rounding contract has its own test, ``test_gpu_rounding_contract.py``).
References are fp64: the oracle's NumPy direct-summation FIR, ``F.grid_sample``, ``F.interpolate``, ``F.pad`` and the
formulas written out.  Bounds:

* pure copies and single correctly rounded products (reflect pad, bucket pack / unpack, crop zero padding, ToRGB's channel
  3, modulate, filter preparation, the TF32 split): bit equality;
* fp32 arithmetic: per element ``|got - ref| <= c * 2^-24 * sum|terms|``, with c the length of the sum plus the few
  roundings around it.  Reductions done with fp32 atomics (grad_bias, grad_noise_weight, ds, ToRGB gw) use the same bound
  with c set by the number of terms: it holds in any summation order, yet a dropped or doubled CTA partial, or a wrong
  small channel next to a large one, exceeds it;
* activation bit masks: every bit equals the fp64 sign of the pre-activation; elements whose pre-activation lies within
  its error bound or 1e-6 max of zero are exempt, and fewer than 1 % may be.

Short vector arguments (biases, styles, ToRGB weights, noise weights) are passed as the head of a buffer whose next elements
are 1e3, so a read past their end fails every time instead of when stale memory happens to differ.

Unreached on purpose (``UNREACHED``): the int64-index instantiations ``bias_act_kernel<4, long>``, ``bias_act_kernel<1,
long>`` and ``modulate_kernel<long>`` need >= 2^31 elements (8 GiB or more per tensor), and the ``smem > 48 KB`` attribute
branch of ``sae_bias_act_backward`` cannot be taken at its 12 000-channel limit ((12 000 + 1) * 4 bytes < 48 KiB).

Importing this module does not touch CUDA: the CPU table check imports ``ROWS`` and ``UNREACHED`` from it."""
import ctypes
import math
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import sae_oracle as O
from oracle.fixtures import rnd

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
SENTINEL = 1e3
SQRT2 = math.sqrt(2)

# kernels no row reaches, with the reason (normalised names, see ``kernel_name``)
UNREACHED = {
    "bias_act_kernel<4,long>": "int64 indexing: needs >= 2^31 elements",
    "bias_act_kernel<1,long>": "int64 indexing: needs >= 2^31 elements",
    "modulate_kernel<long>": "int64 indexing: needs >= 2^32 float4 vectors",
}


def _sep(taps):
    return tuple(float(np.float32(t)) for t in taps)


# separable test taps: asymmetric, so a flipped or transposed filter shows
TAPS = {1: _sep([0.7]), 2: _sep([0.3, 0.9]), 3: _sep([0.25, 0.6, -0.35]), 4: _sep([0.1, 0.45, 0.8, -0.2])}
TAPS_X = {1: _sep([-1.3]), 2: _sep([0.55, -0.15]), 3: _sep([0.4, 0.9, 0.15]), 4: _sep([-0.3, 0.7, 0.5, 0.25])}


def _fir_rows():
    rows = [
        # sae_upfirdn2d: (N, H, W, C, kh, kw, up, down, (px0, px1, py0, py1), storage offset)
        ("fir_generic4_up2_down3_5x3_negpad", "sae_upfirdn2d", "fir_generic_kernel<4>",
         dict(shape=(2, 9, 11, 8), k=(5, 3), up=(2, 2), down=(3, 3), pad=(-1, 2, 3, -2))),
        ("fir_generic4_upx1_upy2", "sae_upfirdn2d", "fir_generic_kernel<4>",
         dict(shape=(1, 6, 7, 4), k=(2, 3), up=(1, 2), down=(2, 1), pad=(1, 1, 0, 1))),
        ("fir_generic1_c3", "sae_upfirdn2d", "fir_generic_kernel<1>",
         dict(shape=(2, 10, 12, 3), k=(3, 3), up=(1, 1), down=(1, 1), pad=(1, 1, 1, 1))),
        ("fir_generic1_c64_offset1", "sae_upfirdn2d", "fir_generic_kernel<1>",
         dict(shape=(1, 9, 8, 64), k=(4, 4), up=(1, 1), down=(1, 1), pad=(2, 1, 2, 1), offset=1)),
        ("fir_strip33_h13", "sae_upfirdn2d", "fir_strip_kernel<3,3,8>",
         dict(shape=(2, 13, 10, 16), k=(3, 3), up=(1, 1), down=(1, 1), pad=(1, 1, 1, 1))),
        ("fir_strip44_h13_w9", "sae_upfirdn2d", "fir_strip_kernel<4,4,8>",
         dict(shape=(2, 13, 9, 8), k=(4, 4), up=(1, 1), down=(1, 1), pad=(2, 1, 2, 1))),
        ("fir_strip44_negpad", "sae_upfirdn2d", "fir_strip_kernel<4,4,8>",
         dict(shape=(1, 15, 14, 4), k=(4, 4), up=(1, 1), down=(1, 1), pad=(-1, 2, 1, -2))),
    ]
    # sae_upfirdn2d_separable: strip kernel, DOWN 1 and 2, 1-4 taps (C = 8 keeps 3 / 4 taps off the TMA kernel)
    for t in (1, 2, 3, 4):
        for down in (1, 2):
            rows.append(("sep_strip_down%d_t%d" % (down, t), "sae_upfirdn2d_separable",
                         "fir_sep_strip_kernel<%d,%d,16,%d>" % (t, t, down),
                         dict(shape=(2, 21, 18, 8), t=t, up=1, down=down, pad=(t // 2, (t - 1) // 2 + 1, (t - 1) // 2, t // 2))))
        for name, pad in (("even", (2, 1, 0, 3)), ("odd", (1, 2, 3, 0))):
            rows.append(("sep_up2_t%d_%spad" % (t, name), "sae_upfirdn2d_separable", "fir_sep_up2_kernel<%d,%d>" % (t, t),
                         dict(shape=(2, 7, 9, 8), t=t, up=2, down=1, pad=pad)))
    rows += [
        ("sep_strip_t4_negpad", "sae_upfirdn2d_separable", "fir_sep_strip_kernel<4,4,16,1>",
         dict(shape=(1, 19, 17, 8), t=4, up=1, down=1, pad=(-1, 2, 1, -2))),
        ("sep_strip_down2_t3_negpad", "sae_upfirdn2d_separable", "fir_sep_strip_kernel<3,3,16,2>",
         dict(shape=(1, 19, 17, 4), t=3, up=1, down=2, pad=(-2, 1, 0, -1))),
        ("sep_up2_t4_negpad", "sae_upfirdn2d_separable", "fir_sep_up2_kernel<4,4>",
         dict(shape=(1, 8, 9, 8), t=4, up=2, down=1, pad=(-1, 0, -2, 1))),
        ("tma33_ragged", "sae_upfirdn2d_separable", "fir_tma_kernel<3,3,0>",
         dict(shape=(2, 21, 19, 64), t=3, up=1, down=1, pad=(1, 1, 1, 1))),
        ("tma44_ragged", "sae_upfirdn2d_separable", "fir_tma_kernel<4,4,0>",
         dict(shape=(2, 20, 23, 32), t=4, up=1, down=1, pad=(2, 1, 1, 2))),
        ("tma33_8x8", "sae_upfirdn2d_separable", "fir_tma_kernel<3,3,0>",
         dict(shape=(2, 8, 8, 32), t=3, up=1, down=1, pad=(1, 1, 1, 1))),
        ("tma44_8x8", "sae_upfirdn2d_separable", "fir_tma_kernel<4,4,0>",
         dict(shape=(1, 8, 8, 32), t=4, up=1, down=1, pad=(2, 1, 2, 1))),
        ("tma44_negpad", "sae_upfirdn2d_separable", "fir_tma_kernel<4,4,0>",
         dict(shape=(1, 14, 13, 32), t=4, up=1, down=1, pad=(-1, 1, -2, 2))),
        # sae_fir_act_backward (MODE 1)
        ("fir_act_bwd_t3_actout_c32", "sae_fir_act_backward", "fir_tma_kernel<3,3,1>",
         dict(shape=(2, 21, 19, 32), t=3, pad=(1, 1, 1, 1), mask=False)),
        ("fir_act_bwd_t4_mask_c96", "sae_fir_act_backward", "fir_tma_kernel<4,4,1>",
         dict(shape=(2, 18, 21, 96), t=4, pad=(1, 2, 2, 1), mask=True)),
        ("fir_act_bwd_t3_mask_c32", "sae_fir_act_backward", "fir_tma_kernel<3,3,1>",
         dict(shape=(1, 9, 10, 32), t=3, pad=(0, 1, 1, 0), mask=True)),
        ("fir_act_bwd_t4_actout_c96", "sae_fir_act_backward", "fir_tma_kernel<4,4,1>",
         dict(shape=(1, 11, 8, 96), t=4, pad=(2, 1, 1, 2), mask=False)),
        # sae_fir_bias_act (MODE 2)
        ("fir_bias_act_t3_bias_noise_c32", "sae_fir_bias_act", "fir_tma_kernel<3,3,2>",
         dict(shape=(2, 21, 19, 32), t=3, pad=(1, 1, 1, 1), bias=True, noise=True)),
        ("fir_bias_act_t4_bias_c96", "sae_fir_bias_act", "fir_tma_kernel<4,4,2>",
         dict(shape=(1, 18, 21, 96), t=4, pad=(2, 1, 1, 2), bias=True, noise=False)),
        ("fir_bias_act_t4_noise_c32", "sae_fir_bias_act", "fir_tma_kernel<4,4,2>",
         dict(shape=(2, 9, 10, 32), t=4, pad=(1, 2, 2, 1), bias=False, noise=True)),
        ("fir_bias_act_t3_plain_c96", "sae_fir_bias_act", "fir_tma_kernel<3,3,2>",
         dict(shape=(1, 8, 8, 96), t=3, pad=(1, 1, 1, 1), bias=False, noise=False)),
    ]
    return rows


def _pointwise_rows():
    F4, F1 = "bias_act_kernel<4,unsigned int>", "bias_act_kernel<1,unsigned int>"
    B4, B1 = "bias_act_bwd_kernel<4>", "bias_act_bwd_kernel<1>"
    rows = [
        # sae_fused_bias_act: (shape, bias, act, grad, noise, storage offset)
        ("ba_f4_c64", "sae_fused_bias_act", F4, dict(shape=(2, 5, 7, 64))),
        ("ba_f4_c4", "sae_fused_bias_act", F4, dict(shape=(3, 5, 4))),
        ("ba_f4_c3_wrap", "sae_fused_bias_act", F4, dict(shape=(8, 3))),
        ("ba_f4_c2", "sae_fused_bias_act", F4, dict(shape=(6, 2))),
        ("ba_c1", "sae_fused_bias_act", F1, dict(shape=(12, 1))),
        ("ba_c1_nhwc", "sae_fused_bias_act", F1, dict(shape=(2, 4, 6, 1))),
        ("ba_c1_grad1", "sae_fused_bias_act", F1, dict(shape=(16, 1), grad=1)),
        ("ba_scalar_c5", "sae_fused_bias_act", F1, dict(shape=(6, 5))),
        ("ba_scalar_misaligned_c64", "sae_fused_bias_act", F1, dict(shape=(3, 64), offset=1)),
        ("ba_scalar_noise_c6", "sae_fused_bias_act", F1, dict(shape=(2, 3, 5, 6), noise=True)),
        ("ba_f4_noise_c64", "sae_fused_bias_act", F4, dict(shape=(2, 3, 5, 64), noise=True)),
        ("ba_f4_grad1_bias", "sae_fused_bias_act", F4, dict(shape=(4, 5, 32), grad=1)),
        ("ba_f4_grad1_nobias", "sae_fused_bias_act", F4, dict(shape=(4, 5, 32), grad=1, bias=False)),
        ("ba_f4_grad2", "sae_fused_bias_act", F4, dict(shape=(4, 8), grad=2)),
        ("ba_f4_linear", "sae_fused_bias_act", F4, dict(shape=(4, 5, 32), act=1)),
        ("ba_scalar_linear_nobias", "sae_fused_bias_act", F1, dict(shape=(7, 3), act=1, bias=False)),
        # NCHW bias (step_b = H * W) through the C ABI: the channel changes inside a float4 (H * W = 6) or not (H * W = 16)
        ("ba_f4_stepb6", "sae_fused_bias_act", F4, dict(shape=(2, 5, 2, 3), nchw=True)),
        ("ba_f4_stepb16", "sae_fused_bias_act", F4, dict(shape=(2, 3, 4, 4), nchw=True)),
        ("ba_scalar_stepb6", "sae_fused_bias_act", F1, dict(shape=(1, 5, 2, 3), nchw=True, offset=1)),
        # sae_bias_act_backward
        ("bab_f4_out", "sae_bias_act_backward", B4, dict(shape=(2, 6, 5, 64))),
        ("bab_f4_mask", "sae_bias_act_backward", B4, dict(shape=(2, 6, 5, 64), mask=True)),
        ("bab_scalar_c5", "sae_bias_act_backward", B1, dict(shape=(7, 3, 5))),
        ("bab_scalar_misaligned_c64", "sae_bias_act_backward", B1, dict(shape=(3, 5, 64), offset=1)),
        ("bab_f4_noise", "sae_bias_act_backward", B4, dict(shape=(2, 6, 5, 32), noise=True)),
        ("bab_f4_mask_noise", "sae_bias_act_backward", B4, dict(shape=(2, 6, 5, 32), noise=True, mask=True)),
        ("bab_scalar_noise_c6", "sae_bias_act_backward", B1, dict(shape=(2, 4, 5, 6), noise=True)),
        ("bab_f4_nobias", "sae_bias_act_backward", B4, dict(shape=(2, 6, 5, 64), want_bias=False)),
        ("bab_f4_c12000", "sae_bias_act_backward", B4, dict(shape=(8, 12000))),
        # sae_modulate(_backward)
        ("mod_f4", "sae_modulate", "modulate_kernel<unsigned int>", dict(shape=(2, 5, 7, 64))),
        ("mod_scalar_c3", "sae_modulate", "modulate_scalar_kernel", dict(shape=(2, 5, 7, 3))),
        ("mod_scalar_s_misaligned", "sae_modulate", "modulate_scalar_kernel", dict(shape=(2, 5, 7, 64), s_offset=1)),
        ("modb_f4_narrow", "sae_modulate_backward", "modulate_bwd_kernel<4>", dict(shape=(2, 6, 5, 64), branch="narrow")),
        ("modb_f4_wide_c2048", "sae_modulate_backward", "modulate_bwd_kernel<4>", dict(shape=(2, 4, 4, 2048), branch="wide")),
        ("modb_scalar_narrow_c5", "sae_modulate_backward", "modulate_bwd_kernel<1>", dict(shape=(2, 6, 5, 5), branch="narrow")),
        ("modb_scalar_wide_c1027", "sae_modulate_backward", "modulate_bwd_kernel<1>", dict(shape=(2, 3, 4, 1027), branch="wide")),
        ("modb_f4_misaligned_dy", "sae_modulate_backward", "modulate_bwd_kernel<1>",
         dict(shape=(2, 3, 4, 64), branch="narrow", offset=1)),
        ("modb_f4_ragged_chunk", "sae_modulate_backward", "modulate_bwd_kernel<4>", dict(shape=(2, 9, 13, 64), branch="narrow")),
        ("modb_f4_n1_many_chunks", "sae_modulate_backward", "modulate_bwd_kernel<4>", dict(shape=(1, 64, 64, 32), branch="narrow")),
        # add_scale, x2 bilinear upsample + merge, reflect pad
        ("add_scale_f4", "sae_add_scale", "add_scale_kernel<4>", dict(n=1024, b=True)),
        ("add_scale_f4_nob", "sae_add_scale", "add_scale_kernel<4>", dict(n=1024, b=False)),
        ("add_scale_scalar_n7", "sae_add_scale", "add_scale_kernel<1>", dict(n=7, b=True)),
        ("add_scale_scalar_n7_nob", "sae_add_scale", "add_scale_kernel<1>", dict(n=7, b=False)),
        ("ups_fwd_h1_w5", "sae_upsample2x_add_scale", "upsample2x_add_kernel", dict(shape=(2, 1, 5, 4))),
        ("ups_fwd_h2_w1", "sae_upsample2x_add_scale", "upsample2x_add_kernel", dict(shape=(2, 2, 1, 4))),
        ("ups_fwd_h2_w2", "sae_upsample2x_add_scale", "upsample2x_add_kernel", dict(shape=(1, 2, 2, 4))),
        ("ups_fwd_h5_w6_c8", "sae_upsample2x_add_scale", "upsample2x_add_kernel", dict(shape=(2, 5, 6, 8))),
        ("ups_bwd_h1_w5", "sae_upsample2x_backward", "upsample2x_bwd_kernel", dict(shape=(2, 1, 5, 4))),
        ("ups_bwd_h2_w1", "sae_upsample2x_backward", "upsample2x_bwd_kernel", dict(shape=(2, 2, 1, 4))),
        ("ups_bwd_h2_w2", "sae_upsample2x_backward", "upsample2x_bwd_kernel", dict(shape=(1, 2, 2, 4))),
        ("ups_bwd_h5_w6_c8", "sae_upsample2x_backward", "upsample2x_bwd_kernel", dict(shape=(2, 5, 6, 8))),
        # pads = (left, right, top, bottom); H - 1 / W - 1 is the largest reflection
        ("reflect_pad_max_lt", "sae_reflect_pad", "reflect_pad_kernel", dict(shape=(2, 5, 7, 8), pads=(6, 2, 4, 1))),
        ("reflect_pad_max_rb", "sae_reflect_pad", "reflect_pad_kernel", dict(shape=(1, 5, 7, 4), pads=(1, 6, 0, 4))),
        ("reflect_pad_bwd_max_lt", "sae_reflect_pad_backward", "reflect_pad_bwd_kernel", dict(shape=(2, 5, 7, 8), pads=(6, 2, 4, 1))),
        ("reflect_pad_bwd_max_rb", "sae_reflect_pad_backward", "reflect_pad_bwd_kernel", dict(shape=(1, 5, 7, 4), pads=(1, 6, 0, 4))),
        ("pad_channels_nchw", "sae_pad_channels", "pad_channels_kernel", dict(shape=(2, 3, 5, 7), c_out=32)),
        ("pad_channels_strided", "sae_pad_channels", "pad_channels_kernel", dict(shape=(2, 3, 5, 7), c_out=8, channels_last=True)),
        # filter preparation
        ("filter_prep_crsk", "sae_filter_prep", "filter_prep_kernel", dict(shape=(6, 5, 3, 3), crsk=True)),
        ("filter_prep_krsc_only", "sae_filter_prep", "filter_prep_kernel", dict(shape=(4, 7, 1, 1), crsk=False)),
        ("filter_modulate_both", "sae_filter_modulate", "filter_modulate_kernel", dict(n=3, shape=(6, 3, 3, 5))),
        ("filter_unprep", "sae_filter_unprep", "filter_unprep_kernel", dict(shape=(6, 3, 3, 5))),
        ("split_tf32_edges", "sae_split_tf32", "split_tf32_kernel", dict()),
        ("bucket_pack", "sae_bucket_pack", "bucket_copy_kernel", dict(sizes=(1, 3, 4, 5, 1000003))),
        ("bucket_unpack_half", "sae_bucket_unpack", "bucket_copy_kernel", dict(sizes=(1, 3, 4, 5, 1000003), scale=0.5)),
        ("bucket_unpack_third", "sae_bucket_unpack", "bucket_copy_kernel", dict(sizes=(1, 3, 4, 5, 1000003), scale=1 / 3)),
    ]
    return rows


def _train_rows():
    rows = []
    # ToRGB: NJ = ceil(C / 128) rounded up to 1, 2, 4, 8; C = 4, 132, 260, 1020 leave lanes idle in every instantiation
    for nj, c in ((1, 4), (2, 132), (4, 260), (8, 1020)):
        rows.append(("torgb_fwd_nj%d_c%d" % (nj, c), "sae_torgb_forward", "torgb_fwd_kernel<%d>" % nj,
                     dict(n=2, hw=(15, 17), c=c)))
        rows.append(("torgb_bwd_nj%d_c%d" % (nj, c), "sae_torgb_backward", "torgb_bwd_kernel<%d>" % nj,
                     dict(n=2, hw=(15, 17), c=c, dy_layout="channels_last" if nj in (2, 8) else "nchw")))
    rows += [
        ("torgb_fwd_one_strip_tail", "sae_torgb_forward", "torgb_fwd_kernel<1>", dict(n=3, hw=(5, 7), c=64)),
        ("torgb_fwd_nobias", "sae_torgb_forward", "torgb_fwd_kernel<2>", dict(n=1, hw=(9, 10), c=256, bias=False)),
        ("torgb_bwd_one_strip_tail", "sae_torgb_backward", "torgb_bwd_kernel<1>", dict(n=3, hw=(5, 7), c=64, dy_layout="nchw")),
        ("torgb_bwd_dx_only", "sae_torgb_backward", "torgb_bwd_kernel<2>", dict(n=2, hw=(6, 6), c=256, dy_layout="channels_last",
                                                                                  want_gw=False)),
        ("torgb_bwd_gw_only", "sae_torgb_backward", "torgb_bwd_kernel<4>", dict(n=2, hw=(6, 6), c=512, dy_layout="nchw",
                                                                                  want_dx=False)),
        # crops: (B, num_crops, C, H, W, S, flips); Q * S * S is never a multiple of 32 here (partial last warp)
        ("crop_s2_one_crop_c3", "sae_crop_gather", "crop_gather_kernel",
         dict(b=2, num_crops=1, c=3, h=12, w=20, s=2, flip="mixed")),
        ("crop_s9_flip_overhang_c1", "sae_crop_gather", "crop_gather_kernel",
         dict(b=1, num_crops=3, c=1, h=12, w=20, s=9, flip="all", overhang=True)),
        ("crop_s17_c4", "sae_crop_gather", "crop_gather_kernel",
         dict(b=2, num_crops=2, c=4, h=12, w=20, s=17, flip="mixed", overhang=True, strided=True)),
        ("crop_bwd_s2_one_crop_c3", "sae_crop_gather_backward", "crop_gather_bwd_kernel",
         dict(b=2, num_crops=1, c=3, h=12, w=20, s=2, flip="mixed")),
        ("crop_bwd_s9_flip_overhang_c1", "sae_crop_gather_backward", "crop_gather_bwd_kernel",
         dict(b=1, num_crops=3, c=1, h=12, w=20, s=9, flip="all", overhang=True)),
        ("crop_bwd_s17_c4", "sae_crop_gather_backward", "crop_gather_bwd_kernel",
         dict(b=2, num_crops=2, c=4, h=12, w=20, s=17, flip="mixed", overhang=True)),
        # Adam: the float4 / scalar loop is a branch inside adam_kernel (n % 4 == 0 and 16-byte aligned p and g)
        ("adam_f4", "sae_adam_step", ("adam_kernel", "adam_advance_kernel"),
         dict(sizes=(64, 1024), branches=("float4", "float4"), grad_scale=1.0)),
        ("adam_scalar_odd", "sae_adam_step", ("adam_kernel", "adam_advance_kernel"),
         dict(sizes=(7, 33), branches=("scalar", "scalar"), grad_scale=1.0)),
        ("adam_scalar_offset1_gscale", "sae_adam_step", ("adam_kernel", "adam_advance_kernel"),
         dict(sizes=(64, 16), offsets=(1, 0), branches=("scalar", "float4"), grad_scale=0.5)),
        ("adam_null_grad_gscale", "sae_adam_step", ("adam_kernel", "adam_advance_kernel"),
         dict(sizes=(12, 40, 5), null=(1,), branches=("float4", None, "scalar"), grad_scale=1 / 3)),
    ]
    return rows


ROWS = _fir_rows() + _pointwise_rows() + _train_rows()
ROW_BY_ID = {r[0]: r for r in ROWS}


def kernel_name(raw):
    """normalised kernel name: no 'void', namespace, argument list, '(int)' casts or blanks"""
    s = raw.replace("(int)", "")
    s = s.split("(", 1)[0]
    s = re.sub(r"^\s*void\s+", "", s).replace("sae::", "")
    return re.sub(r"\s+", "", s)


def expected_kernels(row):
    exp = row[2]
    return {kernel_name(e) for e in ((exp,) if isinstance(exp, str) else exp)}


# --------------------------------------------------------------------------------------------------------- helpers
@pytest.fixture
def kern():
    from swapping_autoencoder_pytorch_b200 import backend
    k = backend.kernels()
    prev = (k.precision, k.round_tf32, k.act_masks, k.fused_fir_act)
    k.precision, k.round_tf32, k.act_masks, k.fused_fir_act = "tf32", False, True, True
    yield k
    k.precision, k.round_tf32, k.act_masks, k.fused_fir_act = prev


def _own_kernels(prof):
    names = set()
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        raw = e.name
        if "at::" in raw or "native::" in raw or raw.startswith(("Memcpy", "Memset")):
            continue
        names.add(kernel_name(raw))
    return names


def _profiled(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, _own_kernels(prof)


class Observer:
    """runs a call under torch.profiler and collects the device kernels it launched (``seen``, a set of normalised names).
    The profiler can deliver a kernel's activity record to the next profiling session instead of its own, so a session
    that drains stale records runs first, and up to three draining sessions collect late records of the row's kernels."""

    def __init__(self, row):
        self.expected = expected_kernels(row)
        self.seen = set()

    def __call__(self, fn):
        _profiled(lambda: None)
        out, seen = _profiled(fn)
        for _ in range(3):
            if self.expected <= seen:
                break
            seen |= _profiled(lambda: None)[1]
        self.seen |= seen
        return out


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _check_rc(kern, rc, what):
    from swapping_autoencoder_pytorch_b200._lib import check
    check(rc, what)


def f32(v):
    return float(np.float32(v))


def dev_f32(t64, offset=0):
    """fp32 device copy of a float64 tensor; offset > 0: the same values at that storage offset (a misaligned view)"""
    flat = t64.reshape(-1).float()
    buf = torch.empty(flat.numel() + offset, dtype=torch.float32, device=DEV)
    buf[offset:].copy_(flat)
    return buf[offset:].view(t64.shape)


def guarded(t64):
    """fp32 device copy of a short vector, followed in storage by SENTINEL values: a read past its end shows"""
    flat = t64.reshape(-1).float()
    buf = torch.full((flat.numel() + 8,), SENTINEL, dtype=torch.float32, device=DEV)
    buf[:flat.numel()].copy_(flat)
    return buf[:flat.numel()].view(t64.shape)


def r32(seed, *shape, scale=1.0):
    """seeded normal values, as float64 copies of fp32 numbers"""
    return (rnd(seed, *shape) * scale).float().double()


def assert_bound(got, ref, mag, c, what):
    """|got - ref| <= c * 2^-24 * mag per element (NaN or a missing element fails)"""
    got = got.detach().double().cpu().reshape(ref.shape)
    err = (got - ref).abs()
    bound = c * U * mag
    bad = ~(err <= bound)
    if bad.any():
        i = int(bad.reshape(-1).nonzero()[0])
        excess = float(((err - bound) / mag.clamp_min(1e-300)).reshape(-1)[bad.reshape(-1)].max())
        raise AssertionError("%s: %d of %d elements exceed %g * 2^-24 * sum|terms| (first at %d: got %r, ref %r, bound %r; worst "
                             "excess %.3g relative to sum|terms|)" % (what, int(bad.sum()), bad.numel(), c, i,
                                                                    float(got.reshape(-1)[i]), float(ref.reshape(-1)[i]),
                                                                    float(bound.reshape(-1)[i]), excess))


def assert_bits(got, ref32, what):
    """bit equality of two fp32 tensors"""
    a = got.detach().contiguous().cpu().view(torch.int32).reshape(-1)
    b = ref32.detach().float().contiguous().cpu().view(torch.int32).reshape(-1)
    same = a == b
    assert same.all(), "%s: %d of %d elements differ bitwise (first at %d)" % (what, int((~same).sum()), same.numel(),
                                                                              int((~same).nonzero()[0]))


def mask_words(pos):
    """activation bit mask of a boolean NHWC tensor (bit e & 31 of word e >> 5), as int32 words"""
    bits = pos.reshape(-1, 32).to(torch.int64)
    w = (bits << torch.arange(32, dtype=torch.int64, device=bits.device)).sum(1)
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)


def check_mask(words, z, zbound, what):
    """every bit equals z > 0 (z: fp64 pre-activation, NHWC order) outside max(zbound, 1e-6 max|z|) of zero; < 1 % exempt"""
    w = words.cpu().to(torch.int64) & 0xFFFFFFFF
    bits = ((w[:, None] >> torch.arange(32)) & 1).reshape(-1).bool()
    zf, zb = z.reshape(-1), zbound.reshape(-1)
    assert bits.numel() == zf.numel()
    band = zf.abs() <= torch.maximum(zb, 1e-6 * zf.abs().max())
    assert band.double().mean() < 0.01, "%s: %.3f of the pre-activations lie in the exempt band" % (what, float(band.double().mean()))
    bad = (bits != (zf > 0)) & ~band
    assert not bad.any(), "%s: %d mask bits disagree with fp64 (first at %d)" % (what, int(bad.sum()), int(bad.nonzero()[0]))


def nchw(t):
    return t.permute(0, 3, 1, 2)


def nhwc(t):
    return t.permute(0, 2, 3, 1)


def fir64(x_nhwc, k, up=(1, 1), down=(1, 1), pad=(0, 0, 0, 0)):
    """(FIR, FIR of magnitudes) in fp64 by the oracle's direct summation; NHWC in, NHWC out"""
    xn = nchw(x_nhwc).numpy()
    kn = np.asarray(k, dtype=np.float64)
    ref = O.fir_numpy(xn, kn, up=up, down=down, pad=pad)
    mag = O.fir_numpy(np.abs(xn), np.abs(kn), up=up, down=down, pad=pad)
    return nhwc(torch.from_numpy(np.ascontiguousarray(ref))), nhwc(torch.from_numpy(np.ascontiguousarray(mag)))


def _seed(row):
    return sum(map(ord, row[0]))


def _ctaps(taps):
    return (ctypes.c_float * len(taps))(*taps)


# ------------------------------------------------------------------------------------------------------------ FIR
def run_upfirdn2d(kern, row, obs):
    a = row[3]
    s = _seed(row)
    x = r32(s, *a["shape"])
    kh, kw = a["k"]
    k = r32(s + 1, kh, kw)
    n, h, w, c = a["shape"]
    (ux, uy), (dx, dy), (px0, px1, py0, py1) = a["up"], a["down"], a["pad"]
    oh = (h * uy + py0 + py1 - kh) // dy + 1
    ow = (w * ux + px0 + px1 - kw) // dx + 1
    xd = dev_f32(x, a.get("offset", 0))
    out = torch.full((n, oh, ow, c), float("nan"), device=DEV)
    obs(lambda: _check_rc(kern, kern.lib.sae_upfirdn2d(_p(xd), _p(dev_f32(k)), _p(out), n, h, w, c, kh, kw, ux, uy, dx, dy,
                                                        px0, px1, py0, py1, 0, _stream()), "sae_upfirdn2d"))
    ref, mag = fir64(x, k, up=(ux, uy), down=(dx, dy), pad=a["pad"])
    assert_bound(out, ref, mag, kh * kw + 2, row[0])


def _sep_ref(x, t, tx, up, down, pad):
    k = np.outer(np.asarray(TAPS[t]), np.asarray(tx))
    return fir64(x, k, up=(up, up), down=(down, down), pad=pad)


def run_upfirdn2d_separable(kern, row, obs):
    a = row[3]
    s = _seed(row)
    x = r32(s, *a["shape"])
    t, up, down = a["t"], a["up"], a["down"]
    px0, px1, py0, py1 = a["pad"]
    n, h, w, c = a["shape"]
    oh = (h * up + py0 + py1 - t) // down + 1
    ow = (w * up + px0 + px1 - t) // down + 1
    xd = dev_f32(x)
    out = torch.full((n, oh, ow, c), float("nan"), device=DEV)
    obs(lambda: _check_rc(kern, kern.lib.sae_upfirdn2d_separable(_p(xd), _ctaps(TAPS[t]), _ctaps(TAPS_X[t]), _p(out), n, h, w, c,
                                                                  t, t, up, down, px0, px1, py0, py1, 0, _stream()),
                          "sae_upfirdn2d_separable"))
    ref, mag = _sep_ref(x, t, TAPS_X[t], up, down, a["pad"])
    assert_bound(out, ref, mag, t * t + 2 * t + 2, row[0])


def _tma_geometry(a):
    n, h, w, c = a["shape"]
    t = a["t"]
    px0, px1, py0, py1 = a["pad"]
    return n, h, w, c, t, (px0, px1, py0, py1), h + py0 + py1 - t + 1, w + px0 + px1 - t + 1


def run_fir_act_backward(kern, row, obs):
    a = row[3]
    s = _seed(row)
    n, h, w, c, t, pad, oh, ow = _tma_geometry(a)
    grad = r32(s, n, h, w, c)
    act = r32(s + 1, n, oh, ow, c)
    alpha, scale = f32(0.2), f32(SQRT2)
    gd, act_d = dev_f32(grad), dev_f32(act)
    gi = torch.full((n, oh, ow, c), float("nan"), device=DEV)
    gb = torch.zeros(c, device=DEV)
    mask = None
    if a["mask"]:
        # the kernel must read the mask, not act_out: the mask here is the sign of a different tensor
        sign_src = r32(s + 2, n, oh, ow, c)
        mask = mask_words(sign_src > 0).to(DEV)
        pos = sign_src > 0
    else:
        pos = act > 0
    obs(lambda: _check_rc(kern, kern.lib.sae_fir_act_backward(_p(gd), _ctaps(TAPS[t]), _ctaps(TAPS_X[t]), _p(act_d), _p(gi), _p(gb),
                                                               n, h, w, c, t, t, *pad, alpha, scale, 0, _p(mask), _stream()),
                          "sae_fir_act_backward"))
    g, mag = _sep_ref(grad, t, TAPS_X[t], 1, 1, pad)
    factor = torch.where(pos, scale, alpha * scale)
    cf = t * t + 2 * t + 4
    assert_bound(gi, g * factor, mag * factor, cf, row[0] + " grad_in")
    npix = n * oh * ow
    assert_bound(gb, (g * factor).sum((0, 1, 2)), (mag * factor).sum((0, 1, 2)), cf + npix, row[0] + " grad_bias")


def run_fir_bias_act(kern, row, obs):
    a = row[3]
    s = _seed(row)
    n, h, w, c, t, pad, oh, ow = _tma_geometry(a)
    x = r32(s, n, h, w, c)
    alpha, scale = f32(0.2), f32(SQRT2)
    bias = r32(s + 1, c) if a["bias"] else None
    noise = r32(s + 2, n, oh, ow) if a["noise"] else None
    nw = torch.tensor([f32(0.37)], dtype=torch.float64) if a["noise"] else None
    xd = dev_f32(x)
    out = torch.full((n, oh, ow, c), float("nan"), device=DEV)
    words = torch.full((n * oh * ow * c // 32,), -0x5A5A5A5B, dtype=torch.int32, device=DEV)
    bd = guarded(bias) if bias is not None else None
    nd = dev_f32(noise) if noise is not None else None
    nwd = guarded(nw) if nw is not None else None
    obs(lambda: _check_rc(kern, kern.lib.sae_fir_bias_act(_p(xd), _ctaps(TAPS[t]), _ctaps(TAPS_X[t]), _p(bd), _p(nd), _p(nwd), _p(out),
                                                           n, h, w, c, t, t, *pad, alpha, scale, 0, _p(words), _stream()),
                          "sae_fir_bias_act"))
    f, mag = _sep_ref(x, t, TAPS_X[t], 1, 1, pad)
    z, zmag = f.clone(), mag.clone()
    if bias is not None:
        z, zmag = z + bias, zmag + bias.abs()
    if noise is not None:
        z, zmag = z + float(nw) * noise[..., None], zmag + abs(float(nw)) * noise.abs()[..., None]
    cf = t * t + 2 * t + 6
    ref = torch.where(z > 0, z, z * alpha) * scale
    assert_bound(out, ref, zmag * scale, cf, row[0])
    check_mask(words, z, cf * U * zmag, row[0] + " mask")


# -------------------------------------------------------------------------------------------------- bias / activation
def run_fused_bias_act(kern, row, obs):
    a = row[3]
    s = _seed(row)
    shape = a["shape"]
    x = r32(s, *shape)
    nchw_bias = a.get("nchw", False)
    c = shape[1] if nchw_bias else shape[-1]
    step_b = int(np.prod(shape[2:])) if nchw_bias else 1
    bias = r32(s + 1, c) if a.get("bias", True) else None
    act, grad = a.get("act", 3), a.get("grad", 0)
    alpha, scale = f32(0.2), f32(SQRT2)
    ref_t = r32(s + 2, *shape) if grad == 1 else None
    noise = nw = None
    if a.get("noise"):
        noise = r32(s + 3, x.numel() // c)
        nw = torch.tensor([f32(-0.61)], dtype=torch.float64)
    xd = dev_f32(x, a.get("offset", 0))
    out = torch.full(shape, float("nan"), device=DEV)
    bd = guarded(bias) if bias is not None else None
    rd = dev_f32(ref_t) if ref_t is not None else None
    nd = dev_f32(noise) if noise is not None else None
    nwd = guarded(nw) if nw is not None else None
    obs(lambda: _check_rc(kern, kern.lib.sae_fused_bias_act(_p(xd), _p(bd), _p(rd), _p(out), x.numel(), step_b,
                                                             c if bias is not None else 1, act, grad, alpha, scale, _p(nd), _p(nwd),
                                                             c, 0, _stream()), "sae_fused_bias_act"))
    flat = x.reshape(-1)
    e = torch.arange(flat.numel())
    t, tmag = flat.clone(), flat.abs()
    if bias is not None:
        ch = (e // step_b) % c
        t, tmag = t + bias[ch], tmag + bias.abs()[ch]
    if noise is not None:
        nz = float(nw) * noise[e // c]
        t, tmag = t + nz, tmag + nz.abs()
    if act == 3:
        sign = ref_t.reshape(-1) if grad == 1 else t
        y = torch.where(sign > 0, t, t * alpha)
    else:
        y = t
    ref = torch.zeros_like(y) if grad == 2 else y * scale
    assert_bound(out.reshape(-1), ref, tmag * scale, 5, row[0])


def run_bias_act_backward(kern, row, obs):
    from swapping_autoencoder_pytorch_b200 import backend
    a = row[3]
    s = _seed(row)
    shape = a["shape"]
    c = shape[-1]
    go = r32(s, *shape)
    outv = r32(s + 1, *shape)
    alpha, scale = f32(0.2), f32(SQRT2)
    god, outd = dev_f32(go, a.get("offset", 0)), dev_f32(outv)
    mask = None
    pos = outv > 0
    if a.get("mask"):
        sign_src = r32(s + 2, *shape)            # the kernel must read the mask, not out
        mask = mask_words(sign_src > 0).to(DEV)
        pos = sign_src > 0
    noise = r32(s + 3, go.numel() // c) if a.get("noise") else None
    want_bias = a.get("want_bias", True)
    nd = dev_f32(noise) if noise is not None else None
    res = obs(lambda: backend.kernels().bias_act_backward(god, outd, alpha, scale, want_bias=want_bias, noise=nd, mask=mask))
    gi, gb, gnw = res
    factor = torch.where(pos, scale, alpha * scale)
    ref_gi = go * factor
    mag_gi = go.abs() * factor
    assert_bound(gi, ref_gi, mag_gi, 3, row[0] + " grad_in")
    rows = go.numel() // c
    if want_bias:
        assert_bound(gb, ref_gi.reshape(-1, c).sum(0), mag_gi.reshape(-1, c).sum(0), rows + 4, row[0] + " grad_bias")
    else:
        assert gb is None
    if noise is not None:
        per = ref_gi.reshape(-1, c) * noise[:, None]
        mag = (mag_gi.reshape(-1, c) * noise.abs()[:, None]).sum()
        assert_bound(gnw, per.sum().reshape(1), mag.reshape(1), go.numel() + 4, row[0] + " grad_noise_weight")


def _mod_branch(c, dy, x, dx):
    """mirror of sae_modulate_backward's choice: float4 when C % 4 == 0 and dy, x, dx are 16-byte aligned; the narrow
    loop when the 256 threads cover the channel groups, the wide one otherwise"""
    vec = c % 4 == 0 and all(t.data_ptr() % 16 == 0 for t in (dy, x, dx))
    return "narrow" if 256 // (c // 4 if vec else c) > 0 else "wide"


def run_modulate(kern, row, obs):
    a = row[3]
    s = _seed(row)
    n, h, w, c = a["shape"]
    x = r32(s, n, h, w, c)
    sv = r32(s + 1, n, c, scale=0.5) + 1
    sv = sv.float().double()
    xd = dev_f32(x)
    sd = dev_f32(sv, a.get("s_offset", 0))
    out = torch.full((n, h, w, c), float("nan"), device=DEV)
    obs(lambda: _check_rc(kern, kern.lib.sae_modulate(_p(xd), _p(sd), _p(out), n, h * w, c, 0, _stream()), "sae_modulate"))
    assert_bits(out, (x * sv[:, None, None, :]).float(), row[0])


def run_modulate_backward(kern, row, obs):
    a = row[3]
    s = _seed(row)
    n, h, w, c = a["shape"]
    dy = r32(s, n, h, w, c)
    x = r32(s + 1, n, h, w, c)
    sv = (r32(s + 2, n, c, scale=0.5) + 1).float().double()
    dyd, xd, sd = dev_f32(dy, a.get("offset", 0)), dev_f32(x), guarded(sv)
    dx = torch.full((n, h, w, c), float("nan"), device=DEV)
    ds = torch.zeros((n, c), device=DEV)
    assert _mod_branch(c, dyd, xd, dx) == a["branch"], row[0]
    obs(lambda: _check_rc(kern, kern.lib.sae_modulate_backward(_p(dyd), _p(xd), _p(sd), _p(dx), _p(ds), n, h * w, c, 0, _stream()),
                          "sae_modulate_backward"))
    assert_bits(dx, (dy * sv[:, None, None, :]).float(), row[0] + " dx")
    assert_bound(ds, (dy * x).sum((1, 2)), (dy * x).abs().sum((1, 2)), h * w + 2, row[0] + " ds")


# ------------------------------------------------------------------------------------------ merges, resampling, pads
def run_add_scale(kern, row, obs):
    a = row[3]
    s = _seed(row)
    n = a["n"]
    av = r32(s, n)
    bv = r32(s + 1, n) if a["b"] else None
    scale = f32(1 / SQRT2)
    ad, bd = dev_f32(av), (dev_f32(bv) if bv is not None else None)
    out = torch.full((n,), float("nan"), device=DEV)
    obs(lambda: _check_rc(kern, kern.lib.sae_add_scale(_p(ad), _p(bd), _p(out), n, scale, 0, _stream()), "sae_add_scale"))
    if bv is None:
        assert_bits(out, (av * scale).float(), row[0])
    else:
        assert_bound(out, (av + bv) * scale, (av.abs() + bv.abs()) * scale, 2, row[0])


def _interp(t64):
    return F.interpolate(t64, scale_factor=2, mode="bilinear", align_corners=False)


def run_upsample2x_add_scale(kern, row, obs):
    a = row[3]
    s = _seed(row)
    n, h, w, c = a["shape"]
    skip = r32(s, n, h, w, c)
    res = r32(s + 1, n, 2 * h, 2 * w, c)
    scale = f32(1 / SQRT2)
    sd, rd = dev_f32(skip), dev_f32(res)
    out = torch.full((n, 2 * h, 2 * w, c), float("nan"), device=DEV)
    obs(lambda: _check_rc(kern, kern.lib.sae_upsample2x_add_scale(_p(sd), _p(rd), _p(out), n, h, w, c, scale, 0, _stream()),
                          "sae_upsample2x_add_scale"))
    ref = (nhwc(_interp(nchw(skip))) + res) * scale
    mag = (nhwc(_interp(nchw(skip.abs()))) + res.abs()) * scale
    assert_bound(out, ref, mag, 8, row[0])


def run_upsample2x_backward(kern, row, obs):
    a = row[3]
    s = _seed(row)
    n, h, w, c = a["shape"]
    dy = r32(s, n, 2 * h, 2 * w, c)
    scale = f32(1 / SQRT2)
    dyd = dev_f32(dy)
    out = torch.full((n, h, w, c), float("nan"), device=DEV)
    obs(lambda: _check_rc(kern, kern.lib.sae_upsample2x_backward(_p(dyd), _p(out), n, h, w, c, scale, 0, _stream()),
                          "sae_upsample2x_backward"))

    def adj(g):
        z = torch.zeros(n, c, h, w, dtype=torch.float64, requires_grad=True)
        gz, = torch.autograd.grad((_interp(z) * nchw(g)).sum(), z)
        return nhwc(gz) * scale
    assert_bound(out, adj(dy), adj(dy.abs()), 16 + 2, row[0])


def run_reflect_pad(kern, row, obs):
    a = row[3]
    s = _seed(row)
    n, h, w, c = a["shape"]
    pl, pr, pt, pb = a["pads"]
    x = r32(s, n, h, w, c)
    xd = dev_f32(x)
    out = torch.full((n, h + pt + pb, w + pl + pr, c), float("nan"), device=DEV)
    obs(lambda: _check_rc(kern, kern.lib.sae_reflect_pad(_p(xd), _p(out), n, h, w, c, pl, pr, pt, pb, _stream()), "sae_reflect_pad"))
    assert_bits(out, nhwc(F.pad(nchw(x), (pl, pr, pt, pb), mode="reflect")), row[0])


def run_reflect_pad_backward(kern, row, obs):
    a = row[3]
    s = _seed(row)
    n, h, w, c = a["shape"]
    pl, pr, pt, pb = a["pads"]
    dy = r32(s, n, h + pt + pb, w + pl + pr, c)
    dyd = dev_f32(dy)
    dx = torch.full((n, h, w, c), float("nan"), device=DEV)
    obs(lambda: _check_rc(kern, kern.lib.sae_reflect_pad_backward(_p(dyd), _p(dx), n, h, w, c, pl, pr, pt, pb, _stream()),
                          "sae_reflect_pad_backward"))

    def adj(g):
        z = torch.zeros(n, c, h, w, dtype=torch.float64, requires_grad=True)
        gz, = torch.autograd.grad((F.pad(z, (pl, pr, pt, pb), mode="reflect") * nchw(g)).sum(), z)
        return nhwc(gz)
    assert_bound(dx, adj(dy), adj(dy.abs()), 9 + 1, row[0])


def run_pad_channels(kern, row, obs):
    a = row[3]
    s = _seed(row)
    n, c, h, w = a["shape"]
    x = r32(s, n, c, h, w)
    xd = dev_f32(x)
    if a.get("channels_last"):
        xd = xd.contiguous(memory_format=torch.channels_last)
    c_out = a["c_out"]
    out = torch.full((n, h, w, c_out), float("nan"), device=DEV)
    obs(lambda: _check_rc(kern, kern.lib.sae_pad_channels(_p(xd), _p(out), n, h * w, c, c_out, xd.stride(0), xd.stride(1), xd.stride(3),
                                                           0, _stream()), "sae_pad_channels"))
    assert_bits(out, F.pad(nhwc(x), (0, c_out - c)), row[0])


def run_filter_prep(kern, row, obs):
    a = row[3]
    s = _seed(row)
    k, c, r, s_ = a["shape"]
    wv = r32(s, k, c, r, s_)
    scale = f32(1 / math.sqrt(c * r * s_))
    wd = dev_f32(wv)
    krsc = torch.full((k, r, s_, c), float("nan"), device=DEV)
    crsk = torch.full((c, r, s_, k), float("nan"), device=DEV) if a["crsk"] else None
    obs(lambda: _check_rc(kern, kern.lib.sae_filter_prep(_p(wd), _p(krsc), _p(crsk), k, c, r, s_, scale, 0, _stream()),
                          "sae_filter_prep"))
    ref = (wv * scale).float()
    assert_bits(krsc, ref.permute(0, 2, 3, 1), row[0] + " krsc")
    if crsk is not None:
        assert_bits(crsk, ref.permute(1, 2, 3, 0), row[0] + " crsk")


def run_filter_modulate(kern, row, obs):
    a = row[3]
    s = _seed(row)
    n = a["n"]
    k, r, s_, c = a["shape"]
    wv = r32(s, k, r, s_, c)
    sv = (r32(s + 1, n, c, scale=0.5) + 1).float().double()
    wd, sd = dev_f32(wv), guarded(sv)
    o1 = torch.full((n, k, r, s_, c), float("nan"), device=DEV)
    o2 = torch.full((n, c, r, s_, k), float("nan"), device=DEV)
    obs(lambda: _check_rc(kern, kern.lib.sae_filter_modulate(_p(wd), _p(sd), _p(o1), _p(o2), n, k, c, r, s_, 0, _stream()),
                          "sae_filter_modulate"))
    ref = (wv[None] * sv[:, None, None, None, :]).float()
    assert_bits(o1, ref, row[0] + " krsc")
    assert_bits(o2, ref.permute(0, 4, 2, 3, 1), row[0] + " crsk")


def run_filter_unprep(kern, row, obs):
    a = row[3]
    s = _seed(row)
    k, r, s_, c = a["shape"]
    g = r32(s, k, r, s_, c)
    scale = f32(1 / math.sqrt(c * r * s_))
    gd = dev_f32(g)
    out = torch.full((k, c, r, s_), float("nan"), device=DEV)
    obs(lambda: _check_rc(kern, kern.lib.sae_filter_unprep(_p(gd), _p(out), k, c, r, s_, scale, _stream()), "sae_filter_unprep"))
    assert_bits(out, (g * scale).float().permute(0, 3, 1, 2), row[0])


def rna_bits(bits):
    """round-to-nearest, ties away, to TF32 on int32 bit patterns (finite inputs)"""
    return (bits + 0x1000) & ~0x1FFF


def run_split_tf32(kern, row, obs):
    rs = np.random.RandomState(_seed(row))
    pats = [0x00000000, 0x00000001, 0x00000FFF, 0x00001000, 0x00001FFF, 0x00003000, 0x007FF000, 0x007FFFFF,
            0x00800000, 0x00801000, 0x00800FFF, 0x00803000, 0x3F801000, 0x3F800FFF, 0x3F803000, 0x3F802FFF,
            0x3FFFF000, 0x3FFFFFFF, 0x7E000000, 0x7E801000, 0x7F000FFF, 0x7F7FE000, 0x7F7FEFFF, 0x0B801001]
    pats += list(rs.randint(0x00800000, 0x7F000000, size=200))              # random normals
    pats += list(rs.randint(0x00000001, 0x00800000, size=40))               # random subnormals
    pats += [(p & ~0x1FFF) | 0x1000 for p in rs.randint(0x00800000, 0x7F000000, size=40)]   # exact ties
    pos = torch.tensor(pats, dtype=torch.int64)
    bits = torch.cat([pos, pos | 0x80000000])
    bits = torch.where(bits >= 2 ** 31, bits - 2 ** 32, bits).to(torch.int32)
    x = bits.view(torch.float32)
    xd = x.to(DEV)
    hi = torch.full_like(xd, float("nan"))
    lo = torch.full_like(xd, float("nan"))
    obs(lambda: _check_rc(kern, kern.lib.sae_split_tf32(_p(xd), _p(hi), _p(lo), x.numel(), _stream()), "sae_split_tf32"))
    hi_ref = rna_bits(bits).view(torch.float32)
    assert_bits(hi, hi_ref, row[0] + " hi")
    d = x - hi_ref                                      # exact in fp32
    lo_ref = rna_bits(d.view(torch.int32)).view(torch.float32)
    assert_bits(lo, lo_ref, row[0] + " lo")
    # the pair carries ~22 significant bits wherever lo is a normal number
    x64 = x.double()
    big = x64.abs() >= 2.0 ** -100
    err = (hi.double().cpu() + lo.double().cpu() - x64).abs()
    assert (err[big] <= 2.0 ** -22 * x64.abs()[big]).all()


def _bucket_layout(sizes):
    offsets, total = [], 0
    for sz in sizes:
        offsets.append(total)
        total += (sz + 3) // 4 * 4            # parallel.GradientBucket._layout: every segment 16-byte aligned
    return offsets, total


BUCKET_SENTINEL = -0x3E3E3E3F                  # an int32 bit pattern no copy produces


def run_bucket(kern, row, obs):
    from swapping_autoencoder_pytorch_b200 import backend
    a = row[3]
    s = _seed(row)
    sizes = a["sizes"]
    offsets, total = _bucket_layout(sizes)
    k = backend.kernels()
    # every tensor is the head of a buffer with sentinel words behind it
    bufs = [torch.full((sz + 4,), BUCKET_SENTINEL, dtype=torch.int32, device=DEV).view(torch.float32) for sz in sizes]
    ts = [b[:sz] for b, sz in zip(bufs, sizes)]
    ptrs = torch.tensor([t.data_ptr() for t in ts], dtype=torch.int64, device=DEV)
    off_t = torch.tensor(offsets, dtype=torch.int64, device=DEV)
    size_t = torch.tensor(sizes, dtype=torch.int64, device=DEV)
    bucket = torch.full((total,), BUCKET_SENTINEL, dtype=torch.int32, device=DEV).view(torch.float32)
    if row[1] == "sae_bucket_pack":
        for i, t in enumerate(ts):
            t.copy_(r32(s + i, t.numel()).float())
        obs(lambda: k.bucket_pack(ptrs, off_t, size_t, len(ts), bucket))
        ref = torch.full((total,), BUCKET_SENTINEL, dtype=torch.int32).view(torch.float32)
        for o, t in zip(offsets, ts):
            ref[o:o + t.numel()] = t.cpu()
        assert_bits(bucket, ref, row[0] + " bucket (padding slots untouched)")
        return
    src = r32(s, total).float()
    bucket.copy_(src)
    scale = a["scale"]
    obs(lambda: k.bucket_unpack(ptrs, off_t, size_t, len(ts), bucket, scale))
    for i, (o, sz) in enumerate(zip(offsets, sizes)):
        # one correctly rounded product: the fp64 product of two fp32 numbers is exact
        want = (src[o:o + sz].double() * f32(scale)).float()
        assert_bits(ts[i], want, "%s tensor %d" % (row[0], i))
        assert (bufs[i][sz:].view(torch.int32) == BUCKET_SENTINEL).all(), "%s: tensor %d written past its end" % (row[0], i)


# ------------------------------------------------------------------------------------------------------------- ToRGB
def _torgb_operands(row):
    a = row[3]
    s = _seed(row)
    n, (h, w), c = a["n"], a["hw"], a["c"]
    x = r32(s, n, h, w, c)
    sv = (r32(s + 1, n, c, scale=0.5) + 1).float().double()
    wv = r32(s + 2, 3, c)
    bias = r32(s + 3, 3) if a.get("bias", True) else None
    wscale = f32(1 / math.sqrt(c))
    # wc[n, o, c] = fl(fl(s * wscale) * w): the combined weights the kernel forms in fp32
    sw = (sv * wscale).float().double()
    wc = (sw[:, None, :] * wv[None]).float().double()
    return n, h, w, c, x, sv, wv, bias, wscale, wc


def run_torgb_forward(kern, row, obs):
    n, h, w, c, x, sv, wv, bias, wscale, wc = _torgb_operands(row)
    xd, sd, wd = dev_f32(x), guarded(sv), guarded(wv)
    bd = guarded(bias) if bias is not None else None
    y = torch.full((n, h, w, 4), float("nan"), device=DEV)
    obs(lambda: _check_rc(kern, kern.lib.sae_torgb_forward(_p(xd), _p(sd), _p(wd), _p(bd), _p(y), n, h, w, c, wscale, 0, _stream()),
                          "sae_torgb_forward"))
    ref = torch.einsum("nhwc,noc->nhwo", x, wc)
    mag = torch.einsum("nhwc,noc->nhwo", x.abs(), wc.abs())
    if bias is not None:
        ref, mag = ref + bias, mag + bias.abs()
    assert_bound(y[..., :3], ref, mag, c + 4, row[0])
    assert_bits(y[..., 3], torch.zeros(n, h, w), row[0] + " channel 3")


def run_torgb_backward(kern, row, obs):
    a = row[3]
    n, h, w, c, x, sv, wv, _, wscale, wc = _torgb_operands(row)
    dy = r32(_seed(row) + 4, n, 3, h, w)
    if a["dy_layout"] == "channels_last":
        buf = torch.full((n, h, w, 4), float("nan"), device=DEV)
        buf[..., :3] = dev_f32(nhwc(dy).contiguous())
        dyd = buf.permute(0, 3, 1, 2)[:, :3]
    else:
        dyd = dev_f32(dy)
    xd, sd, wd = dev_f32(x), guarded(sv), guarded(wv)
    want_dx, want_gw = a.get("want_dx", True), a.get("want_gw", True)
    dx = torch.full((n, h, w, c), float("nan"), device=DEV) if want_dx else None
    gw = torch.zeros((n, 3, c), device=DEV) if want_gw else None
    obs(lambda: _check_rc(kern, kern.lib.sae_torgb_backward(_p(dyd), _p(xd), _p(sd), _p(wd), _p(dx), _p(gw), n, h, w, c, wscale,
                                                             *dyd.stride(), 0, _stream()), "sae_torgb_backward"))
    if want_dx:
        ref = torch.einsum("nohw,noc->nhwc", dy, wc)
        mag = torch.einsum("nohw,noc->nhwc", dy.abs(), wc.abs())
        assert_bound(dx, ref, mag, 3 + 2, row[0] + " dx")
    if want_gw:
        ref = torch.einsum("nohw,nhwc->noc", dy, x)
        mag = torch.einsum("nohw,nhwc->noc", dy.abs(), x.abs())
        assert_bound(gw, ref, mag, h * w + 2, row[0] + " gw")


# ------------------------------------------------------------------------------------------------------------- crops
def _crop_operands(row):
    """crop parameters on a dyadic grid: every sampling coordinate is exact in fp32 and fp64 alike, so the fp64 reference
    samples at the kernel's coordinates and only the bilinear sums differ"""
    a = row[3]
    rs = np.random.RandomState(_seed(row))
    q = a["b"] * a["num_crops"]
    if a["flip"] == "all":
        flip = -np.ones(q)
    else:
        flip = np.where(np.arange(q) % 2 == 0, 1.0, -1.0)
    if a.get("overhang"):
        scale = rs.randint(12, 21, size=(q, 2)) / 16.0          # up to 1.25: crops reach past the image
        offset = rs.randint(-40, 41, size=(q, 2)) / 128.0
    else:
        scale = rs.randint(6, 15, size=(q, 2)) / 16.0
        offset = rs.randint(-12, 13, size=(q, 2)) / 128.0
    return q, torch.tensor(flip), torch.tensor(scale), torch.tensor(offset)


def _crop_grid(q, flip, scale, offset, num_crops, s):
    lin = torch.linspace(-1, 1, s, dtype=torch.float64)
    gx = (lin[None, None, :] * flip[:, None, None]) * scale[:, 0, None, None] + offset[:, 0, None, None]
    gy = lin[None, :, None] * scale[:, 1, None, None] + offset[:, 1, None, None]
    return torch.stack(torch.broadcast_tensors(gx, gy), dim=-1)          # [Q, S, S, 2] = (x, y)


def _sample(x64, grid, num_crops):
    src = x64.repeat_interleave(num_crops, dim=0)
    return F.grid_sample(src, grid, mode="bilinear", padding_mode="zeros", align_corners=False)


def run_crop_gather(kern, row, obs):
    from swapping_autoencoder_pytorch_b200 import backend
    a = row[3]
    b, nc, c, h, w, s = a["b"], a["num_crops"], a["c"], a["h"], a["w"], a["s"]
    q, flip, scale, offset = _crop_operands(row)
    x = r32(_seed(row), b, c, h, w)
    xd = dev_f32(x)
    if a.get("strided"):
        xd = xd.contiguous(memory_format=torch.channels_last)
    out = torch.full((q, s, s, 32), float("nan"), device=DEV)
    fd, sd, od = guarded(flip), guarded(scale), guarded(offset)
    obs(lambda: backend.kernels().crop_gather(xd, fd, sd, od, nc, s, 32, out=out))
    grid = _crop_grid(q, flip, scale, offset, nc, s)
    ref = nhwc(_sample(x, grid, nc))
    mag = nhwc(_sample(x.abs(), grid, nc))
    assert_bound(out[..., :c], ref, mag, 4 + 2, row[0])
    assert_bits(out[..., c:], torch.zeros(q, s, s, 32 - c), row[0] + " zero padding")


def run_crop_gather_backward(kern, row, obs):
    from swapping_autoencoder_pytorch_b200 import backend
    a = row[3]
    b, nc, c, h, w, s = a["b"], a["num_crops"], a["c"], a["h"], a["w"], a["s"]
    q, flip, scale, offset = _crop_operands(row)
    dy = r32(_seed(row) + 1, q, c, s, s)
    buf = torch.full((q, s, s, 32), float("nan"), device=DEV)              # the padded NHWC layout the patch discriminator uses
    buf[..., :c] = dev_f32(nhwc(dy).contiguous())
    dyd = buf.permute(0, 3, 1, 2)
    fd, sd, od = guarded(flip), guarded(scale), guarded(offset)
    dx = obs(lambda: backend.kernels().crop_gather_backward(dyd, fd, sd, od, nc, c, h, w))
    grid = _crop_grid(q, flip, scale, offset, nc, s)

    def adj(g):
        z = torch.zeros(b, c, h, w, dtype=torch.float64, requires_grad=True)
        gz, = torch.autograd.grad((_sample(z, grid, nc) * g).sum(), z)
        return gz
    # terms per input pixel: per crop, the output rows (columns) whose bilinear foot covers it are at most 2 / step + 1
    # apart, step = the crop's source spacing in pixels; the kernel also adds the zero-weight neighbours of that range
    step_y = (scale[:, 1] * (2.0 / (s - 1)) * h / 2).min()
    step_x = (scale[:, 0] * (2.0 / (s - 1)) * w / 2).min()
    terms = nc * (math.ceil(2 / float(step_y)) + 2) * (math.ceil(2 / float(step_x)) + 2)
    assert_bound(dx, adj(dy), adj(dy.abs()), terms + 2, row[0])


# -------------------------------------------------------------------------------------------------------------- Adam
def _adam_ref_step(p, g, m, v, t, lr, b1, b2, eps, gs):
    """one torch.optim.Adam step in fp64 from the kernel's previous fp32 state; returns values and error bounds"""
    gr = g * gs
    m1 = m + (1 - b1) * (gr - m)
    v1 = b2 * v + (1 - b2) * gr * gr
    bc1 = 1 - b1 ** t
    bc2s = math.sqrt(1 - b2 ** t)
    den = v1.sqrt() / bc2s + eps
    upd = lr / bc1 * m1 / den
    p1 = p - upd
    bm = 5 * U * (m.abs() + (1 - b1) * (gr.abs() + m.abs()))
    bv = 6 * U * v1
    # the kernel's bias corrections 1 - powf(beta, t) cancel: a powf error of <= 4 ulp becomes 4u / (1 - beta^t) relative
    rel = U * (5 / (1 - b1 ** t) + 2.5 / (1 - b2 ** t) + 12) + 0.5 * bv / v1.clamp_min(1e-300)
    bp = 2 * U * p.abs() + upd.abs() * rel + lr / bc1 * bm / den
    return p1, m1, v1, bm, bv, bp


def _adam_branch(p, g):
    """mirror of adam_kernel's loop choice"""
    return "float4" if p.numel() % 4 == 0 and p.data_ptr() % 16 == 0 and g.data_ptr() % 16 == 0 else "scalar"


def run_adam(kern, row, obs):
    from swapping_autoencoder_pytorch_b200 import backend
    a = row[3]
    s = _seed(row)
    sizes = a["sizes"]
    offs = a.get("offsets", (0,) * len(sizes))
    null = set(a.get("null", ()))
    lr, b1, b2, eps = f32(2e-3), f32(0.5), f32(0.99), f32(1e-8)
    gs = f32(a["grad_scale"])
    params = []
    for i, (sz, o) in enumerate(zip(sizes, offs)):
        buf = torch.zeros(sz + o, device=DEV)
        buf[o:] = r32(s + i, sz).float().to(DEV)
        params.append(buf[o:])
    layout = [0]
    for sz in sizes:
        layout.append(layout[-1] + (sz + 3) // 4 * 4)
    total = layout[-1]
    exp_avg = torch.zeros(total, device=DEV)
    exp_avg_sq = torch.zeros(total, device=DEV)
    steps = torch.zeros(len(sizes), device=DEV)
    off_t = torch.tensor(layout[:-1], dtype=torch.int64, device=DEV)
    size_t = torch.tensor(sizes, dtype=torch.int64, device=DEV)
    cache = backend.PointerTables(len(sizes), torch.device(DEV))
    for step in range(1, 4):
        grads = [None if i in null else (r32(s + 100 * step + i, sz) * 0.1).float().to(DEV) for i, sz in enumerate(sizes)]
        for i, (p, g) in enumerate(zip(params, grads)):
            assert (_adam_branch(p, g) if g is not None else None) == a["branches"][i], (row[0], i)
        before = [(p.double().cpu(), exp_avg[o:o + sz].double().cpu(), exp_avg_sq[o:o + sz].double().cpu())
                  for p, o, sz in zip(params, layout, sizes)]
        before_bits = [(p.clone(), exp_avg[o:o + sz].clone(), exp_avg_sq[o:o + sz].clone()) for p, o, sz in zip(params, layout, sizes)]
        obs(lambda: kern.adam_step(params, grads, off_t, size_t, exp_avg, exp_avg_sq, steps, lr, b1, b2, eps, gs, cache))
        for i, (p, o, sz) in enumerate(zip(params, layout, sizes)):
            what = "%s step %d tensor %d" % (row[0], step, i)
            m_k, v_k = exp_avg[o:o + sz], exp_avg_sq[o:o + sz]
            if i in null:
                for t, t0 in zip((p, m_k, v_k), before_bits[i]):
                    assert_bits(t, t0, what + " (no gradient: untouched)")
                continue
            p0, m0, v0 = before[i]
            p1, m1, v1, bm, bv, bp = _adam_ref_step(p0, grads[i].double().cpu(), m0, v0, step, lr, b1, b2, eps, gs)
            assert_bound(m_k, m1, bm / U, 1, what + " exp_avg")
            assert_bound(v_k, v1, bv / U, 1, what + " exp_avg_sq")
            assert_bound(p, p1, bp / U, 1, what + " param")
    want_steps = torch.tensor([0.0 if i in null else 3.0 for i in range(len(sizes))])
    assert torch.equal(steps.cpu(), want_steps), steps


RUNNERS = {
    "sae_upfirdn2d": run_upfirdn2d,
    "sae_upfirdn2d_separable": run_upfirdn2d_separable,
    "sae_fir_act_backward": run_fir_act_backward,
    "sae_fir_bias_act": run_fir_bias_act,
    "sae_fused_bias_act": run_fused_bias_act,
    "sae_bias_act_backward": run_bias_act_backward,
    "sae_modulate": run_modulate,
    "sae_modulate_backward": run_modulate_backward,
    "sae_add_scale": run_add_scale,
    "sae_upsample2x_add_scale": run_upsample2x_add_scale,
    "sae_upsample2x_backward": run_upsample2x_backward,
    "sae_reflect_pad": run_reflect_pad,
    "sae_reflect_pad_backward": run_reflect_pad_backward,
    "sae_pad_channels": run_pad_channels,
    "sae_filter_prep": run_filter_prep,
    "sae_filter_modulate": run_filter_modulate,
    "sae_filter_unprep": run_filter_unprep,
    "sae_split_tf32": run_split_tf32,
    "sae_bucket_pack": run_bucket,
    "sae_bucket_unpack": run_bucket,
    "sae_torgb_forward": run_torgb_forward,
    "sae_torgb_backward": run_torgb_backward,
    "sae_crop_gather": run_crop_gather,
    "sae_crop_gather_backward": run_crop_gather_backward,
    "sae_adam_step": run_adam,
}


@pytest.mark.parametrize("row_id", [r[0] for r in ROWS])
def test_bandwidth_path(kern, row_id):
    row = ROW_BY_ID[row_id]
    obs = Observer(row)
    try:
        RUNNERS[row[1]](kern, row, obs)
    except AssertionError as e:
        raise AssertionError("%s [kernels launched: %s]" % (e, sorted(obs.seen))) from None
    assert obs.seen == expected_kernels(row), "%s launched %s, expected %s" % (row_id, sorted(obs.seen), sorted(expected_kernels(row)))
