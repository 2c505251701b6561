"""GPU (H100): the fused conv epilogue (``sae_conv_epilogue``: bias, NoiseInjection, leaky-ReLU, gain, residual merge, TF32
rounding, activation bit mask) on every launch path of the forward and data-gradient convolutions, against fp64.

Each case names the kernel path it must take and asserts it: the wgmma kernel at BLOCK_N 128 / 64 / 32, several images per
pixel tile, 1x1, the stride-2 data gradient's parity classes (four non-empty, and R or S == 1 where some classes receive no
tap), the transposed-convolution geometry, per-sample filters, and the generic mma.sync kernel's loaders, its three store
paths (float4 staging, float2, scalar) and split-K.  For every case and epilogue variant:

* values: rounding off, TF32-representable conv operands (products exact), arbitrary fp32 epilogue operands, against
  F.conv2d in fp64 followed by the header's epilogue formula in fp64, 2e-5 max-norm relative;
* rounding: with ``round_tf32`` the output is ``rna_tf32`` of the unrounded output, bit for bit (split-K, whose fp32
  atomics sum in a varying order: TF32-representable and within 2^-11 |ref| + 2e-5 max |ref| of fp64);
* kernel agreement: impl = 0, 1 and 2 agree within 2e-5 where both kernels take the shape;
* activation mask: every bit equals ``conv + bias + nw * noise > 0`` in fp64 (elements within 1e-4 max of zero exempt; fewer
  than 1 % may be), the data gradient's buffer pre-filled with a sentinel so unwritten words show.

A subset also runs in the fp32 precision mode (split-TF32 kernels, nothing rounded on storage) on arbitrary fp32 operands."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.fixtures import rel_err, rnd
from swapping_autoencoder_pytorch_b200 import backend
from swapping_autoencoder_pytorch_b200.backend import make_geom

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = 2e-5
SENTINEL = -0x5A5A5A5B          # 0xA5A5A5A5 as an int32


def tf32(t):
    """round-to-nearest (ties away) to TF32, as a float64 tensor — what cvt.rna.tf32.f32 does to an fp32 value"""
    bits = t.float().contiguous().view(torch.int32)
    return ((bits + 0x1000) & ~0x1FFF).view(torch.float32).double()


def rna_bits(t):
    """the int32 bit patterns of rna_tf32(t) for an fp32 tensor"""
    return (t.contiguous().view(torch.int32) + 0x1000) & ~0x1FFF


def f32(v):
    return float(np.float32(v))


@pytest.fixture
def kern():
    k = backend.kernels()
    prev = (k.conv_impl, k.precision, k.round_tf32, k.act_masks)
    k.conv_impl, k.precision, k.round_tf32, k.act_masks = 0, "tf32", True, True
    yield k
    k.conv_impl, k.precision, k.round_tf32, k.act_masks = prev


# ------------------------------------------------------------------------------------------------ the path table
# (id, direction, geometry args of make_geom, P/Q override or None, impl passed, expected path)
#   direction: "fprop" / "dgrad" / "fprop_ps" / "dgrad_ps" (per-sample filters)
#   path: "wgmma", "generic:<store>" with store in float4 / float2 / scalar, "splitk"
CASES = [
    ("wg_fprop_bn128", "fprop", (2, 16, 16, 64, 128, 3, 3, 1, 1, 1), None, 0, "wgmma"),
    ("wg_fprop_bn64_ragged", "fprop", (2, 19, 21, 64, 192, 3, 3, 1, 1, 1), None, 0, "wgmma"),
    ("wg_fprop_bn32_stride2", "fprop", (3, 17, 17, 32, 96, 3, 3, 2, 0, 0), None, 0, "wgmma"),
    ("wg_fprop_images_per_tile", "fprop", (8, 4, 4, 64, 64, 3, 3, 1, 1, 1), None, 0, "wgmma"),
    ("wg_fprop_1x1", "fprop", (2, 32, 32, 32, 128, 1, 1, 1, 0, 0), None, 0, "wgmma"),
    ("wg_dgrad_stride1", "dgrad", (2, 16, 16, 64, 128, 3, 3, 1, 1, 1), None, 0, "wgmma"),
    ("wg_dgrad_stride2_4cls", "dgrad", (2, 33, 33, 64, 128, 3, 3, 2, 0, 0), None, 0, "wgmma"),
    ("wg_dgrad_stride2_1x1", "dgrad", (2, 16, 16, 64, 128, 1, 1, 2, 0, 0), None, 0, "wgmma"),
    ("wg_dgrad_stride2_1x1_odd", "dgrad", (2, 15, 15, 64, 64, 1, 1, 2, 0, 0), None, 0, "wgmma"),
    ("wg_dgrad_stride2_3x1", "dgrad", (2, 16, 16, 64, 64, 3, 1, 2, 1, 0), None, 0, "wgmma"),
    ("wg_dgrad_transposed", "dgrad", (2, 17, 17, 64, 128, 3, 3, 2, 0, 0), (8, 8), 0, "wgmma"),
    ("wg_fprop_per_sample", "fprop_ps", (2, 32, 32, 64, 128, 3, 3, 1, 1, 1), None, None, "wgmma"),
    ("wg_dgrad_per_sample", "dgrad_ps", (2, 32, 32, 64, 128, 3, 3, 1, 1, 1), None, None, "wgmma"),
    ("gen_fprop_forced", "fprop", (2, 16, 16, 64, 128, 3, 3, 1, 1, 1), None, 1, "generic:float4"),
    ("gen_dgrad_forced", "dgrad", (2, 16, 16, 64, 128, 3, 3, 1, 1, 1), None, 1, "generic:float4"),
    ("gen_dgrad_stride2_1x1_forced", "dgrad", (2, 16, 16, 64, 128, 1, 1, 2, 0, 0), None, 1, "generic:float4"),
    ("gen_fprop_c3", "fprop", (2, 12, 12, 3, 32, 3, 3, 1, 1, 1), None, 0, "generic:float4"),
    ("gen_fprop_k6", "fprop", (2, 10, 10, 16, 6, 3, 3, 1, 1, 1), None, 0, "generic:float2"),
    ("gen_fprop_k5", "fprop", (2, 10, 10, 16, 5, 3, 3, 1, 1, 1), None, 0, "generic:scalar"),
    ("gen_fprop_k3", "fprop", (2, 9, 11, 8, 3, 3, 3, 1, 1, 1), None, 0, "generic:scalar"),
    ("gen_dgrad_c6", "dgrad", (2, 10, 10, 6, 16, 3, 3, 1, 1, 1), None, 0, "generic:float2"),
    ("gen_dgrad_c3_stride2", "dgrad", (2, 11, 11, 3, 16, 3, 3, 2, 0, 0), None, 0, "generic:scalar"),
    # linears as stylegan2_op/conv.py::linear issues them: 1x1 maps, always the generic kernel
    ("splitk_linear_fprop", "fprop", (16, 1, 1, 2048, 512, 1, 1, 1, 0, 0), None, 1, "splitk"),
    ("splitk_linear_dgrad", "dgrad", (16, 1, 1, 2048, 512, 1, 1, 1, 0, 0), None, 1, "splitk"),
]
CASE_BY_ID = {c[0]: c for c in CASES}

SQRT2 = math.sqrt(2)
VARIANTS = {
    "none": {},
    "bias_lrelu": dict(bias=True, act=3, alpha=0.2, gain=SQRT2),
    "bias_lrelu_noise": dict(bias=True, act=3, alpha=0.2, gain=SQRT2, noise=True),
    "residual": dict(residual=True, res_scale=1 / SQRT2),
    "all": dict(bias=True, act=3, alpha=0.2, gain=SQRT2, noise=True, residual=True, res_scale=1 / SQRT2),
    "bias_linear": dict(bias=True, act=1, gain=1.7),
    "bias_only": dict(bias=True),          # the split-K rows' twin: any epilogue term turns split-K off
}
SPLITK_VARIANTS = ("none", "bias_only")
GENERAL_VARIANTS = ("none", "bias_lrelu", "bias_lrelu_noise", "residual", "all", "bias_linear")


def _geom(case):
    _, _, args, pq, _, _ = case
    if pq is None:
        return make_geom(*args)
    return make_geom(*args, P=pq[0], Q=pq[1])


def _is_dgrad(direction):
    return direction.startswith("dgrad")


def _out_dims(g, direction):
    """(N, channels, H, W) of the kernel's output and (M rows, output columns, reduction length) of its GEMM"""
    if _is_dgrad(direction):
        return (g.N, g.C, g.H, g.W), (g.N * g.H * g.W, g.C, g.R * g.S * g.K)
    return (g.N, g.K, g.P, g.Q), (g.N * g.P * g.Q, g.K, g.R * g.S * g.C)


def generic_store(ncol):
    """the generic kernel's store path for an output of ncol columns (conv_gather_kernel's epilogue)"""
    return "float4" if ncol % 4 == 0 else "float2" if ncol % 2 == 0 else "scalar"


def splitk_qualifies(g, direction, plain):
    """mirror of launch_gather's split-K rule: a plain epilogue, at most 16 CTAs, at least 16 k-blocks (and > 1 split)"""
    _, (m, ncol, kdim) = _out_dims(g, direction)
    bn = 128 if ncol > 64 else 64 if ncol > 32 else 32
    ctas = -(-m // 128) * -(-ncol // bn)
    kblocks = -(-kdim // 32)
    return plain and ctas <= 16 and kblocks >= 16 and min(kblocks // 4, 32) > 1


def _is_plain(spec):
    return not spec.get("bias") and not spec.get("noise") and not spec.get("residual") and spec.get("act", 1) == 1 \
        and spec.get("gain", 1.0) == 1.0


def _check_path(kern, case, spec):
    """asserts the case's kernel path; returns True when the call runs split-K.  Besides the linears, the generic rows of
    512 pixels and 576-long reductions split K too when the epilogue is plain (4 CTAs, 18 k-blocks)."""
    cid, direction, _, _, impl, path = case
    g = _geom(case)
    (_, ncol, _) = _out_dims(g, direction)[1]
    d = 1 if _is_dgrad(direction) else 0
    if direction.endswith("_ps"):
        assert kern.conv_modulated_ok(g), cid                      # only the wgmma kernel implements per-sample filters
        return False
    eligible = kern.conv_impl_for(g, d)
    if path == "wgmma":
        assert eligible == 2 and impl in (0, 2), cid
        return False
    assert eligible == (2 if impl == 1 else 1), cid                 # impl 1: forced onto the generic kernel a shape wgmma takes
    split = splitk_qualifies(g, direction, _is_plain(spec))
    if path == "splitk":
        assert split == _is_plain(spec), cid
    else:
        assert path == "generic:" + generic_store(ncol), (cid, generic_store(ncol))
    return split


# ------------------------------------------------------------------------------------------------ operands and reference
def _operands(case, fp32_operands=False):
    """conv operands (float64 NCHW / KCRS; TF32-representable unless fp32_operands) and per-sample styles"""
    cid, direction, _, _, _, _ = case
    g = _geom(case)
    seed = sum(map(ord, cid))
    q = (lambda t: t.float().double()) if fp32_operands else tf32
    wscale = 1 / math.sqrt(g.R * g.S * (g.K if _is_dgrad(direction) else g.C))
    w = q(rnd(seed + 1, g.K, g.C, g.R, g.S) * wscale)
    if _is_dgrad(direction):
        src = q(rnd(seed + 2, g.N, g.K, g.P, g.Q))
    else:
        src = q(rnd(seed + 2, g.N, g.C, g.H, g.W))
    s = (rnd(seed + 3, g.N, g.C) * 0.5 + 1.0) if direction.endswith("_ps") else None
    return g, src, w, s


def _epi_operands(case, spec):
    """arbitrary fp32 epilogue operands (float64 values of fp32 numbers), keyed by the conv_* keyword names"""
    cid, direction, _, _, _, _ = case
    g = _geom(case)
    (n, c, h, w), _ = _out_dims(g, direction)
    seed = 1000 + sum(map(ord, cid))
    e = {}
    if spec.get("bias"):
        e["bias"] = rnd(seed, c).float().double()
    if spec.get("noise"):
        e["noise"] = rnd(seed + 1, n, h, w).float().double()
        e["noise_weight"] = torch.tensor([f32(0.37)], dtype=torch.float64)
    if spec.get("residual"):
        e["residual"] = rnd(seed + 2, n, c, h, w).float().double()
    return e


def _conv_ref(case, g, src, w, per_sample_w=None):
    """the fp64 accumulator, NCHW.  per_sample_w: [N, K, C, R, S] filters (the ones the kernel read)"""
    _, direction, _, _, _, _ = case
    pad = (g.pad_t, g.pad_l)
    dgrad = _is_dgrad(direction)
    outs = []
    for i in range(g.N if per_sample_w is not None else 1):
        wi = (per_sample_w[i] if per_sample_w is not None else w).to(DEV)
        si = (src[i:i + 1] if per_sample_w is not None else src).to(DEV)
        if dgrad:
            x = torch.zeros(si.shape[0], g.C, g.H, g.W, dtype=torch.float64, device=DEV, requires_grad=True)
            y = F.conv2d(x, wi, stride=g.stride, padding=pad)
            assert tuple(y.shape[2:]) == (g.P, g.Q)
            out, = torch.autograd.grad((y * si).sum(), x)
        else:
            out = F.conv2d(si, wi, stride=g.stride, padding=pad)
            assert tuple(out.shape[2:]) == (g.P, g.Q)
        outs.append(out.cpu())
    return torch.cat(outs)


def _epi_ref(acc, spec, e):
    """the header's epilogue formula in fp64; returns (pre-activation z, output)"""
    z = acc.clone()
    if "bias" in e:
        z = z + e["bias"].view(1, -1, 1, 1)
    if "noise" in e:
        z = z + e["noise_weight"] * e["noise"][:, None]
    v = torch.where(z > 0, z, z * f32(spec["alpha"])) if spec.get("act", 1) == 3 else z
    v = v * f32(spec.get("gain", 1.0))
    if "residual" in e:
        v = (v + e["residual"]) * f32(spec["res_scale"])
    return z, v


def _nhwc(t):
    return t.float().to(DEV).permute(0, 2, 3, 1).contiguous()


def _run(kern, case, g, src, w, s, spec, e, round_tf32, impl=None, mask_buf=None):
    """one call of the case's entry point; returns (output NHWC fp32 on the device, mask words or None, per-sample filters)"""
    _, direction, _, _, case_impl, _ = case
    impl = case_impl if impl is None else impl
    kw = dict(round_tf32=round_tf32)
    if "bias" in e:
        kw["bias"] = e["bias"].float().to(DEV)
    if "noise" in e:
        kw["noise"] = e["noise"].float().to(DEV).reshape(-1).contiguous()
        kw["noise_weight"] = e["noise_weight"].float().to(DEV)
    if "residual" in e:
        kw["residual"] = _nhwc(e["residual"])
    for k in ("act", "alpha", "gain", "res_scale"):
        if k in spec:
            kw[k] = spec[k]
    w_krsc = w.float().to(DEV).permute(0, 2, 3, 1).contiguous()
    if direction == "fprop":
        y = kern.conv_fprop(_nhwc(src), w_krsc, g, impl=impl, **kw)
        return y, backend.act_mask_of(y), None
    if direction == "dgrad":
        if mask_buf is not None:
            kw["act_mask"] = mask_buf
        return kern.conv_dgrad(_nhwc(src), w_krsc, g, impl=impl, **kw), mask_buf, None
    s_dev = s.float().to(DEV)
    if direction == "fprop_ps":
        wn, _ = kern.filter_modulate(w_krsc, s_dev, want_krsc=True, want_crsk=False)
        y = kern.conv_fprop_per_sample(_nhwc(src), wn, g, **kw)
        return y, backend.act_mask_of(y), wn.double().cpu().permute(0, 1, 4, 2, 3)          # [N,K,C,R,S]
    _, wn = kern.filter_modulate(w_krsc, s_dev, want_krsc=False, want_crsk=True)
    if mask_buf is not None:
        kw["act_mask"] = mask_buf
    dx = kern.conv_dgrad_per_sample(_nhwc(src), wn, g, **kw)
    return dx, mask_buf, wn.double().cpu().permute(0, 4, 1, 2, 3)                             # [N,C,R,S,K] -> [N,K,C,R,S]


def _wants_mask(case, spec):
    """the wgmma kernels write the mask; the cases where the variant has an activation take one"""
    return case[5] == "wgmma" and spec.get("act", 1) == 3


def _new_mask_buf(case):
    g = _geom(case)
    (n, c, h, w), _ = _out_dims(g, case[1])
    return torch.full((n * c * h * w // 32,), SENTINEL, dtype=torch.int32, device=DEV)


def _check_mask(mask, z):
    """every bit of the mask words equals z > 0 (z: fp64 pre-activation, NCHW) outside a band of 1e-4 max|z| around 0"""
    assert mask is not None
    words = mask.cpu().to(torch.int64) & 0xFFFFFFFF
    bits = ((words[:, None] >> torch.arange(32)) & 1).reshape(-1).bool()
    zf = z.permute(0, 2, 3, 1).reshape(-1)
    assert bits.numel() == zf.numel()
    band = zf.abs() <= 1e-4 * zf.abs().max()
    assert band.float().mean() < 0.01, float(band.float().mean())
    bad = (bits != (zf > 0)) & ~band
    assert not bad.any(), "%d mask bits disagree with fp64 (first at %d)" % (int(bad.sum()), int(bad.nonzero()[0]))


def _nchw64(y):
    return y.permute(0, 3, 1, 2).double().cpu()


_ACC = {}


def _reference(case, g, src, w, per_sample_w):
    key = case[0]
    if per_sample_w is not None or key not in _ACC:
        acc = _conv_ref(case, g, src, w, per_sample_w)
        if per_sample_w is not None:
            return acc
        _ACC[key] = acc
    return _ACC[key]


PARAMS = [(c[0], v) for c in CASES for v in (SPLITK_VARIANTS if c[5] == "splitk" else GENERAL_VARIANTS)]


@pytest.mark.parametrize("case_id,variant", PARAMS)
def test_conv_epilogue_vs_fp64(kern, case_id, variant):
    case = CASE_BY_ID[case_id]
    spec = VARIANTS[variant]
    split = _check_path(kern, case, spec)
    g, src, w, s = _operands(case)
    e = _epi_operands(case, spec)
    want_mask = _wants_mask(case, spec)
    buf_off = _new_mask_buf(case) if want_mask else None
    off, mask_off, wn = _run(kern, case, g, src, w, s, spec, e, False, mask_buf=buf_off)
    acc = _reference(case, g, src, w, wn)
    z, ref = _epi_ref(acc, spec, e)
    assert rel_err(_nchw64(off), ref) < TOL, rel_err(_nchw64(off), ref)

    buf_on = _new_mask_buf(case) if want_mask else None
    on, mask_on, _ = _run(kern, case, g, src, w, s, spec, e, True, mask_buf=buf_on)
    on_bits = on.contiguous().view(torch.int32)
    if split:
        assert not (on_bits & 0x1FFF).any(), "split-K output with round_tf32 is not TF32-representable"
        err = (_nchw64(on) - ref).abs()
        bound = 2.0 ** -11 * ref.abs() + TOL * ref.abs().max()
        assert (err <= bound).all(), float((err - bound).max())
    else:
        same = on_bits == rna_bits(off)
        assert same.all(), "%d of %d elements differ from rna_tf32(unrounded output)" % (int((~same).sum()), same.numel())

    if want_mask:
        _check_mask(mask_off, z)
        _check_mask(mask_on, z)
        assert torch.equal(mask_on, mask_off)
    elif case[5] != "wgmma" and spec.get("act", 1) == 3 and case[1] == "fprop":
        assert mask_off is None          # the generic kernel writes no mask, and none is asked of it


AGREE_CASES = [c[0] for c in CASES if c[5] == "wgmma" and not c[1].endswith("_ps")]


@pytest.mark.parametrize("variant", GENERAL_VARIANTS)
@pytest.mark.parametrize("case_id", AGREE_CASES)
def test_conv_epilogue_impl_agreement(kern, case_id, variant):
    """the wgmma kernel (impl 2, and impl 0 which picks it) and the generic kernel (impl 1) compute the same epilogue"""
    case = CASE_BY_ID[case_id]
    spec = VARIANTS[variant]
    g, src, w, s = _operands(case)
    e = _epi_operands(case, spec)
    outs = {impl: _run(kern, case, g, src, w, s, spec, e, False, impl=impl)[0] for impl in (0, 1, 2)}
    assert rel_err(outs[1], outs[2]) < TOL, rel_err(outs[1], outs[2])
    assert rel_err(outs[0], outs[2]) < TOL, rel_err(outs[0], outs[2])


FP32_CASES = ["wg_fprop_bn128", "wg_fprop_bn64_ragged", "wg_fprop_bn32_stride2", "wg_dgrad_stride2_4cls",
              "wg_dgrad_stride2_1x1", "wg_fprop_per_sample", "wg_dgrad_per_sample", "gen_fprop_c3",
              "splitk_linear_fprop", "splitk_linear_dgrad"]


@pytest.mark.parametrize("case_id", FP32_CASES)
def test_conv_epilogue_fp32_mode(kern, case_id):
    """split-TF32 kernels (BLOCK_N 64 / 32 instantiations, the generic SPLIT kernel incl. split-K) with the full epilogue on
    arbitrary fp32 operands; the fp32 mode stores unrounded values even though the TF32 rounding policy is on"""
    case = CASE_BY_ID[case_id]
    variant = "none" if case[5] == "splitk" else "all"          # any epilogue term would turn split-K off
    spec = VARIANTS[variant]
    kern.precision = "fp32"
    g, src, w, s = _operands(case, fp32_operands=True)
    e = _epi_operands(case, spec)
    _check_path(kern, case, spec)
    y, _, wn = _run(kern, case, g, src, w, s, spec, e, None)
    _, ref = _epi_ref(_conv_ref(case, g, src, w, wn), spec, e)
    assert rel_err(_nchw64(y), ref) < TOL, rel_err(_nchw64(y), ref)
    assert (y.contiguous().view(torch.int32) & 0x1FFF).any(), "fp32 mode output was rounded to TF32"
