"""GPU (H100): the tap groups of the forward / data-gradient wgmma convolution (``tc_plan_groups`` in conv_wgmma.cu) against
fp64 ``F.conv2d``, one case per branch of the planner.

Taps with the same ox whose oy differ by stride * d share one A box of th + span rows, each tap reading its tile d * tw rows
into it; that needs one-image tiles of width 8 or 16, and every other tile falls back to one box of th rows per tap.  The
cases cover BLOCK_N 128 / 64 / 32, tw = 16 and tw = 8 tiles, zero-filled halo rows (pad 1), pad 0 and pad_t != pad_l, a
ragged last tile row, 3x3 stride 2, the stride-2 data gradient's parity classes (2-tap and 1-tap columns, and 1x1 with
classes no tap reaches), the several-images-per-tile fallback (8x8 and 4x4 maps) and per-sample filters.

* TF32 mode: TF32-representable operands (products exact), 2e-5 max-norm relative to fp64;
* fp32 mode (split-TF32 kernels): arbitrary fp32 operands, 2e-5;
* one reuse case with bias / noise / leaky-ReLU: values and every activation-mask bit against fp64;
* deterministic mode on a reuse case: bitwise equal from call to call."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle.fixtures import rel_err, rnd
from swapping_autoencoder_pytorch_b200 import backend
from swapping_autoencoder_pytorch_b200.backend import make_geom

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = 2e-5

# (id, direction, make_geom args (N, H, W, C, K, R, S, stride, pad_t, pad_l)); direction "fprop" / "dgrad" / "*_ps"
CASES = [
    ("fprop_bn128_tw16_pad1", "fprop", (2, 32, 32, 64, 128, 3, 3, 1, 1, 1)),
    ("fprop_bn64_ragged", "fprop", (2, 21, 37, 64, 192, 3, 3, 1, 1, 1)),
    ("fprop_bn32_tw8", "fprop", (2, 24, 8, 32, 96, 3, 3, 1, 1, 1)),
    ("fprop_pad0", "fprop", (2, 20, 20, 64, 64, 3, 3, 1, 0, 0)),
    ("fprop_pad_t2_l0", "fprop", (2, 18, 18, 64, 128, 3, 3, 1, 2, 0)),
    ("fprop_stride2_pad0", "fprop", (2, 33, 33, 64, 128, 3, 3, 2, 0, 0)),
    ("fprop_stride2_pad1", "fprop", (2, 32, 32, 32, 64, 3, 3, 2, 1, 1)),
    ("fprop_1x1_stride2", "fprop", (2, 31, 31, 64, 128, 1, 1, 2, 0, 0)),
    ("fprop_8x8_images_per_tile", "fprop", (4, 8, 8, 64, 128, 3, 3, 1, 1, 1)),
    ("fprop_4x4_images_per_tile", "fprop", (8, 4, 4, 64, 64, 3, 3, 1, 1, 1)),
    ("dgrad_bn128_tw16", "dgrad", (2, 32, 32, 128, 64, 3, 3, 1, 1, 1)),
    ("dgrad_bn64_tw8_ragged", "dgrad", (2, 20, 8, 64, 96, 3, 3, 1, 1, 1)),
    ("dgrad_pad_t0_l2", "dgrad", (2, 18, 18, 32, 64, 3, 3, 1, 0, 2)),
    ("dgrad_stride2_pad0", "dgrad", (2, 33, 33, 64, 128, 3, 3, 2, 0, 0)),
    ("dgrad_stride2_pad1", "dgrad", (2, 32, 32, 128, 64, 3, 3, 2, 1, 1)),
    ("dgrad_1x1_stride2", "dgrad", (2, 16, 16, 64, 128, 1, 1, 2, 0, 0)),
    ("dgrad_8x8_images_per_tile", "dgrad", (4, 8, 8, 64, 128, 3, 3, 1, 1, 1)),
    ("fprop_per_sample", "fprop_ps", (2, 32, 32, 64, 128, 3, 3, 1, 1, 1)),
    ("dgrad_per_sample", "dgrad_ps", (2, 32, 32, 64, 128, 3, 3, 1, 1, 1)),
]
CASE_BY_ID = {c[0]: c for c in CASES}


def tf32(t):
    """round-to-nearest (ties away) to TF32, as a float64 tensor"""
    bits = t.float().contiguous().view(torch.int32)
    return ((bits + 0x1000) & ~0x1FFF).view(torch.float32).double()


@pytest.fixture
def kern():
    k = backend.kernels()
    prev = (k.conv_impl, k.precision, k.round_tf32, k.act_masks, k.deterministic)
    k.conv_impl, k.precision, k.round_tf32, k.act_masks, k.deterministic = 0, "tf32", True, True, False
    yield k
    k.conv_impl, k.precision, k.round_tf32, k.act_masks, k.deterministic = prev


def _nhwc(t):
    return t.float().to(DEV).permute(0, 2, 3, 1).contiguous()


def _setup(kern, case, fp32_operands):
    """asserts the wgmma path; returns (geometry, float64 NCHW source, float64 KCRS filter, per-sample scales or None)"""
    cid, direction, args = case
    g = make_geom(*args)
    dgrad = direction.startswith("dgrad")
    if direction.endswith("_ps"):
        assert kern.conv_modulated_ok(g), cid
    else:
        assert kern.conv_impl_for(g, 1 if dgrad else 0) == 2, cid
    seed = sum(map(ord, cid))
    q = (lambda t: t.float().double()) if fp32_operands else tf32
    w = q(rnd(seed + 1, g.K, g.C, g.R, g.S) / math.sqrt(g.R * g.S * (g.K if dgrad else g.C)))
    src = q(rnd(seed + 2, g.N, g.K, g.P, g.Q) if dgrad else rnd(seed + 2, g.N, g.C, g.H, g.W))
    s = rnd(seed + 3, g.N, g.C) * 0.5 + 1.0 if direction.endswith("_ps") else None
    return g, src, w, s


def _run(kern, case, g, src, w, s, **epi):
    """(output NHWC on the device, per-sample filters [N, K, C, R, S] the kernel read, or None)"""
    direction = case[1]
    w_krsc = w.float().to(DEV).permute(0, 2, 3, 1).contiguous()
    if direction == "fprop":
        return kern.conv_fprop(_nhwc(src), w_krsc, g, **epi), None
    if direction == "dgrad":
        return kern.conv_dgrad(_nhwc(src), w_krsc, g, **epi), None
    if direction == "fprop_ps":
        wn, _ = kern.filter_modulate(w_krsc, s.float().to(DEV), want_krsc=True, want_crsk=False)
        return kern.conv_fprop_per_sample(_nhwc(src), wn, g, **epi), wn.double().cpu().permute(0, 1, 4, 2, 3)
    _, wn = kern.filter_modulate(w_krsc, s.float().to(DEV), want_krsc=False, want_crsk=True)
    return kern.conv_dgrad_per_sample(_nhwc(src), wn, g, **epi), wn.double().cpu().permute(0, 4, 1, 2, 3)


def _reference(case, g, src, w, wn):
    """fp64 F.conv2d (or its input gradient), NCHW"""
    dgrad = case[1].startswith("dgrad")
    outs = []
    for i in range(g.N if wn is not None else 1):
        wi = (wn[i] if wn is not None else w).to(DEV)
        si = (src[i:i + 1] if wn is not None else src).to(DEV)
        if dgrad:
            x = torch.zeros(si.shape[0], g.C, g.H, g.W, dtype=torch.float64, device=DEV, requires_grad=True)
            y = F.conv2d(x, wi, stride=g.stride, padding=(g.pad_t, g.pad_l))
            assert tuple(y.shape[2:]) == (g.P, g.Q)
            out, = torch.autograd.grad((y * si).sum(), x)
        else:
            out = F.conv2d(si, wi, stride=g.stride, padding=(g.pad_t, g.pad_l))
            assert tuple(out.shape[2:]) == (g.P, g.Q)
        outs.append(out.cpu())
    return torch.cat(outs)


def _nchw64(y):
    return y.permute(0, 3, 1, 2).double().cpu()


@pytest.mark.parametrize("case_id", [c[0] for c in CASES])
def test_tap_groups_tf32_vs_fp64(kern, case_id):
    case = CASE_BY_ID[case_id]
    g, src, w, s = _setup(kern, case, fp32_operands=False)
    y, wn = _run(kern, case, g, src, w, s, round_tf32=False)
    err = rel_err(_nchw64(y), _reference(case, g, src, w, wn))
    assert err < TOL, err


@pytest.mark.parametrize("case_id", [c[0] for c in CASES])
def test_tap_groups_fp32_mode_vs_fp64(kern, case_id):
    kern.precision = "fp32"
    case = CASE_BY_ID[case_id]
    g, src, w, s = _setup(kern, case, fp32_operands=True)
    y, wn = _run(kern, case, g, src, w, s)
    err = rel_err(_nchw64(y), _reference(case, g, src, w, wn))
    assert err < TOL, err


@pytest.mark.parametrize("case_id", ["fprop_bn128_tw16_pad1", "dgrad_bn64_tw8_ragged"])
def test_tap_groups_epilogue_and_mask(kern, case_id):
    """bias + NoiseInjection + leaky-ReLU on a reuse case: values and every activation-mask bit against fp64"""
    case = CASE_BY_ID[case_id]
    g, src, w, s = _setup(kern, case, fp32_operands=False)
    dgrad = case[1] == "dgrad"
    n, c, h, wd = (g.N, g.C, g.H, g.W) if dgrad else (g.N, g.K, g.P, g.Q)
    bias = rnd(7, c).float().double()
    noise = rnd(8, n, h, wd).float().double()
    nw = float(torch.tensor(0.37, dtype=torch.float32))
    epi = dict(round_tf32=False, bias=bias.float().to(DEV), noise=noise.float().to(DEV).reshape(-1).contiguous(),
               noise_weight=torch.tensor([nw], device=DEV), act=3, alpha=0.2, gain=math.sqrt(2))
    if dgrad:
        epi["act_mask"] = torch.full((n * c * h * wd // 32,), -0x5A5A5A5B, dtype=torch.int32, device=DEV)
    y, _ = _run(kern, case, g, src, w, s, **epi)
    mask = epi["act_mask"] if dgrad else backend.act_mask_of(y)
    z = _reference(case, g, src, w, None) + bias.view(1, -1, 1, 1) + nw * noise[:, None]
    alpha, gain = float(torch.tensor(0.2, dtype=torch.float32)), float(torch.tensor(math.sqrt(2), dtype=torch.float32))
    ref = torch.where(z > 0, z, z * alpha) * gain
    assert rel_err(_nchw64(y), ref) < TOL, rel_err(_nchw64(y), ref)
    words = mask.cpu().to(torch.int64) & 0xFFFFFFFF
    bits = ((words[:, None] >> torch.arange(32)) & 1).reshape(-1).bool()
    zf = z.permute(0, 2, 3, 1).reshape(-1)
    band = zf.abs() <= 1e-4 * zf.abs().max()
    assert band.float().mean() < 0.01
    assert not ((bits != (zf > 0)) & ~band).any()


@pytest.mark.parametrize("case_id", ["fprop_bn128_tw16_pad1", "dgrad_stride2_pad0"])
def test_tap_groups_deterministic_twins(kern, case_id):
    """the deterministic entry points run the same kernel: bitwise equal from call to call, and within 2e-5 of fp64"""
    kern.deterministic = True
    case = CASE_BY_ID[case_id]
    g, src, w, s = _setup(kern, case, fp32_operands=False)
    a, _ = _run(kern, case, g, src, w, s, round_tf32=False)
    b, _ = _run(kern, case, g, src, w, s, round_tf32=False)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert rel_err(_nchw64(a), _reference(case, g, src, w, None)) < TOL
