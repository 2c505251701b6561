"""GPU (H100): the fp32 precision mode (``CudaKernels.precision = "fp32"`` / ``SAE_PRECISION=fp32``): split-TF32 (3xTF32)
convolutions and linears, nothing rounded to TF32 on storage.

Operands here are arbitrary fp32 values (not pre-rounded to TF32).  A split operand carries about 22 significant bits, so a
product is off by about 2^-22 instead of TF32's 2^-11; the bounds below are fp32-level: 2e-5 max-norm relative per op,
2e-4 for network outputs (and within 4x of cuDNN in strict fp32 on the same inputs), 1e-3 relative L2 for R1 and its weight
gradients (TF32 mode: 2e-2, DESIGN.md §2).  When SAE_PARITY_RECORD names a JSON file, the measured errors are added to it
(as tests/test_gpu_parity_full.py does)."""
import json
import math
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import sae_oracle as O
from oracle.fixtures import TINY, rel_err, rel_l2, rnd
from swapping_autoencoder_pytorch_b200 import backend, default_options
from swapping_autoencoder_pytorch_b200.backend import make_geom
from tests.test_gpu_parity import CONV_CASES

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL_OP = 2e-5
TOL_NET = 2e-4
TOL_R1 = 1e-3
RECORD = {}


@pytest.fixture(scope="module", autouse=True)
def _write_record():
    yield
    path = os.environ.get("SAE_PARITY_RECORD")
    if RECORD and path:
        old = json.load(open(path)) if os.path.exists(path) else {}
        old.update(RECORD)
        json.dump(old, open(path, "w"), indent=1, sort_keys=True)


def cuda(t):
    return t.float().to(DEV)


def f32(t):
    """the fp32 value of a (float64) tensor, as float64: the exact operand both sides see"""
    return t.float().double()


def nhwc(t):
    return cuda(t).permute(0, 2, 3, 1).contiguous()


@pytest.fixture
def fp32_mode():
    kern = backend.kernels()
    prev = kern.precision
    kern.precision = "fp32"
    yield kern
    kern.precision = prev


def _conv_case(kern, case, impl, seed=11):
    n, h, w_, c, k, r, stride, pad = case
    x = f32(rnd(seed, n, c, h, w_))
    wt = f32(rnd(seed + 1, k, c, r, r) / math.sqrt(c * r * r))
    xr, wr = x.clone().requires_grad_(), wt.clone().requires_grad_()
    yr = F.conv2d(xr, wr, stride=stride, padding=pad)
    dy = f32(rnd(seed + 2, *yr.shape))
    gxr, gwr = torch.autograd.grad((yr * dy).sum(), [xr, wr])
    g = make_geom(n, h, w_, c, k, r, r, stride, pad, pad)
    prev, kern.conv_impl = kern.conv_impl, impl
    try:
        xg, wg, dyg = nhwc(x), nhwc(wt), nhwc(dy)
        y = kern.conv_fprop(xg, wg, g).permute(0, 3, 1, 2)
        gx = kern.conv_dgrad(dyg, wg, g).permute(0, 3, 1, 2)
        gw = kern.conv_wgrad(dyg, xg, g).permute(0, 3, 1, 2)
    finally:
        kern.conv_impl = prev
    return rel_err(y, yr), rel_err(gx, gxr), rel_err(gw, gwr)


# ------------------------------------------------------------------------------------------------ 1. every conv direction
@pytest.mark.parametrize("impl", [1, 0])
@pytest.mark.parametrize("case", CONV_CASES)
def test_conv_fprop_dgrad_wgrad_fp32(case, impl, fp32_mode):
    e = _conv_case(fp32_mode, case, impl)
    RECORD.setdefault("fp32_mode.conv", {})["%s impl %d" % (case, impl)] = e
    assert max(e) < TOL_OP, (case, impl, e)


def test_tf32_mode_misses_the_fp32_bound():
    """the bound above separates the modes: on the deep-K cases the same arbitrary operands in TF32 mode are well above it"""
    kern = backend.kernels()
    assert kern.precision == "tf32"
    worst = max(max(_conv_case(kern, case, 0)) for case in CONV_CASES if case[3] * case[5] ** 2 >= 2304)
    RECORD["tf32_mode.conv_deep_k_worst"] = worst
    assert worst > 5 * TOL_OP, worst


# ------------------------------------------------------------------------------------------------ 2. per-sample, modulated, transposed, linear
def test_per_sample_and_modulated_fp32(fp32_mode):
    kern = fp32_mode
    n, h, c, k, r = 2, 32, 64, 128, 3
    g = make_geom(n, h, h, c, k, r, r, 1, 1, 1)
    assert kern.conv_modulated_ok(g)
    x, dy = f32(rnd(21, n, c, h, h)), f32(rnd(22, n, k, h, h))
    w, s = f32(rnd(23, k, c, r, r) / math.sqrt(c * r * r)), f32(rnd(24, n, c) + 1.5)
    # fp64 truth: image i convolved with w * s[i]  (== conv of x * s with the shared w)
    xr, wr, sr = x.clone().requires_grad_(), w.clone().requires_grad_(), s.clone().requires_grad_()
    xs = xr * sr[:, :, None, None]
    yr = F.conv2d(xs, wr, padding=1)
    gxs, gwr, gsr = torch.autograd.grad((yr * dy).sum(), [xs, wr, sr], retain_graph=True)
    gxr = gxs * s[:, :, None, None]                 # data gradient w.r.t. x of the per-sample filters
    w_krsc = nhwc(w)
    wn, wnt = kern.filter_modulate(w_krsc, cuda(s), want_krsc=True, want_crsk=True)
    y = kern.conv_fprop_per_sample(nhwc(x), wn, g).permute(0, 3, 1, 2)
    gx = kern.conv_dgrad_per_sample(nhwc(dy), wnt, g).permute(0, 3, 1, 2)
    gw, gs = kern.conv_wgrad_modulated(nhwc(dy), nhwc(x), cuda(s), w_krsc, g)
    errs = {"fprop": rel_err(y, yr), "dgrad": rel_err(gx, gxr), "dW": rel_err(gw.permute(0, 3, 1, 2), gwr),
            "ds": rel_err(gs, gsr)}
    RECORD["fp32_mode.per_sample"] = errs
    assert max(errs.values()) < TOL_OP, errs


def test_conv_transpose_and_linear_fp32(fp32_mode):
    from swapping_autoencoder_pytorch_b200.stylegan2_op import conv_transpose2d, linear
    errs = {}
    for i, (xs, ws) in enumerate((((2, 64, 9, 9), (64, 32, 3, 3)), ((2, 128, 17, 15), (128, 96, 3, 3)))):
        x, w = f32(rnd(1 + i, *xs)), f32(rnd(5 + i, *ws) / 24)
        errs["convT%d" % i] = rel_err(conv_transpose2d(cuda(x), cuda(w)), F.conv_transpose2d(x, w, stride=2))
    for i, (m, kin, kout) in enumerate(((16, 2048, 512), (6, 512, 1), (2, 8192, 512))):
        xl, wl = f32(rnd(10 + i, m, kin)), f32(rnd(20 + i, kout, kin) / math.sqrt(kin))
        xg, wg = cuda(xl).requires_grad_(), cuda(wl).requires_grad_()
        yl = linear(xg, wg)
        dy = f32(rnd(30 + i, m, kout))
        gx, gw = torch.autograd.grad((yl * cuda(dy)).sum(), [xg, wg])
        errs["linear%d" % i] = rel_err(yl, F.linear(xl, wl))
        errs["linear%d.dx" % i] = rel_err(gx, dy @ wl)
        errs["linear%d.dw" % i] = rel_err(gw, dy.t() @ xl)
    RECORD["fp32_mode.transpose_linear"] = errs
    assert max(errs.values()) < TOL_OP, errs


# ------------------------------------------------------------------------------------------------ 3 + 4. 256^2 networks and R1
@pytest.fixture(scope="module")
def nets_256():
    from tests import test_gpu_parity_full as PF
    kern = backend.kernels()
    prev = kern.precision
    kern.precision = "fp32"
    cfg = "256_default_bs2_fp32"
    try:
        opt, copt, model, oracle, real = PF._forward_parity(cfg, dict(crop_size=256, batch_size=2), 2, 8, with_context=True,
                                                            tol=TOL_NET)
    finally:
        kern.precision = prev
    return PF, PF.PARITY[cfg], opt, copt, model, oracle, real


def test_default_nets_256_fp32_against_oracle(nets_256):
    _, parity, *_ = nets_256
    rows = {}
    for name, who in parity.items():
        ours, ref = who["sae_b200"], who["torch_cudnn_fp32"]
        key = "rel_max_natural_scale" if "rel_max_natural_scale" in ours else "rel_max"
        rows[name] = (ours[key], ref[key])
    RECORD["fp32_mode.nets_256 (ours, torch_cudnn_fp32)"] = rows
    assert set(rows) >= {"E.sp", "E.gl", "G.rec", "D.pred", "Dpatch.feat_agg", "Dpatch.feat", "Dpatch.pred"}, sorted(rows)
    assert all(a < TOL_NET for a, _ in rows.values()), rows
    assert all(a <= 4 * b for a, b in rows.values()), rows


def test_r1_256_fp32_against_oracle(nets_256, fp32_mode):
    from swapping_autoencoder_pytorch_b200 import util
    PF, _, opt, copt, model, oracle, real = nets_256
    draws = PF._CropDraws()
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(O, "draw_crop_parameters", lambda b, o: draws.draw(b, o.patch_min_scale, o.patch_max_scale))
        mp.setattr(util, "draw_crop_parameters",
                   lambda b, sr, device: tuple(t.float().to(device) for t in draws.draw(b, sr[0], sr[1])))
        wD = oracle.D["stylegan2_D.convs.3.conv1.Conv.weight"].requires_grad_()
        wP = oracle.Dp["convs.2.conv2.Conv.weight"].requires_grad_()
        draws.reseed(3)
        ref_r1 = oracle.r1_loss(real)["D_R1"]
        ref_gD, ref_gP = torch.autograd.grad(ref_r1.mean(), [wD, wP])
        draws.reseed(3)
        r1 = model(cuda(real), command="compute_R1_loss")["D_R1"]
        gD, gP = torch.autograd.grad(r1.mean(), [getattr(model.D.stylegan2_D.convs, "3").conv1.Conv.weight,
                                                 getattr(model.Dpatch.convs, "2").conv2.Conv.weight])
    errs = {"D_R1": rel_l2(r1, ref_r1), "gD": rel_l2(gD, ref_gD), "gP": rel_l2(gP, ref_gP)}
    RECORD["fp32_mode.r1_256_rel_l2"] = errs
    assert max(errs.values()) < TOL_R1, errs


# ------------------------------------------------------------------------------------------------ 5. mode switching and graphs
def _trainer(**over):
    import swapping_autoencoder_pytorch_b200 as S
    opt = default_options(**dict(TINY, num_gpus=1, **over))
    torch.manual_seed(0)
    model = S.create_model(opt)
    return S.create_optimizer(opt, model)


def test_mode_switch_recaptures_graphs(monkeypatch):
    """D, G and R1 half-steps replayed from CUDA graphs in fp32 mode match eager fp32-mode runs from the same state; back in
    TF32 mode new graphs are captured and reproduce the losses of the TF32 run taken before the excursion, and a network forward
    is bit-identical to the one taken before it."""
    from swapping_autoencoder_pytorch_b200.stylegan2_layers import NoiseInjection
    from tests.test_gpu_graphs import _sync_state

    def zero_noise(self, image, noise=None):
        if self.image_size is None:
            self.image_size = image.shape
        b, _, h, w = image.shape
        return image.new_empty(b, 1, h, w).zero_()
    monkeypatch.setattr(NoiseInjection, "resolve_noise", zero_noise)
    det = dict(lambda_PatchGAN=0.0, lambda_patch_R1=0.0)
    kern = backend.kernels()
    assert kern.precision == "tf32"
    real = torch.randn(2, 3, 64, 64, device=DEV, generator=torch.Generator(DEV).manual_seed(5)).clamp(-1, 1)
    ts, te, tg = _trainer(cuda_graphs=False, **det), _trainer(cuda_graphs=False, **det), _trainer(cuda_graphs=True, **det)
    kinds = ("D", "G", "R1")

    def losses(tr, kind):
        _sync_state(ts, tr)                   # every half-step starts from the same parameters and Adam state
        out = tr._run(kind, real.clone())
        return {k: float(v.detach().mean()) for k, v in out.items() if not k.startswith("_")}

    def rel(a, b):
        assert a.keys() == b.keys()
        return max(abs(a[k] - b[k]) / max(abs(b[k]), 1e-2) for k in a)

    with torch.no_grad():
        _sync_state(ts, te)
        sp_before = te.model.singlegpu_model.E(real)[0].clone()
    tf32_ref = {kind: losses(te, kind) for kind in kinds}
    kern.precision = "fp32"
    try:
        fp32_rows = []
        for _ in range(4):                    # 2 eager warm-up calls per body, then capture, then replay
            for kind in kinds:
                fp32_rows.append((kind, rel(losses(tg, kind), losses(te, kind))))
        assert tg.graphs.disabled is None, (tg.graphs.disabled, tg.graphs.last_traceback)
        assert {(k[0], k[2]) for k in tg.graphs.captured} == {(kind, "fp32") for kind in kinds}, sorted(tg.graphs.captured)
        fp32_loss = {kind: losses(te, kind) for kind in kinds}
    finally:
        kern.precision = "tf32"
    RECORD["mode_switch"] = {"fp32 graph vs eager": max(r for _, r in fp32_rows)}
    assert max(r for _, r in fp32_rows) < 1e-5, fp32_rows
    assert max(rel(fp32_loss[kind], tf32_ref[kind]) for kind in kinds) > 1e-6      # the modes really differ
    tf32_rows = []
    for _ in range(4):
        for kind in kinds:
            tf32_rows.append((kind, rel(losses(tg, kind), tf32_ref[kind])))
    assert tg.graphs.disabled is None, (tg.graphs.disabled, tg.graphs.last_traceback)
    assert {(k[0], k[2]) for k in tg.graphs.captured} == {(kind, p) for kind in kinds for p in ("fp32", "tf32")}
    RECORD["mode_switch"]["tf32 graph after fp32 vs tf32 before"] = max(r for _, r in tf32_rows)
    assert max(r for _, r in tf32_rows) < 1e-6, tf32_rows
    with torch.no_grad():
        _sync_state(ts, te)
        sp_after = te.model.singlegpu_model.E(real)[0]
    assert torch.equal(sp_before, sp_after)
