"""GPU (H100): the deterministic mode end to end (backend.CudaKernels.deterministic / SAE_DETERMINISTIC /
torch.use_deterministic_algorithms).

* the bandwidth twins (bias + activation, style modulation, FIR + activation, ToRGB backward) on each launch branch: bitwise
  equal plainly, after an independent launch on a second stream, and under CUDA-graph replay; fp64 within bound;
* the kernels a D, D + R1 and G half-step launch in the mode: none of them is an atomic kernel; with the mode off, none of
  them is a deterministic one;
* trajectories: two trainers from one seed, 8 half-steps with crops, noise and the patch discriminator, eager and with CUDA
  graphs, in both precisions: losses, parameters and Adam moments bitwise equal after every half-step;
* eager against graph replay, teacher-forced: bitwise equal losses and gradients;
* two processes: equal SHA-256 of the parameters after 6 half-steps;
* torch.use_deterministic_algorithms(True) alone turns the mode on, with torch's NaN filling of uninitialised memory."""
import ctypes
import hashlib
import os
import subprocess
import sys

import pytest
import torch

from oracle.fixtures import TINY, rel_err, rnd
from swapping_autoencoder_pytorch_b200 import _lib, backend, default_options
from tests.test_gpu_deterministic import _det_call, _p, _three_ways
from tests.test_gpu_graphs import _teacher_forced_run

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def kern():
    k = backend.kernels()
    prev = (k.precision, k.deterministic, k.round_tf32)
    yield k
    k.precision, k.deterministic, k.round_tf32 = prev


def _mask_of(o):
    """the activation bit mask of o (bit i & 31 of word i >> 5: element i > 0)"""
    b = (o.reshape(-1, 32) > 0).to(torch.int64) << torch.arange(32, device=o.device)
    w = b.sum(1)
    return ((w + 2 ** 31) % 2 ** 32 - 2 ** 31).to(torch.int32)


# ------------------------------------------------------------------------------------------------ bandwidth twins
@pytest.mark.parametrize("c,noise,mask,offset", [(64, False, False, 0), (64, True, False, 0), (64, False, True, 0),
                                                  (5, True, False, 0), (64, False, False, 1), (2048, False, False, 0)],
                         ids=["f4", "f4_noise", "f4_mask", "scalar_c5_noise", "scalar_misaligned", "f4_c2048"])
def test_bias_act_backward_det(c, noise, mask, offset):
    n, h, w = 3, 9, 11
    size = n * h * w * c
    go = torch.randn(size + offset, device=DEV)[offset:]
    out = torch.randn(size, device=DEV)
    gi = torch.empty(size + offset, device=DEV)[offset:]
    gb = torch.full((c,), 0.5, device=DEV)
    nz = torch.randn(n * h * w, device=DEV) if noise else None
    gnw = torch.full((1,), -1.0, device=DEV) if noise else None
    m = _mask_of(out) if mask else None
    alpha, scale = 0.2, 1.4142
    outs = [gb, gi] + ([gnw] if noise else [])
    res, init = _three_ways(lambda: _det_call("sae_bias_act_backward_det", (
        _p(go), None if mask else _p(out), _p(gi), _p(gb), size, c, alpha, scale, _p(nz), c, _p(gnw), 0, _p(m))), outs)
    y32 = torch.where(out > 0, go, go * alpha) * scale           # the kernel's fp32 arithmetic, element by element
    assert torch.equal(res[1], y32)
    y = y32.double()
    assert rel_err(res[0].double(), y.reshape(-1, c).sum(0) + 0.5) < 1e-5
    if noise:
        ref = (y.reshape(-1, c).sum(1) * nz.double()).sum() - 1.0
        assert abs(float(res[2]) - float(ref)) <= 1e-5 * float(y.abs().reshape(-1, c).sum(1).mul(nz.double().abs()).sum())


@pytest.mark.parametrize("shape", [(2, 6, 5, 64), (1, 64, 64, 32), (2, 4, 4, 2048), (2, 6, 5, 5), (2, 3, 4, 1027)],
                         ids=["f4_narrow", "f4_narrow_many_chunks", "f4_wide", "scalar_narrow", "scalar_wide"])
def test_modulate_backward_det(shape):
    n, h, w, c = shape
    dy, x = torch.randn(n, h, w, c, device=DEV), torch.randn(n, h, w, c, device=DEV)
    s = torch.randn(n, c, device=DEV)
    dx = torch.empty_like(x)
    ds = torch.full((n, c), 0.25, device=DEV)
    (ds_, dx_), _ = _three_ways(lambda: _det_call("sae_modulate_backward_det", (
        _p(dy), _p(x), _p(s), _p(dx), _p(ds), n, h * w, c, 0)), [ds, dx])
    assert torch.equal(dx_, (dy * s[:, None, None, :]))
    ref = (dy.double() * x.double()).sum((1, 2)) + 0.25
    assert rel_err(ds_.double(), ref) < 1e-5


@pytest.mark.parametrize("t,shape,pad,mask", [(3, (2, 21, 19, 32), (1, 1, 1, 1), False), (4, (2, 18, 21, 96), (1, 2, 2, 1), True)],
                         ids=["t3_actout", "t4_mask"])
def test_fir_act_backward_det(kern, t, shape, pad, mask):
    n, h, w, c = shape
    taps = [1.0, 2.0, 1.0] if t == 3 else [1.0, 3.0, 3.0, 1.0]
    ty = (ctypes.c_float * t)(*taps)
    px0, px1, py0, py1 = pad
    oh, ow = h + py0 + py1 - t + 1, w + px0 + px1 - t + 1
    g = torch.randn(n, h, w, c, device=DEV)
    act = torch.randn(n, oh, ow, c, device=DEV)
    gi = torch.empty_like(act)
    gb = torch.full((c,), 1.0, device=DEV)
    m = _mask_of(act) if mask else None
    (gi_, gb_), _ = _three_ways(lambda: _det_call("sae_fir_act_backward_det", (
        _p(g), ty, ty, None if mask else _p(act), _p(gi), _p(gb), n, h, w, c, t, t, px0, px1, py0, py1, 0.2, 1.4142, 0, _p(m))),
        [gi, gb])
    # grad_in equal to the fused (atomic) kernel's up to the order of the two scale factors (alpha * scale there, (v * alpha) *
    # scale here: a last-bit difference on the negative branch); the bias gradient within the fp64 bound
    gi2 = torch.empty_like(act)
    gb2 = torch.zeros(c, device=DEV)
    _lib.check(_lib.load().sae_fir_act_backward(_p(g), ty, ty, None if mask else _p(act), _p(gi2), _p(gb2), n, h, w, c, t, t,
                                                px0, px1, py0, py1, 0.2, 1.4142, 0, _p(m), None), "fir_act_backward")
    torch.cuda.synchronize()
    assert rel_err(gi_.double(), gi2.double()) < 1e-6
    assert rel_err(gb_.double(), gi2.double().sum((0, 1, 2)) + 1.0) < 1e-5


@pytest.mark.parametrize("c,layout", [(64, "nchw"), (256, "channels_last"), (512, "nchw"), (1024, "channels_last")])
def test_torgb_backward_det(c, layout):
    n, h, w = 2, 15, 17
    x = torch.randn(n, h, w, c, device=DEV)
    s, wt = torch.randn(n, c, device=DEV), torch.randn(3, c, device=DEV)
    dy = torch.randn(n, 3, h, w, device=DEV)
    if layout == "channels_last":
        dy = dy.contiguous(memory_format=torch.channels_last)
    dx = torch.empty_like(x)
    gw = torch.full((n, 3, c), -0.5, device=DEV)
    (gw_, dx_), _ = _three_ways(lambda: _det_call("sae_torgb_backward_det", (
        _p(dy), _p(x), _p(s), _p(wt), _p(dx), _p(gw), n, h, w, c, 0.1, dy.stride(0), dy.stride(1), dy.stride(2), dy.stride(3), 0)),
        [gw, dx])
    ref = torch.einsum("nohw,nhwc->noc", dy.double(), x.double()) - 0.5
    assert rel_err(gw_.double(), ref) < 1e-5
    dxr = torch.einsum("nohw,oc->nhwc", dy.double(), wt.double()) * s.double()[:, None, None, :] * 0.1
    assert rel_err(dx_.double(), dxr) < 1e-5


# ------------------------------------------------------------------------------------------------ training
def _trainer(**over):
    import swapping_autoencoder_pytorch_b200 as S
    opt = default_options(**dict(TINY, num_gpus=1, **over))
    torch.manual_seed(0)
    model = S.create_model(opt)
    return S.create_optimizer(opt, model)


def _real():
    return torch.randn(2, 3, 64, 64, device=DEV, generator=torch.Generator(DEV).manual_seed(5)).clamp(-1, 1)


def _snapshot(tr, out):
    ms = tr.model.singlegpu_model
    st = [o._state() for o in (tr.optimizer_G, tr.optimizer_D)]
    return ([float(v) for v in out.values()], [p.detach().clone() for p in ms.parameters()],
            [t.clone() for s in st for t in (s.exp_avg, s.exp_avg_sq, s.steps)])


def _trajectory(graphs, steps=8):
    tr = _trainer(cuda_graphs=graphs, R1_once_every=2)
    torch.manual_seed(123)
    real = _real()
    snaps = []
    for _ in range(steps):
        out = tr.train_one_step({"real_A": real}, 0)
        snaps.append(_snapshot(tr, out))
    if graphs:
        assert tr.graphs.disabled is None, (tr.graphs.disabled, tr.graphs.last_traceback)
    return snaps


def _bitwise(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize("precision", ["tf32", "fp32"])
@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
def test_trajectories_bitwise(kern, precision, graphs):
    kern.precision, kern.deterministic = precision, True
    a, b = _trajectory(graphs), _trajectory(graphs)
    for step, (sa, sb) in enumerate(zip(a, b)):
        assert sa[0] == sb[0], (step, sa[0], sb[0])
        for x, y in zip(sa[1] + sa[2], sb[1] + sb[2]):
            assert _bitwise(x, y), step


ATOMIC = ("bias_act_bwd_kernel", "modulate_bwd_kernel", "torgb_bwd_kernel")
DET_TEMPLATED = ("conv_gather_kernel", "conv_wgrad_kernel", "wgrad_wg_kernel", "wgrad_split_kernel")


def _launched(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "sae::" in e.name}


def _classify(name):
    """'atomic' for a kernel that reduces with float atomics, 'det' for a deterministic-mode kernel, None otherwise"""
    base = name.split("sae::", 1)[1].split("<")[0].split("(")[0]
    targs = name.split("(")[0]
    if base in ATOMIC or (base == "fir_tma_kernel" and targs.replace(" ", "").endswith(",1>")):
        return "atomic"
    if base.endswith("_det_kernel") or base == "det_reduce_kernel":
        return "det"
    if base in DET_TEMPLATED:
        return "det" if targs.replace(" ", "").endswith("true>") else "atomic"
    return None


@pytest.mark.parametrize("precision", ["tf32", "fp32"])
def test_launch_set(kern, precision):
    kern.precision = precision
    tr = _trainer(cuda_graphs=False, R1_once_every=1)
    real = _real()
    for det, forbidden in ((True, "atomic"), (False, "det")):
        kern.deterministic = det
        names = _launched(lambda: [tr.train_one_step({"real_A": real}, 0) for _ in range(2)])   # D + R1, then G
        assert names
        bad = sorted(n for n in names if _classify(n) == forbidden)
        assert not bad, (det, bad)
        if det:
            assert any(_classify(n) == "det" for n in names)


def test_eager_against_graph_bitwise(kern, monkeypatch):
    from swapping_autoencoder_pytorch_b200.stylegan2_layers import NoiseInjection

    def zero_noise(self, image, noise=None):
        if self.image_size is None:
            self.image_size = image.shape
        b, _, h, w = image.shape
        return image.new_empty(b, 1, h, w).zero_()
    monkeypatch.setattr(NoiseInjection, "resolve_noise", zero_noise)
    kern.deterministic = True
    tg, rows = _teacher_forced_run(_real(), dict(lambda_PatchGAN=0.0, lambda_patch_R1=0.0, R1_once_every=2))
    assert tg.graphs.disabled is None, (tg.graphs.disabled, tg.graphs.last_traceback)
    assert {r[2] for r in rows} >= {"replay"}
    assert all(r[3] == 0.0 and r[4] == 0.0 for r in rows), rows


SCRIPT = r"""
import hashlib, torch
from oracle.fixtures import TINY
import swapping_autoencoder_pytorch_b200 as S
opt = S.default_options(**dict(TINY, num_gpus=1, R1_once_every=2))
torch.manual_seed(0)
tr = S.create_optimizer(opt, S.create_model(opt))
torch.manual_seed(123)
real = torch.randn(2, 3, 64, 64, device="cuda", generator=torch.Generator("cuda").manual_seed(5)).clamp(-1, 1)
for _ in range(6):
    tr.train_one_step({"real_A": real}, 0)
h = hashlib.sha256()
for p in tr.model.singlegpu_model.parameters():
    h.update(p.detach().cpu().numpy().tobytes())
print(h.hexdigest())
"""


def test_two_processes_same_digest():
    env = dict(os.environ, SAE_DETERMINISTIC="1", PYTHONPATH=ROOT)
    digests = [subprocess.run([sys.executable, "-s", "-c", SCRIPT], cwd=ROOT, env=env, capture_output=True, text=True,
                              timeout=600) for _ in range(2)]
    for d in digests:
        assert d.returncode == 0, d.stderr[-2000:]
    a, b = (d.stdout.strip().splitlines()[-1] for d in digests)
    assert len(a) == 64 and a == b


def test_torch_flag_turns_the_mode_on(kern):
    kern.deterministic = False
    prev_fill = torch.utils.deterministic.fill_uninitialized_memory
    torch.use_deterministic_algorithms(True)
    torch.utils.deterministic.fill_uninitialized_memory = True
    try:
        assert kern.deterministic_mode()
        a, b = _trajectory(False, steps=3), _trajectory(False, steps=3)
    finally:
        torch.use_deterministic_algorithms(False)
        torch.utils.deterministic.fill_uninitialized_memory = prev_fill
    assert not kern.deterministic_mode()
    for sa, sb in zip(a, b):
        assert sa[0] == sb[0] and all(v == v for v in sa[0])
        for x, y in zip(sa[1] + sa[2], sb[1] + sb[2]):
            assert _bitwise(x, y)
