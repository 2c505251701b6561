"""GPU (H100): the deterministic conv entry points (the _det twins of include/sae_b200.h).

Every case runs its twin three times into destinations that already hold a non-zero value: plainly, right after a large
independent launch on a second stream, and captured into a CUDA graph and replayed.  The three results must be bitwise
identical, must equal initial value + result, and must agree with fp64 within the bound the existing test of that path
uses (operands pre-rounded to TF32, so only the summation order differs from fp64)."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from oracle.fixtures import rel_err, rnd
from swapping_autoencoder_pytorch_b200 import _lib
from swapping_autoencoder_pytorch_b200.backend import make_geom

pytestmark = pytest.mark.gpu
DEV = "cuda"


def tf32(t):
    bits = t.float().contiguous().view(torch.int32)
    return ((bits + 0x1000) & ~0x1FFF).view(torch.float32).double()


def nhwc(t):
    return t.float().to(DEV).permute(0, 2, 3, 1).contiguous()


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _det_call(name, args):
    """size query, then the call with a workspace; returns the workspace size"""
    lib = _lib.load()
    fn = getattr(lib, name)
    size = ctypes.c_int64(0)
    _lib.check(fn(*args, None, ctypes.byref(size), None), name)
    ws = torch.empty(max(size.value, 1), dtype=torch.uint8, device=DEV)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(fn(*args, _p(ws), ctypes.byref(size), stream), name)
    return size.value


def _three_ways(run, outs):
    """run() writes into the tensors `outs` (accumulating); returns the three results of the plain, the perturbed and the
    graph-replayed call, each from the same initial values"""
    init = [o.clone() for o in outs]
    results = []

    def reset():
        for o, i in zip(outs, init):
            o.copy_(i)

    reset()
    run()
    torch.cuda.synchronize()
    results.append([o.clone() for o in outs])
    # a large independent launch on a second stream, overlapping the call
    reset()
    side = torch.cuda.Stream()
    big = torch.randn(64 * 1024 * 1024, device=DEV)
    with torch.cuda.stream(side):
        for _ in range(4):
            big.mul_(1.0001).add_(1e-3)
    run()
    torch.cuda.synchronize()
    results.append([o.clone() for o in outs])
    # CUDA graph: capture on a side stream (the allocator serves the workspace from the graph's pool), replay
    reset()
    cap = torch.cuda.Stream()
    cap.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(cap):
        with torch.cuda.graph(g, stream=cap):
            run()
    torch.cuda.synchronize()
    reset()
    g.replay()
    torch.cuda.synchronize()
    results.append([o.clone() for o in outs])
    for r in results[1:]:
        for a, b in zip(results[0], r):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    return results[0], init


def _wgrad_ref(x, dy, k, r, stride, pad):
    w = torch.zeros(k, x.shape[1], r, r, dtype=torch.float64, device=DEV, requires_grad=True)
    y = F.conv2d(x.to(DEV), w, stride=stride, padding=pad)
    gw, = torch.autograd.grad((y * dy.to(DEV)).sum(), w)
    return gw.cpu()


WGRAD_CASES = [
    # (n, h, w, c, k, r, stride, pad, impl, name)
    (2, 37, 45, 64, 128, 3, 1, 1, 0, "sae_conv2d_wgrad_det"),          # wgmma TMA pipeline, ragged boxes
    (2, 64, 64, 32, 128, 3, 1, 1, 0, "sae_conv2d_wgrad_det"),          # C = 32: a tile spans four taps
    (4, 64, 64, 128, 32, 3, 1, 1, 0, "sae_conv2d_wgrad_det"),          # Ko = 32: an idle warpgroup
    (2, 129, 129, 128, 256, 3, 2, 0, 0, "sae_conv2d_wgrad_det"),       # stride 2
    (2, 37, 45, 64, 128, 3, 1, 1, 1, "sae_conv2d_wgrad_det"),          # impl = 1: mma.sync
    (2, 20, 20, 48, 64, 3, 1, 1, 0, "sae_conv2d_wgrad_det"),           # C % 32 != 0: mma.sync
    (2, 20, 20, 3, 32, 3, 1, 1, 0, "sae_conv2d_wgrad_det"),            # C = 3: scalar loader
    (2, 37, 45, 64, 128, 3, 1, 1, 0, "sae_conv2d_wgrad_3xtf32_det"),   # split-TF32 wgmma
    (2, 37, 45, 64, 128, 3, 1, 1, 1, "sae_conv2d_wgrad_3xtf32_det"),   # split-TF32 mma.sync
]


@pytest.mark.parametrize("case", WGRAD_CASES, ids=lambda c: "%s_c%d_k%d_s%d_impl%d" % (c[9][11:-4], c[3], c[4], c[6], c[8]))
def test_wgrad_det(case):
    n, h, w_, c, k, r, stride, pad, impl, name = case
    g = make_geom(n, h, w_, c, k, r, r, stride, pad, pad)
    x = tf32(rnd(31, n, c, h, w_))
    dy = tf32(rnd(32, n, k, g.P, g.Q))
    xd, dyd = nhwc(x), nhwc(dy)
    dw = torch.full((k, r, r, c), 0.25, device=DEV)
    (out,), (init,) = _three_ways(lambda: _det_call(name, (_p(dyd), _p(xd), _p(dw), ctypes.byref(g), impl)), [dw])
    ref = _wgrad_ref(x, dy, k, r, stride, pad) + 0.25
    assert rel_err((out).permute(0, 3, 1, 2), ref) < 2e-5, rel_err(out.permute(0, 3, 1, 2), ref)


@pytest.mark.parametrize("name", ["sae_conv2d_wgrad_modulated_det", "sae_conv2d_wgrad_modulated_3xtf32_det"])
@pytest.mark.parametrize("ko,pad", [(32, 1), (64, 1), (256, 1), (64, 101)])
def test_wgrad_modulated_det(name, ko, pad):
    """C = 64 with 3x3 taps (the smallest C the modulated kernels take): a 128-column tile carries two taps of the same
    channels, so the ds slot map must keep them apart; Ko = 256 gives two M tiles, Ko = 32 / 64 an idle warpgroup.
    pad = 101 (24 x 24 input, 224 x 224 output) is past the wgmma kernel's padding limit: the mma.sync kernel's modulated
    drain, whose ds slots are per warp row (64 output channels)"""
    n, h, c, r = (4, 32, 64, 3) if pad == 1 else (1, 24, 64, 3)
    g = make_geom(n, h, h, c, ko, r, r, 1, pad, pad)
    assert _lib.load().sae_conv2d_query_impl(ctypes.byref(g), 2) == (2 if pad == 1 else 1)
    x, dy = tf32(rnd(51, n, c, h, h)), tf32(rnd(52, n, ko, g.P, g.Q))
    w, s = tf32(rnd(53, ko, c, r, r) / math.sqrt(c * r * r)), tf32(rnd(54, n, c) + 1.5)
    xr, wr, sr = x.to(DEV), w.to(DEV).requires_grad_(), s.to(DEV).requires_grad_()
    yr = F.conv2d(xr * sr[:, :, None, None], wr, padding=pad)
    gwr, gsr = torch.autograd.grad((yr * dy.to(DEV)).sum(), [wr, sr])
    dyd, xd, sd, wd = nhwc(dy), nhwc(x), s.float().to(DEV).contiguous(), nhwc(w)
    dw = torch.full((ko, r, r, c), -0.5, device=DEV)
    ds = torch.full((n, c), 2.0, device=DEV)
    (gw, gs), _ = _three_ways(
        lambda: _det_call(name, (_p(dyd), _p(xd), _p(sd), _p(wd), _p(dw), _p(ds), ctypes.byref(g))), [dw, ds])
    assert rel_err(gw.permute(0, 3, 1, 2), gwr.cpu() - 0.5) < 2e-5
    assert rel_err(gs, gsr.cpu() + 2.0) < 2e-5


@pytest.mark.parametrize("name,split", [("sae_conv2d_fprop_det", False), ("sae_conv2d_fprop_3xtf32_det", True),
                                        ("sae_conv2d_dgrad_det", False), ("sae_conv2d_dgrad_3xtf32_det", True)])
@pytest.mark.parametrize("round_tf32", [0, 1])
def test_split_k_linear_det(name, split, round_tf32):
    """the generic kernel's split K (a deep linear: M = 4 rows, K = 512): partials summed in split order, then rounded"""
    m, cin, cout = 4, 512, 256
    x = tf32(rnd(71, m, cin))
    w = tf32(rnd(72, cout, cin) / math.sqrt(cin))
    dgrad = "dgrad" in name
    if dgrad:
        g = make_geom(m, 1, 1, cout, cin, 1, 1, 1, 0, 0)       # dx [m, cout] from dy [m, cin] and wt [cout, cin]
    else:
        g = make_geom(m, 1, 1, cin, cout, 1, 1, 1, 0, 0)
    xd = x.float().to(DEV).contiguous()
    wd = w.float().to(DEV).contiguous()
    y = torch.full((m, cout), 7.0, device=DEV)               # overwritten, as by the atomic twin
    e = _lib.ConvEpilogue()
    e.alpha, e.gain, e.res_scale, e.act, e.round_tf32 = 0.2, 1.0, 1.0, 1, round_tf32
    wlo = torch.zeros_like(wd)                               # the operands are TF32 already: their low halves are zero
    size = []

    def run():
        args = (_p(xd), _p(wd)) + ((_p(wlo),) if split else ()) + (_p(y), ctypes.byref(g), ctypes.byref(e), 1)
        size.append(_det_call(name, args))

    (out,), _ = _three_ways(run, [y])
    assert size[0] > 0, "expected a split-K launch"
    ref = x.to(DEV) @ w.to(DEV).t()
    assert rel_err(out.double().cpu(), ref.cpu()) < (1e-3 if round_tf32 else 2e-5)
    if round_tf32:
        assert torch.equal(out, tf32(out).float().to(DEV))
