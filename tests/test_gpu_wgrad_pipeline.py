"""GPU (H100): the TMA-fed, warp-specialised weight-gradient kernel (csrc/wgrad_wgmma.cu) — pixel boxes with ragged and
zero-filled edges, column tiles spanning several taps, output-channel tiles partly or wholly past Ko, pixel splits of every
size, the style-modulated drain, and the shapes that must stay on the mma.sync kernel."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle.fixtures import rel_err, rnd
from swapping_autoencoder_pytorch_b200 import backend
from swapping_autoencoder_pytorch_b200.backend import make_geom

pytestmark = pytest.mark.gpu
DEV = "cuda"


def tf32(t):
    """round-to-nearest (ties away) to TF32, as a float64 tensor — what cvt.rna.tf32.f32 does to an fp32 value"""
    bits = t.float().contiguous().view(torch.int32)
    return ((bits + 0x1000) & ~0x1FFF).view(torch.float32).double()


def nhwc(t):
    return t.float().to(DEV).permute(0, 2, 3, 1).contiguous()


@pytest.fixture
def kern():
    k = backend.kernels()
    prev = (k.conv_impl, k.precision)
    k.conv_impl, k.precision = 0, "tf32"
    yield k
    k.conv_impl, k.precision = prev


def _wgrad_ref(x, dy, k, r, stride, pad):
    """fp64 weight gradient on the GPU: d/dw of sum(conv2d(x, w) * dy)"""
    w = torch.zeros(k, x.shape[1], r, r, dtype=torch.float64, device=DEV, requires_grad=True)
    y = F.conv2d(x.to(DEV), w, stride=stride, padding=pad)
    gw, = torch.autograd.grad((y * dy.to(DEV)).sum(), w)
    return gw.cpu()


WGRAD_CASES = [
    # (n, h, w, c, k, r, stride, pad)
    (2, 37, 45, 64, 128, 3, 1, 1),          # ragged boxes: H, W not multiples of the box
    (2, 37, 45, 64, 128, 3, 1, 0),          # ... pad 0
    (2, 129, 129, 128, 256, 3, 2, 0),       # stride 2 on odd sizes
    (2, 257, 257, 32, 64, 3, 2, 0),
    (2, 255, 255, 128, 256, 1, 2, 0),       # 1x1 stride 2
    (2, 64, 64, 32, 128, 3, 1, 1),          # C = 32: a 128-column tile spans four taps
    (2, 64, 64, 64, 128, 3, 1, 1),          # C = 64: two taps per tile
    (4, 64, 64, 128, 32, 3, 1, 1),          # Ko = 32: the second warpgroup has no rows
    (4, 64, 64, 128, 64, 3, 1, 1),          # Ko = 64
    (2, 32, 32, 512, 512, 3, 1, 1),         # several M and N tiles
    (8, 4, 4, 256, 256, 3, 1, 1),           # 4x4 maps: two images per 32-pixel box
    (6, 4, 4, 64, 32, 3, 1, 0),             # 2x2 outputs, eight images per box
    (16, 128, 160, 32, 32, 3, 1, 1),        # ~39 boxes per CTA: the 4-stage ring wraps ~10 times
    (1, 8, 8, 128, 128, 3, 1, 1),           # two boxes in all: fewer chunks than SMs
]


@pytest.mark.parametrize("case", WGRAD_CASES)
def test_wgrad_pipeline_vs_fp64(kern, case):
    n, h, w_, c, k, r, stride, pad = case
    g = make_geom(n, h, w_, c, k, r, r, stride, pad, pad)
    assert kern.conv_impl_for(g, 2) == 2
    # operands pre-rounded to TF32: products are exact in fp32, only the summation order differs from fp64
    x = tf32(rnd(31, n, c, h, w_))
    dy = tf32(rnd(32, n, k, g.P, g.Q))
    gw = kern.conv_wgrad(nhwc(dy), nhwc(x), g).permute(0, 3, 1, 2)
    ref = _wgrad_ref(x, dy, k, r, stride, pad)
    assert rel_err(gw, ref) < 2e-5, rel_err(gw, ref)


def test_wgrad_pipeline_matches_mma_sync_on_fp32_operands(kern):
    """arbitrary fp32 operands: both kernels round them to TF32 (cvt.rna) on the way in, so they agree to summation order"""
    n, h, c, k = 4, 48, 128, 256
    g = make_geom(n, h, h, c, k, 3, 3, 1, 1, 1)
    x, dy = nhwc(rnd(41, n, c, h, h)), nhwc(rnd(42, n, k, h, h))
    new = kern.conv_wgrad(dy, x, g)
    old = kern.conv_wgrad(dy, x, g, impl=1)
    assert rel_err(new, old) < 1e-5, rel_err(new, old)


def test_wgrad_modulated_pipeline_vs_fp64(kern):
    """dW and ds of the style-modulated convolution; 8 images, so every column tile drains several images"""
    n, h, c, k, r = 8, 32, 64, 128, 3
    g = make_geom(n, h, h, c, k, r, r, 1, 1, 1)
    assert kern.conv_modulated_ok(g)
    x, dy = tf32(rnd(51, n, c, h, h)), tf32(rnd(52, n, k, h, h))
    w, s = tf32(rnd(53, k, c, r, r) / math.sqrt(c * r * r)), tf32(rnd(54, n, c) + 1.5)
    xr, wr, sr = x.to(DEV), w.to(DEV).requires_grad_(), s.to(DEV).requires_grad_()
    yr = F.conv2d(xr * sr[:, :, None, None], wr, padding=1)
    gwr, gsr = torch.autograd.grad((yr * dy.to(DEV)).sum(), [wr, sr])
    gw, gs = kern.conv_wgrad_modulated(nhwc(dy), nhwc(x), s.float().to(DEV), nhwc(w), g)
    assert rel_err(gw.permute(0, 3, 1, 2), gwr.cpu()) < 2e-5
    assert rel_err(gs, gsr.cpu()) < 2e-5


@pytest.mark.parametrize("c,k", [(48, 64), (64, 96 + 4), (3, 32), (32, 3)])
def test_wgrad_outside_pipeline_takes_mma_sync(kern, c, k):
    """channel counts that are not multiples of 32 dispatch to the mma.sync kernel, and it computes them"""
    n, h = 2, 20
    g = make_geom(n, h, h, c, k, 3, 3, 1, 1, 1)
    assert kern.conv_impl_for(g, 2) == 1
    x, dy = tf32(rnd(61, n, c, h, h)), tf32(rnd(62, n, k, h, h))
    gw = kern.conv_wgrad(nhwc(dy), nhwc(x), g).permute(0, 3, 1, 2)
    ref = _wgrad_ref(x, dy, k, 3, 1, 1)
    assert rel_err(gw, ref) < 2e-5, rel_err(gw, ref)
