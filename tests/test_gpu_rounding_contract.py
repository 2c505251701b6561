"""GPU (H100): the TF32 storage contract of every pointwise / FIR / layout entry point that takes ``round_tf32``.

With the policy on, each full-tensor output must be rna_tf32 (cvt.rna: round to nearest, ties away) of the output the same
kernel stores with the policy off, bit for bit: the rounding is the last operation before the store, on every branch of the
entry point (vector and scalar loaders, the separable FIR's TMA-tiled and plain kernels, each (up, down) pair).  The inputs
are arbitrary fp32 values, so almost every stored value has low mantissa bits to round away.

Outputs accumulated with fp32 atomics are exempt (their summation order varies between runs, and they are never an operand of
a tensor-core convolution): listed in EXEMPT below.  The conv entry points are covered by tests/test_gpu_conv_epilogue.py."""
import math

import pytest
import torch

from swapping_autoencoder_pytorch_b200 import backend

pytestmark = pytest.mark.gpu
DEV = "cuda"

EXEMPT = {
    "bias_act_backward: grad_bias": "per-channel sum with fp32 atomics",
    "bias_act_backward: grad_noise_weight": "scalar sum with fp32 atomics",
    "fir_act_backward: grad_bias": "per-channel sum with fp32 atomics",
    "modulate_backward: ds": "per-(image, channel) sum with fp32 atomics",
    "torgb_backward: gw": "[N, 3, C] sum over pixels with fp32 atomics",
    "conv wgrad / wgrad_modulated: dw, ds": "split-pixel sums with fp32 atomics (no round_tf32 argument)",
}


@pytest.fixture
def kern():
    k = backend.kernels()
    prev = (k.precision, k.round_tf32)
    k.precision = "tf32"
    yield k
    k.precision, k.round_tf32 = prev


def _randn(seed, *shape):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(*shape, device=DEV, generator=gen)


def rna_bits(t):
    return (t.contiguous().view(torch.int32) + 0x1000) & ~0x1FFF


def _off_on(kern, fn):
    kern.round_tf32 = False
    off = fn()
    kern.round_tf32 = True
    on = fn()
    return off, on


def _assert_rounded(off, on, what):
    assert on.shape == off.shape, what
    assert (off.contiguous().view(torch.int32) & 0x1FFF).any(), "%s: the unrounded output is already TF32" % what
    same = on.contiguous().view(torch.int32) == rna_bits(off)
    assert same.all(), "%s: %d of %d elements are not rna_tf32 of the unrounded output" % (what, int((~same).sum()),
                                                                                           same.numel())


TAPS4 = (0.125, 0.375, 0.375, 0.125)
TAPS3 = (0.25, 0.5, 0.25)


def _fir_kernel(taps):
    t = torch.tensor(taps, device=DEV)
    return torch.outer(t, t).contiguous()


# (id, channels, kernel taps, up, down, pad, separable)
FIR_CASES = [
    ("generic_strip_4x4", 8, TAPS4, 1, 1, (2, 1, 2, 1), False),
    ("generic_vec_up2", 8, TAPS4, 2, 1, (2, 1, 2, 1), False),
    ("generic_vec_down2", 8, TAPS3, 1, 2, (1, 1, 1, 1), False),
    ("generic_scalar", 3, TAPS3, 1, 1, (1, 1, 1, 1), False),
    ("separable_tma_11", 32, TAPS4, 1, 1, (2, 1, 2, 1), True),
    ("separable_11", 8, TAPS4, 1, 1, (2, 1, 2, 1), True),
    ("separable_12", 8, TAPS4, 1, 2, (1, 1, 1, 1), True),
    ("separable_21", 8, TAPS4, 2, 1, (2, 1, 2, 1), True),
]


@pytest.mark.parametrize("case", FIR_CASES, ids=[c[0] for c in FIR_CASES])
def test_upfirdn2d_rounding(kern, case):
    _, c, taps, up, down, pad, separable = case
    x = _randn(1, 2, 16, 16, c)
    k = _fir_kernel(taps)
    fn = lambda: kern.upfirdn2d(x, k, up, up, down, down, *pad, taps=(taps, taps) if separable else None)   # noqa: E731
    _assert_rounded(*_off_on(kern, fn), "upfirdn2d " + case[0])


@pytest.mark.parametrize("c", [8, 5])
@pytest.mark.parametrize("with_noise", [False, True])
def test_bias_act_rounding(kern, c, with_noise):
    """c = 8: the float4 kernel (size_x % 4 == 0); c = 5 on 3 x 5 x 5 pixels: the scalar one"""
    x = _randn(2, 3, 5, 5, c)
    b = _randn(3, c)
    noise = _randn(4, 3 * 5 * 5) if with_noise else None
    nw = torch.tensor([0.37], device=DEV) if with_noise else None
    fn = lambda: kern.bias_act(x, b, None, 3, 0, 0.2, math.sqrt(2), noise=noise, noise_weight=nw)   # noqa: E731
    _assert_rounded(*_off_on(kern, fn), "bias_act")


@pytest.mark.parametrize("c", [8, 5])
@pytest.mark.parametrize("with_noise", [False, True])
def test_bias_act_backward_rounding(kern, c, with_noise):
    g, out = _randn(5, 3, 5, 5, c), _randn(6, 3, 5, 5, c)
    noise = _randn(7, 3 * 5 * 5) if with_noise else None
    fn = lambda: kern.bias_act_backward(g, out, 0.2, math.sqrt(2), want_bias=True, noise=noise)[0]   # noqa: E731
    _assert_rounded(*_off_on(kern, fn), "bias_act_backward grad_in")


def test_fir_bias_act_rounding(kern):
    x = _randn(8, 2, 16, 16, 32)
    b, noise, nw = _randn(9, 32), _randn(10, 2 * 16 * 16), torch.tensor([0.37], device=DEV)

    def fn():
        y = kern.fir_bias_act(x, (TAPS4, TAPS4), (2, 1, 2, 1), b, noise, nw, 0.2, math.sqrt(2))
        assert y is not None
        return y
    _assert_rounded(*_off_on(kern, fn), "fir_bias_act")


def test_fir_act_backward_rounding(kern):
    g, act_out = _randn(11, 2, 16, 16, 32), _randn(12, 2, 16, 16, 32)

    def fn():
        r = kern.fir_act_backward(g, (TAPS4, TAPS4), act_out, (2, 1, 2, 1), 0.2, math.sqrt(2), want_bias=True)
        assert r is not None
        return r[0]
    _assert_rounded(*_off_on(kern, fn), "fir_act_backward grad_in")


@pytest.mark.parametrize("c", [8, 5])
def test_modulate_rounding(kern, c):
    """c = 8: the float4 kernels; c = 5: the scalar ones"""
    x, s, dy = _randn(13, 2, 6, 7, c), _randn(14, 2, c), _randn(15, 2, 6, 7, c)
    _assert_rounded(*_off_on(kern, lambda: kern.modulate(x, s)), "modulate")
    _assert_rounded(*_off_on(kern, lambda: kern.modulate_backward(dy, x, s)[0]), "modulate_backward dx")


@pytest.mark.parametrize("n", [64, 63])
@pytest.mark.parametrize("with_b", [False, True])
def test_add_scale_rounding(kern, n, with_b):
    """n = 64: add_scale_kernel<4>; n = 63: add_scale_kernel<1>"""
    a, b = _randn(16, n), _randn(17, n) if with_b else None
    _assert_rounded(*_off_on(kern, lambda: kern.add_scale(a, b, 1 / math.sqrt(2))), "add_scale")


def test_upsample2x_rounding(kern):
    skip, res, dy = _randn(18, 2, 5, 6, 8), _randn(19, 2, 10, 12, 8), _randn(20, 2, 10, 12, 8)
    _assert_rounded(*_off_on(kern, lambda: kern.upsample2x_add_scale(skip, res, 1 / math.sqrt(2))), "upsample2x_add_scale")
    _assert_rounded(*_off_on(kern, lambda: kern.upsample2x_backward(dy, 1 / math.sqrt(2))), "upsample2x_backward")


def test_pad_channels_rounding(kern):
    """an NCHW source (stride_c = H*W) and a channels-last one (stride_c = 1)"""
    x_nchw = _randn(21, 2, 3, 7, 7)
    x_cl = _randn(22, 2, 7, 7, 3).permute(0, 3, 1, 2)
    _assert_rounded(*_off_on(kern, lambda: kern.pad_channels(x_nchw, 8)), "pad_channels NCHW")
    _assert_rounded(*_off_on(kern, lambda: kern.pad_channels(x_cl, 8)), "pad_channels channels-last")


def test_filter_layouts_rounding(kern):
    """filter_prep and filter_modulate, both output layouts each"""
    w = _randn(23, 16, 8, 3, 3)
    off, on = _off_on(kern, lambda: kern.filter_prep(w, 1 / math.sqrt(72)))
    _assert_rounded(off[0], on[0], "filter_prep krsc")
    _assert_rounded(off[1], on[1], "filter_prep crsk")
    w_krsc, s = _randn(24, 16, 3, 3, 8), _randn(25, 2, 8)
    off, on = _off_on(kern, lambda: kern.filter_modulate(w_krsc, s, want_krsc=True, want_crsk=True))
    _assert_rounded(off[0], on[0], "filter_modulate nkrsc")
    _assert_rounded(off[1], on[1], "filter_modulate ncrsk")


def test_crop_gather_rounding(kern):
    gen = torch.Generator().manual_seed(26)
    q, num_crops = 6, 3
    flip = (torch.randint(0, 2, (q,), generator=gen) * 2 - 1).float().to(DEV)
    scale = (torch.rand(q, 2, generator=gen) * 0.4 + 0.5).to(DEV)
    offset = ((torch.rand(q, 2, generator=gen) * 2 - 1) * (1 - scale.cpu())).to(DEV)
    x = _randn(27, 2, 3, 40, 40)
    _assert_rounded(*_off_on(kern, lambda: kern.crop_gather(x, flip, scale, offset, num_crops, 17, 32)), "crop_gather")


def test_torgb_rounding(kern):
    x, s, w, b = _randn(28, 2, 8, 8, 32), _randn(29, 2, 32), _randn(30, 3, 32), _randn(31, 3)
    dy = _randn(32, 2, 3, 8, 8)
    off, on = _off_on(kern, lambda: kern.torgb_forward(x, s, w, b, 1 / math.sqrt(32)))
    _assert_rounded(off[..., :3], on[..., :3], "torgb_forward")
    assert not on[..., 3].any() and not off[..., 3].any()
    _assert_rounded(*_off_on(kern, lambda: kern.torgb_backward(dy, x, s, w, 1 / math.sqrt(32))[0]), "torgb_backward dx")
