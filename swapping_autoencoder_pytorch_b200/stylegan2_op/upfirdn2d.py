"""upfirdn2d with first- and second-order autograd, on the sm_90a FIR kernel.

Mirrors the public function and the two autograd.Function classes of the reference
(models/networks/stylegan2_op/upfirdn2d.py:24-159): forward = upsample / pad / FIR / downsample, backward = the
same primitive with the flipped taps, up and down exchanged and the "gradient padding", backward-of-backward =
the forward primitive again.  Tensors keep the reference's logical NCHW shape; storage is channels-last so the
kernel sees [major=N, H, W, minor=C] directly (the reference reshapes to [B*C, H, W, 1], upfirdn2d.py:104).
"""
import torch
from torch.autograd import Function

from .. import backend
from ..backend import nchw, nhwc


def _out_extent(n_in, up, down, p0, p1, k):
    return (n_in * up + p0 + p1 - k) // down + 1


class UpFirDn2dBackward(Function):
    """grad_input = upfirdn2d(grad_output, flipped taps, up<->down, g_pad)  (reference upfirdn2d.py:24-90)."""

    @staticmethod
    def forward(ctx, grad_output, kernel, grad_kernel, up, down, pad, g_pad, in_size, out_size, taps=None):
        gx0, gx1, gy0, gy1 = g_pad
        g = backend.kernels().upfirdn2d(nhwc(grad_output), grad_kernel, down[0], down[1], up[0], up[1],
                                        gx0, gx1, gy0, gy1, taps=_flip_taps(taps))
        # the adjoint can come out larger than the input when the forward dropped trailing rows; never here
        assert g.shape[1] == in_size[2] and g.shape[2] == in_size[3], (tuple(g.shape), tuple(in_size))
        ctx.save_for_backward(kernel)
        ctx.cfg = (up, down, pad, taps)
        return nchw(g)

    @staticmethod
    def backward(ctx, gradgrad_input):
        kernel, = ctx.saved_tensors
        up, down, pad, taps = ctx.cfg
        gg = backend.kernels().upfirdn2d(nhwc(gradgrad_input), kernel, up[0], up[1], down[0], down[1], *pad, taps=taps)
        return nchw(gg), None, None, None, None, None, None, None, None, None


class UpFirDn2d(Function):
    """Forward primitive (reference upfirdn2d.py:93-147)."""

    @staticmethod
    def forward(ctx, input, kernel, up, down, pad, taps=None):
        up_x, up_y = up
        down_x, down_y = down
        px0, px1, py0, py1 = pad
        kh, kw = kernel.shape
        _, _, in_h, in_w = input.shape
        out_h = _out_extent(in_h, up_y, down_y, py0, py1, kh)
        out_w = _out_extent(in_w, up_x, down_x, px0, px1, kw)
        # padding of the adjoint operator (reference :116-119)
        g_pad = (kw - px0 - 1,
                 in_w * up_x - out_w * down_x + px0 - up_x + 1,
                 kh - py0 - 1,
                 in_h * up_y - out_h * down_y + py0 - up_y + 1)
        ctx.save_for_backward(kernel, torch.flip(kernel, [0, 1]))
        ctx.cfg = (up, down, pad, g_pad, tuple(input.shape), (out_h, out_w), taps)
        out = backend.kernels().upfirdn2d(nhwc(input), kernel, up_x, up_y, down_x, down_y, px0, px1, py0, py1, taps=taps)
        return nchw(out)

    @staticmethod
    def backward(ctx, grad_output):
        kernel, flipped = ctx.saved_tensors
        up, down, pad, g_pad, in_size, out_size, taps = ctx.cfg
        grad_input = UpFirDn2dBackward.apply(grad_output, kernel, flipped, up, down, pad, g_pad, in_size, out_size, taps)
        return grad_input, None, None, None, None, None


def _flip_taps(taps):
    return None if taps is None else (tuple(reversed(taps[0])), tuple(reversed(taps[1])))


def upfirdn2d(input, kernel, up=1, down=1, pad=(0, 0), taps=None):
    """Same signature and semantics as reference upfirdn2d.py:150-159 (same pad on x and y).
    ``taps`` (extension): host-side 1-D factors ``(taps_y, taps_x)`` with ``kernel == outer(taps_y, taps_x)``; the
    FIR modules, which build ``kernel`` from a 1-D tap list, pass them to select the separable kernel."""
    return UpFirDn2d.apply(input, kernel, (up, up), (down, down), (pad[0], pad[1], pad[0], pad[1]), taps)
