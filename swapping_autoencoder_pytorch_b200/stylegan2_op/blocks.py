"""Block-level autograd Functions: one node per residual block instead of one per operator.

Why: autograd sums the gradients of a tensor that feeds two branches with a separate ``add`` pass.  In the
discriminators' ResBlock (reference models/networks/stylegan2_layers.py:672-693) the block input feeds ``conv1`` and the
blurred ``skip`` branch, so every backward pays a read-read-write pass over the largest activation of the block
(1.07 GB at 128 channels x 256 x 256 x 32 images).  A hand-ordered block backward lets the last data-gradient kernel add
the other branch's gradient in its epilogue (``residual`` of the conv kernels) — the sum never exists as a pass.

Second order (R1, reference swapping_autoencoder_model.py:138-185).  The R1 penalty differentiates the gradient of the
prediction with respect to the IMAGE (or the crops): ``autograd.grad(pred, [real], create_graph=True)`` then
``penalty.backward()``.  A discriminator is piecewise linear in its input — bilinear convolutions, linear FIRs, and leaky-ReLU
masks that are constant almost everywhere — so for a block  y = M2 C2 B2 M1 C1 x + Cs Bs x  (C: conv, B: blur, M: mask x gain)

    first backward      dx = C1' M1 B2' C2' M2 dy + Bs' Cs' dy                         (the fused data-gradient chain)
    second backward     given the cotangent v of dx:
                          d(dy) = M2 C2 B2 M1 C1 v + Cs Bs v                           (the block's forward on v, saved masks)
                          dW1 = wgrad(M1 B2' C2' M2 dy, v)    dW2 = wgrad(M2 dy, B2 M1 C1 v)    dWs = wgrad(dy, Bs v)

i.e. forward + data-gradient chain + tangent forward + one weight gradient per conv = 4 forward-equivalents, all on the
block's fused kernels (``_ResBlockDataGrad``).  That path is taken inside ``data_gradients_only()`` — the scope
``compute_R1_loss`` opens to say that recorded backward passes are asked for data gradients only.  Outside that scope a
recorded backward re-evaluates the block with the per-operator differentiable Functions of conv.py / fused_act.py /
upfirdn2d.py and differentiates THAT (general, slower; what the reference's own unchanged model file gets).
"""
import os

import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from .. import backend
from ..backend import make_geom, nchw, nhwc
from . import conv as C
from .upfirdn2d import _flip_taps, upfirdn2d


_enabled = [os.environ.get("SAE_FUSED_BLOCKS", "1") != "0"]


def fused_blocks_enabled():
    return _enabled[0]


def set_fused_blocks(flag):
    """switch between block-level and per-operator autograd nodes (tests compare the two); returns the previous value"""
    prev, _enabled[0] = _enabled[0], bool(flag)
    return prev


class per_operator_blocks:
    """``with per_operator_blocks():`` — build per-operator autograd nodes inside the scope.  A caller that knows it
    will differentiate the backward (compute_R1_loss) uses it to skip the block node's forward, which the node would
    have to repeat in per-operator form anyway once the backward is recorded."""

    def __enter__(self):
        self.prev = set_fused_blocks(False)

    def __exit__(self, *exc):
        set_fused_blocks(self.prev)
        return False


class data_gradients_only:
    """``with data_gradients_only():`` — promise of the caller (compute_R1_loss) that every backward pass recorded inside the
    scope (``create_graph=True``) is asked for gradients with respect to activations only (the image, the crops).  The
    recorded backward then skips the weight / bias gradients it would otherwise compute, record and throw away, and the
    fused blocks use their closed-form double backward."""

    def __enter__(self):
        self.prev = C.set_data_gradients_only(True)

    def __exit__(self, *exc):
        C.set_data_gradients_only(self.prev)
        return False


class FirSpec:
    """a Blur module's parameters as plain host data + the derived adjoint padding (upfirdn2d.py UpFirDn2d.forward)"""

    def __init__(self, kernel, pad, taps, down):
        self.kernel, self.pad, self.taps, self.down = kernel, (int(pad[0]), int(pad[1])), taps, int(down)

    def out_extent(self, n):
        return (n + self.pad[0] + self.pad[1] - self.kernel.shape[0]) // self.down + 1

    def forward(self, k, x):
        p0, p1 = self.pad
        return k.upfirdn2d(x, self.kernel, 1, 1, self.down, self.down, p0, p1, p0, p1, taps=self.taps)

    def _adjoint_pad(self, g, in_h, in_w):
        p0 = self.pad[0]
        kh, kw = self.kernel.shape
        d = self.down
        out_h, out_w = g.shape[1], g.shape[2]
        return kw - p0 - 1, in_w - out_w * d + p0, kh - p0 - 1, in_h - out_h * d + p0

    def adjoint(self, k, g, in_h, in_w):
        """gradient w.r.t. the FIR input of extent (in_h, in_w): flipped taps, up <-> down, gradient padding"""
        d = self.down
        out = k.upfirdn2d(g, torch.flip(self.kernel, [0, 1]), d, d, 1, 1, *self._adjoint_pad(g, in_h, in_w),
                          taps=_flip_taps(self.taps))
        assert out.shape[1] == in_h and out.shape[2] == in_w, (tuple(out.shape), in_h, in_w)
        return out

    def adjoint_into_activation(self, k, g, act_out, slope, gain, want_bias, mask=None):
        """``bias_act_backward(adjoint(g), act_out)`` — in one kernel when the fused FIR + activation-backward kernel
        takes the shape (the blurred gradient then never exists in HBM), as two launches otherwise.
        mask: the activation bit mask of ``act_out`` if its producer wrote one"""
        in_h, in_w = act_out.shape[1], act_out.shape[2]
        if self.down == 1 and self.taps is not None:
            hit = k.fir_act_backward(g, _flip_taps(self.taps), act_out, self._adjoint_pad(g, in_h, in_w), slope, gain,
                                     want_bias=want_bias, mask=mask)
            if hit is not None:
                return hit
        gi, gb, _ = k.bias_act_backward(self.adjoint(k, g, in_h, in_w), act_out, slope, gain, want_bias=want_bias, mask=mask)
        return gi, gb


class _FirNoiseBiasAct(Function):
    """lrelu(blur(x) + noise_weight * noise + bias) * gain — the Blur behind the generator's transposed convolution and the
    StyledConv tail after it (stylegan2_layers.py:306-309, :398-405) in ONE kernel (``sae_fir_bias_act``): the blurred tensor
    never exists in HBM.  Backward: masked gradient + bias / noise-weight gradients in one pass, then the adjoint FIR.
    Generator only, hence once-differentiable."""

    @staticmethod
    def forward(ctx, x, spec, noise, noise_weight, bias, slope, gain):
        k = backend.kernels()
        xh = nhwc(x)
        p0, p1 = spec.pad
        noise_flat = noise.reshape(-1).contiguous() if noise is not None else None
        nw = noise_weight.contiguous() if noise is not None else None
        out = None
        if spec.taps is not None and spec.down == 1:
            out = k.fir_bias_act(xh, spec.taps, (p0, p1, p0, p1), bias.contiguous(), noise_flat, nw, slope, gain)
        if out is None:
            out = k.bias_act(spec.forward(k, xh), bias.contiguous(), None, 3, 0, slope, gain, noise=noise_flat, noise_weight=nw)
        ctx.spec, ctx.cfg = spec, (slope, gain, tuple(noise.shape) if noise is not None else None, xh.shape[1], xh.shape[2])
        ctx.act_mask = backend.act_mask_of(out)
        ctx.save_for_backward(out, noise_flat, nw)
        return nchw(out)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        out, noise_flat, nw = ctx.saved_tensors
        slope, gain, noise_shape, in_h, in_w = ctx.cfg
        k = backend.kernels()
        gi, gb, gnw = k.bias_act_backward(nhwc(dy), out, slope, gain, want_bias=True, noise=noise_flat, mask=ctx.act_mask)
        dx = nchw(ctx.spec.adjoint(k, gi, in_h, in_w)) if ctx.needs_input_grad[0] else None
        g_noise = None
        if noise_flat is not None and ctx.needs_input_grad[2]:
            g_noise = (gi.sum(dim=3) * nw).reshape(noise_shape)
        return dx, None, g_noise, gnw, gb, None, None


def fir_noise_bias_act(x, spec, noise, noise_weight, bias, slope, gain):
    """``fused_leaky_relu(upfirdn2d(x, kernel, pad=spec.pad) + noise_weight * noise, bias, slope, gain)`` in one pass"""
    return _FirNoiseBiasAct.apply(x, spec, noise, noise_weight, bias, slope, gain)


class ResBlockSpec:
    """host-side constants of one ResBlock (scales, activation constants, the two FIRs)"""

    def __init__(self, s1, s2, ss, slope, gain1, gain2, blur2, blur_s):
        self.s1, self.s2, self.ss, self.slope, self.gain1, self.gain2 = s1, s2, ss, slope, gain1, gain2
        self.blur2, self.blur_s = blur2, blur_s


def resblock_unfused(x, w1, b1, w2, b2, ws, spec):
    """The block as a composition of the per-operator differentiable Functions (first and second order)."""
    o1 = C.conv2d_bias_act(x, w1, b1, stride=1, padding=1, negative_slope=spec.slope, scale=spec.gain1, wscale=spec.s1)
    bl = upfirdn2d(o1, spec.blur2.kernel, pad=spec.blur2.pad, taps=spec.blur2.taps)
    o2 = C.conv2d_bias_act(bl, w2, b2, stride=2, padding=0, negative_slope=spec.slope, scale=spec.gain2, wscale=spec.s2)
    h = upfirdn2d(x, spec.blur_s.kernel, down=2, pad=spec.blur_s.pad, taps=spec.blur_s.taps)
    return C.conv2d_residual(h, ws, o2, 1.0, stride=1, padding=0, wscale=spec.ss)


class _ResBlockDataGrad(Function):
    """dx of the fused block as a differentiable function of (dy, w1, w2, ws): the recorded form of the block's data
    gradient inside ``data_gradients_only()``.  Its backward is the closed form in the module docstring."""

    @staticmethod
    def forward(ctx, dy, w1, w2, ws, o1, o2, w1k, w1t, w2k, w2t, wsk, wst, spec, geoms, masks):
        k = backend.kernels()
        g1, g2, gs = geoms
        m1, m2 = masks
        dyh = nhwc(dy)
        gi2, _, _ = k.bias_act_backward(dyh, o2, spec.slope, spec.gain2, want_bias=False, mask=m2)
        dh = k.conv_dgrad(dyh, wsk, gs, w_crsk=wst)
        dxs = spec.blur_s.adjoint(k, dh, g1.H, g1.W)
        dbl = k.conv_dgrad(gi2, w2k, g2, w_crsk=w2t)
        gi1, _ = spec.blur2.adjoint_into_activation(k, dbl, o1, spec.slope, spec.gain1, False, mask=m1)
        dx = k.conv_dgrad(gi1, w1k, g1, w_crsk=w1t, residual=dxs, res_scale=1.0)
        ctx.spec, ctx.geoms, ctx.masks = spec, geoms, masks
        ctx.save_for_backward(dyh, gi2, gi1, o1, o2, w1k, w2k, wsk)
        return nchw(dx)

    @staticmethod
    @once_differentiable
    def backward(ctx, v):
        dyh, gi2, gi1, o1, o2, w1k, w2k, wsk = ctx.saved_tensors
        spec = ctx.spec
        g1, g2, gs = ctx.geoms
        m1, m2 = ctx.masks
        k = backend.kernels()
        need = ctx.needs_input_grad
        vh = nhwc(v)
        # tangent forward through the linearised block: no biases, the saved leaky-ReLU masks
        r = None
        if need[0] or need[2]:
            p1 = k.conv_fprop(vh, w1k, g1, prepared=True)
            q1, _, _ = k.bias_act_backward(p1, o1, spec.slope, spec.gain1, want_bias=False, mask=m1)
            r = spec.blur2.forward(k, q1)
        hv = spec.blur_s.forward(k, vh) if (need[0] or need[3]) else None
        d_dy = None
        if need[0]:
            p2 = k.conv_fprop(r, w2k, g2, prepared=True)
            t2, _, _ = k.bias_act_backward(p2, o2, spec.slope, spec.gain2, want_bias=False, mask=m2)
            d_dy = nchw(k.conv_fprop(hv, wsk, gs, prepared=True, residual=t2, res_scale=1.0))
        unprep = k.filter_unprep
        dw1 = unprep(k.conv_wgrad(gi1, vh, g1), spec.s1) if need[1] else None
        dw2 = unprep(k.conv_wgrad(gi2, r, g2), spec.s2) if need[2] else None
        dws = unprep(k.conv_wgrad(dyh, hv, gs), spec.ss) if need[3] else None
        return (d_dy, dw1, dw2, dws) + (None,) * 11


class _ResBlockFused(Function):
    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2, ws, spec):
        k = backend.kernels()
        n, c, hh, ww = x.shape
        co = w2.shape[0]
        w1k, w1t = C.prep_filter(w1, spec.s1)
        w2k, w2t = C.prep_filter(w2, spec.s2)
        wsk, wst = C.prep_filter(ws, spec.ss)
        xh = nhwc(x)
        g1 = make_geom(n, hh, ww, c, c, 3, 3, 1, 1, 1)
        o1 = k.conv_fprop(xh, w1k, g1, prepared=True, bias=b1.contiguous(), act=3, alpha=spec.slope, gain=spec.gain1)
        bl = spec.blur2.forward(k, o1)
        g2 = make_geom(n, bl.shape[1], bl.shape[2], c, co, 3, 3, 2, 0, 0)
        o2 = k.conv_fprop(bl, w2k, g2, prepared=True, bias=b2.contiguous(), act=3, alpha=spec.slope, gain=spec.gain2)
        h = spec.blur_s.forward(k, xh)
        gs = make_geom(n, h.shape[1], h.shape[2], c, co, 1, 1, 1, 0, 0)
        assert (gs.P, gs.Q) == (g2.P, g2.Q), ("ResBlock branches disagree", gs.key(), g2.key())
        y = k.conv_fprop(h, wsk, gs, prepared=True, residual=o2, res_scale=1.0)
        ctx.spec, ctx.geoms = spec, (g1, g2, gs)
        ctx.masks = (backend.act_mask_of(o1), backend.act_mask_of(o2))        # activation bit masks written by the two convs
        ctx.save_for_backward(x, w1, b1, w2, b2, ws, o1, bl, o2, h, w1k, w1t, w2k, w2t, wsk, wst)
        return nchw(y)

    @staticmethod
    def backward(ctx, dy):
        x, w1, b1, w2, b2, ws, o1, bl, o2, h, w1k, w1t, w2k, w2t, wsk, wst = ctx.saved_tensors
        spec = ctx.spec
        need = ctx.needs_input_grad
        if torch.is_grad_enabled() and C.data_gradients_only_active():
            # R1: the recorded backward is asked for dx only; closed-form double backward (module docstring)
            dx = None
            if need[0]:
                dx = _ResBlockDataGrad.apply(dy, w1, w2, ws, o1, o2, w1k, w1t, w2k, w2t, wsk, wst, spec, ctx.geoms, ctx.masks)
            return (dx, None, None, None, None, None, None)
        if torch.is_grad_enabled():
            # the backward is being recorded by a general caller: differentiate the per-operator composition instead
            ins = [t for t, nd in zip((x, w1, b1, w2, b2, ws), need) if nd]
            with torch.enable_grad():
                y = resblock_unfused(x, w1, b1, w2, b2, ws, spec)
                got = iter(torch.autograd.grad(y, ins, dy, create_graph=True, allow_unused=True))
            return tuple(next(got) if nd else None for nd in need[:6]) + (None,)
        k = backend.kernels()
        g1, g2, gs = ctx.geoms
        m1, m2 = ctx.masks
        dyh = nhwc(dy)
        need_x, need_w = need[0], (need[1] or need[3] or need[5])
        gi2, gb2, _ = k.bias_act_backward(dyh, o2, spec.slope, spec.gain2, want_bias=need[4], mask=m2)
        # skip branch: 1x1 conv <- decimating blur
        dws = k.conv_wgrad(dyh, h, gs) if need[5] else None
        dxs = None
        if need_x:
            dh = k.conv_dgrad(dyh, wsk, gs, w_crsk=wst)
            dxs = spec.blur_s.adjoint(k, dh, g1.H, g1.W)
        # main branch: conv2 (stride 2) <- blur <- conv1
        dw2 = k.conv_wgrad(gi2, bl, g2) if need[3] else None
        dx = gi1 = gb1 = dw1 = None
        if need_x or need[1] or need[2]:
            dbl = k.conv_dgrad(gi2, w2k, g2, w_crsk=w2t)
            gi1, gb1 = spec.blur2.adjoint_into_activation(k, dbl, o1, spec.slope, spec.gain1, need[2], mask=m1)
            if need[1]:
                dw1 = k.conv_wgrad(gi1, nhwc(x), g1)
            if need_x:
                # the other branch's gradient is added in this kernel's epilogue: no separate accumulation pass
                dx = nchw(k.conv_dgrad(gi1, w1k, g1, w_crsk=w1t, residual=dxs, res_scale=1.0))
        unprep = k.filter_unprep
        return (dx,
                unprep(dw1, spec.s1) if dw1 is not None else None, gb1 if need[2] else None,
                unprep(dw2, spec.s2) if dw2 is not None else None, gb2 if need[4] else None,
                unprep(dws, spec.ss) if dws is not None else None, None)


def resblock(x, w1, b1, w2, b2, ws, spec):
    """conv1 (3x3) -> blur -> conv2 (3x3, stride 2), plus blur-decimate -> 1x1 skip, merged as (out + skip) / sqrt(2)
    with the factor pre-folded into ``spec.gain2`` / ``spec.ss`` (reference stylegan2_layers.py:672-693)."""
    return _ResBlockFused.apply(x, w1, b1, w2, b2, ws, spec)
