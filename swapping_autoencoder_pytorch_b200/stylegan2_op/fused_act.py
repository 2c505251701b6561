"""Fused bias + leaky-ReLU (+ NoiseInjection) with first- and second-order autograd.

Mirrors reference models/networks/stylegan2_op/fused_act.py:23-96 (FusedLeakyReLUFunction, its Backward function
with a differentiable backward, the FusedLeakyReLU module and fused_leaky_relu).  The backward pass fuses the
per-channel bias-gradient reduction into the masking kernel (the reference runs a separate .sum, :41).
"""
import torch
from torch import nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from .. import backend
from ..backend import nchw, nhwc


def _cl(t):
    """the kernels' layout of an activation: NHWC for a feature map, a [B, C] matrix as it is"""
    return nhwc(t) if t.dim() > 2 else t.contiguous()


def _uncl(t):
    return nchw(t) if t.dim() > 2 else t


class FusedLeakyReLUFunctionBackward(Function):
    @staticmethod
    def forward(ctx, grad_output, out, negative_slope, scale, mask=None):
        """mask: activation bit mask of ``out`` if its producer wrote one (backend.act_mask_of) — the first-order pass then reads
        1 bit per element instead of ``out``; the second-order pass below keeps using ``out``"""
        ctx.save_for_backward(out)
        ctx.cfg = (negative_slope, scale)
        gi, gb, _ = backend.kernels().bias_act_backward(_cl(grad_output), _cl(out), negative_slope, scale,
                                                        want_bias=True, mask=mask)
        return _uncl(gi), gb

    @staticmethod
    def backward(ctx, gradgrad_input, gradgrad_bias):
        out, = ctx.saved_tensors
        negative_slope, scale = ctx.cfg
        # same mask applied to (gg_input + gg_bias[c])  — reference fused_act.py:45-52
        if gradgrad_input is None:
            gradgrad_input = torch.zeros_like(out)
        gg = backend.kernels().bias_act(_cl(gradgrad_input), gradgrad_bias.contiguous() if gradgrad_bias is not None else None,
                                        _cl(out), 3, 1, negative_slope, scale)
        return _uncl(gg), None, None, None, None


class FusedLeakyReLUFunction(Function):
    @staticmethod
    def forward(ctx, input, bias, negative_slope, scale):
        out = backend.kernels().bias_act(_cl(input), bias.contiguous(), None, 3, 0, negative_slope, scale)
        out = _uncl(out)
        ctx.save_for_backward(out)
        ctx.cfg = (negative_slope, scale)
        return out

    @staticmethod
    def backward(ctx, grad_output):
        out, = ctx.saved_tensors
        negative_slope, scale = ctx.cfg
        # detached mask: see _ConvBiasAct.backward (stylegan2_op/conv.py)
        grad_input, grad_bias = FusedLeakyReLUFunctionBackward.apply(grad_output, out.detach(), negative_slope, scale)
        return grad_input, grad_bias, None, None


class _NoiseBiasLeakyReLU(Function):
    """lrelu(x + w * noise + b) * scale in one pass: NoiseInjection (stylegan2_layers.py:328-351) folded into
    FusedLeakyReLU.  Used only by the generator, which is never differentiated twice (SURVEY.md §8 a16)."""

    @staticmethod
    def forward(ctx, input, noise, noise_weight, bias, negative_slope, scale):
        k = backend.kernels()
        noise_cl = noise.reshape(-1).contiguous()          # [B,1,H,W] -> one value per pixel
        out = _uncl(k.bias_act(_cl(input), bias.contiguous(), None, 3, 0, negative_slope, scale,
                               noise=noise_cl, noise_weight=noise_weight.contiguous()))
        ctx.save_for_backward(out, noise_cl, noise_weight)
        ctx.cfg = (negative_slope, scale, tuple(noise.shape))
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        out, noise_cl, noise_weight = ctx.saved_tensors
        negative_slope, scale, noise_shape = ctx.cfg
        gi, gb, gnw = backend.kernels().bias_act_backward(_cl(grad_output), _cl(out), negative_slope, scale,
                                                          want_bias=True, noise=noise_cl)
        gi = _uncl(gi)
        g_noise = None
        if ctx.needs_input_grad[1]:        # trainable fixed_noise (base_network.py:41-49)
            g_noise = (gi.sum(dim=1, keepdim=True) * noise_weight).reshape(noise_shape)
        return gi, g_noise, gnw, gb, None, None


class FusedLeakyReLU(nn.Module):
    """reference fused_act.py:77-86"""

    def __init__(self, channel, negative_slope=0.2, scale=2 ** 0.5):
        super().__init__()
        self.bias = nn.Parameter(torch.zeros(channel))
        self.negative_slope = negative_slope
        self.scale = scale

    def forward(self, input):
        return fused_leaky_relu(input, self.bias, self.negative_slope, self.scale)


def fused_leaky_relu(input, bias, negative_slope=0.2, scale=2 ** 0.5):
    """reference fused_act.py:89-96 (the custom-kernel branch; there is no native fallback here)"""
    return FusedLeakyReLUFunction.apply(input, bias, negative_slope, scale)


def fused_noise_bias_leaky_relu(input, noise, noise_weight, bias, negative_slope=0.2, scale=2 ** 0.5):
    return _NoiseBiasLeakyReLU.apply(input, noise, noise_weight, bias, negative_slope, scale)
