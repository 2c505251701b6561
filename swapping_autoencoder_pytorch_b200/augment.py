"""Adaptive discriminator augmentation (extension; INTEGRATION.md §2h).

StyleGAN2-ADA's 'bgc' pipeline (Karras et al., NeurIPS 2020, §2-3 and Appendix B) at its default strengths, applied to every
image the image discriminator D sees, with one probability p for every transform, and p tuned on the device from the sign
of D's logits on the (augmented) reals.  Per image:

* geometric: G_inv (x-flip, rotation by 90°, integer translation, isotropic scale, rotation, anisotropic scale, rotation,
  fractional translation), executed as reflect pad by (W - 1, H - 1) -> sym6 2x upsample -> bilinear sample on the
  transformed grid (sae_augment_sample, one fused kernel) -> sym6 2x downsample (the upfirdn2d kernels).  An image whose
  G_inv is exactly I is copied, not resampled;
* colour: C (brightness, contrast, luma flip, hue rotation, saturation), rgb <- C[:3, :3] rgb + C[:3, 3] (sae_augment_color).

The operator is affine in the image, so its backward is its (linear) adjoint and the adjoint's backward is the linear part
of the operator: ``augment`` is twice differentiable, which R1 (closed-form D double backward) needs.  Nothing here rounds to
TF32, in either precision mode.
"""
import math

import torch

from . import _lib, backend
from .backend import nchw

# StyleGAN2-ADA's sym6 wavelet low-pass (sums to sqrt(2)); the filter below is it normalised to sum 1
SYM6 = (0.015404109327027373, 0.0034907120842174702, -0.11799011114819057, -0.048311742585633, 0.4910559419267466,
        0.787641141030194, 0.3379294217276218, -0.07263752278646252, -0.021060292512300564, 0.04472490177066578,
        0.0017677118642428036, -0.007800708325034148)
_F = tuple(v / sum(SYM6) for v in SYM6)
_DOWN_TAPS = tuple(reversed(_F))          # the downsampling filter is flipped (ADA's flip_filter=True)


def _fir_kernel(ref, taps):
    """the 2-D filter outer(taps, taps) on ref's device and dtype, built once (the eager warm-up calls build it, outside any
    capture)"""
    key = (ref.device, ref.dtype, taps)
    k = _fir_kernel.cache.get(key)
    if k is None:
        t = torch.tensor(taps, dtype=ref.dtype)
        k = torch.outer(t, t).to(ref.device)
        _fir_kernel.cache[key] = k
    return k


_fir_kernel.cache = {}


def _downsample(s):
    """S (NHWC [N, 2(H + 6), 2(W + 6), 4]) -> NHWC [N, H, W, 4]: upfirdn2d(S, flip(f) (x) flip(f), down=2, pad=(-1, -1)).  The
    fourth channel is zero: four channels let the FIR kernel move one float4 per pixel"""
    return backend.kernels().upfirdn2d(s, _fir_kernel(s, _DOWN_TAPS), 1, 1, 2, 2, -1, -1, -1, -1, round_tf32=False)


def _downsample_adjoint(g):
    """adjoint of ``_downsample``: NHWC [N, H, W, 4] -> [N, 2(H + 6), 2(W + 6), 4] (upfirdn2d's gradient padding; the
    adjoint's filter is the forward's flipped, f (x) f)"""
    return backend.kernels().upfirdn2d(g, _fir_kernel(g, _F), 2, 2, 1, 1, 12, 11, 12, 11, round_tf32=False)


def _apply(x, rec, offset, copy_identity):
    """the operator: logical [N, 3, H, W] (any strides) -> NHWC [N, H, W, 3]"""
    k = backend.kernels()
    return k.augment_color(x, _downsample(k.augment_sample(x, rec, copy_identity)), rec, offset=offset,
                           copy_identity=copy_identity)


def _adjoint(dy, rec, copy_identity):
    """the adjoint of the operator's linear part: logical [N, 3, H, W] (any strides) -> NHWC [N, H, W, 3]"""
    k = backend.kernels()
    gc = k.augment_color_adjoint(dy, rec)
    return k.augment_sample_adjoint(_downsample_adjoint(gc), gc, rec, dy.shape[2], dy.shape[3], copy_identity)


# The operator and its adjoint are torch.library custom ops whose registered backwards call each other: the operator's backward
# is the adjoint, the adjoint's backward the operator's linear part (offset=False), so autograd differentiates it twice.
@torch.library.custom_op("sae_b200::augment", mutates_args=())
def _augment_op(x: torch.Tensor, rec: torch.Tensor, offset: bool, copy_identity: bool) -> torch.Tensor:
    return nchw(_apply(x, rec, offset, copy_identity))


@torch.library.custom_op("sae_b200::augment_adjoint", mutates_args=())
def _augment_adjoint_op(dy: torch.Tensor, rec: torch.Tensor, copy_identity: bool) -> torch.Tensor:
    return nchw(_adjoint(dy, rec, copy_identity))


def _save_rec(ctx, inputs, output):
    ctx.save_for_backward(inputs[1])
    ctx.copy_identity = inputs[-1]


def _augment_backward(ctx, grad):
    rec, = ctx.saved_tensors
    return _augment_adjoint_op(grad, rec, ctx.copy_identity), None, None, None


def _augment_adjoint_backward(ctx, gg):
    rec, = ctx.saved_tensors
    return _augment_op(gg, rec, False, ctx.copy_identity), None, None


torch.library.register_autograd("sae_b200::augment", _augment_backward, setup_context=_save_rec)
torch.library.register_autograd("sae_b200::augment_adjoint", _augment_adjoint_backward, setup_context=_save_rec)


def linear(x, rec, copy_identity=True):
    """the operator without the colour offset (its linear part), twice differentiable"""
    return _augment_op(x, rec, False, bool(copy_identity))


def adjoint(dy, rec, copy_identity=True):
    """the adjoint of the linear part, twice differentiable"""
    return _augment_adjoint_op(dy, rec, bool(copy_identity))


def augment(x, rec, copy_identity=True):
    """x: logical [N, 3, H, W] fp32 images; rec: [N, SAE_AUG_RECORD] per-image records (``params``).  Returns the augmented
    images, logical [N, 3, H, W] (channels-last storage); twice differentiable in x.  copy_identity=False forces images
    whose G_inv is I through the resampler as well (tests)."""
    return _augment_op(x, rec, True, bool(copy_identity))


def draw(n, device, dtype=torch.float32):
    """the per-image draws of one call: uniforms [n, SAE_AUG_UNIFORMS] and normals [n, SAE_AUG_NORMALS], from torch's
    generator of ``device`` (capturable in a CUDA graph); their number does not depend on p"""
    u = torch.rand(n, _lib.SAE_AUG_UNIFORMS, device=device, dtype=dtype)
    z = torch.randn(n, _lib.SAE_AUG_NORMALS, device=device, dtype=dtype)
    return u, z


def params(u, z, p, h, w):
    """per-image records (G_inv, C) from the draws and the one-element device probability p, for h x w images"""
    return backend.kernels().augment_params(u, z, p, h, w)


class AugmentPipe:
    """The augmentation and its probability p (opt.augment_p, opt.ada_target; INTEGRATION.md §2h).  p is a one-element fp32
    device tensor and ``acc`` the four fp64 sums of ``score_stats`` over D's logits on the augmented reals; both live
    outside any CUDA-graph pool and are updated in place, so captured half-steps read and write them on every replay.

    * ``__call__(images)``: one draw for all of them (the model passes real, rec and mix concatenated), one launch for the
      records, then the operator;
    * ``observe(logits)``: the D step adds the signs of D(real) to ``acc`` (one launch, capturable);
    * ``adjust(images_per_update)``: after every ``interval``-th D update, one launch moves p by
      sign(E[sign(D(real))] - target) * images * interval / (kimg * 1000) and clears ``acc``; with more than one rank the
      sums are all-reduced first, so p stays bitwise identical on every rank."""

    def __init__(self, p, target, kimg, interval, device, world=1):
        self.target, self.kimg, self.interval, self.world = float(target), float(kimg), int(interval), world
        self.p = torch.full((1,), float(p), dtype=torch.float32, device=device)
        self.acc = torch.zeros(4, dtype=torch.float64, device=device)

    def tuning(self):
        return self.target > 0.0

    def __call__(self, images):
        n, _, h, w = images.shape
        u, z = draw(n, images.device, images.dtype)
        rec = params(u, z, self.p.to(images.dtype), h, w)
        return augment(images, rec)

    @torch.no_grad()
    def observe(self, logits):
        if self.tuning():
            backend.kernels().score_stats(logits.detach(), self.acc)

    @torch.no_grad()
    def adjust(self, images_per_update):
        """images_per_update: the D update's images on this rank (the world factor is applied here)"""
        if self.world > 1:
            import torch.distributed as dist
            dist.all_reduce(self.acc)
        step = images_per_update * self.world * self.interval / (self.kimg * 1000.0)
        backend.kernels().ada_adjust(self.p, self.acc, step, self.target)

    def value(self):
        return float(self.p.item())

    def state_dict(self):
        return {"p": self.p.detach().clone(), "acc": self.acc.detach().clone()}

    def load_state_dict(self, sd):
        """in place: captured graphs hold p and acc"""
        with torch.no_grad():
            self.p.copy_(torch.as_tensor(sd["p"]).reshape(1))
            self.acc.copy_(torch.as_tensor(sd["acc"]).reshape(4))


def check_options(p, target, kimg, interval):
    """ValueError for an out-of-range augmentation option; True when the augmentation is on"""
    if not (math.isfinite(p) and p >= 0.0):
        raise ValueError("opt.augment_p must be a finite number >= 0, got %r" % (p,))
    if not (math.isfinite(target) and 0.0 <= target < 1.0):
        raise ValueError("opt.ada_target must lie in [0, 1), got %r" % (target,))
    if not (math.isfinite(kimg) and kimg > 0.0):
        raise ValueError("opt.ada_kimg must be a finite number > 0, got %r" % (kimg,))
    if isinstance(interval, bool) or not isinstance(interval, int) or interval < 1:
        raise ValueError("opt.ada_interval must be a positive integer, got %r" % (interval,))
    return p > 0.0 or target > 0.0
