"""Tensor-level entry points of the hot path: thin wrappers that allocate outputs with torch and pass raw
device pointers + the current CUDA stream to the C ABI (include/sae_b200.h).

All activations here are *physical* NHWC: contiguous ``[N, H, W, C]`` (or ``[B, C]``) fp32 CUDA tensors.
The autograd layer in ``stylegan2_op`` converts from / to the logical NCHW shapes the reference's modules
expose.  ``set_kernels`` lets the CPU test-suite swap in an emulation built on the oracle so the host-side
autograd logic can be grad-checked without a GPU; the product never does that — ``CudaKernels`` raises if
the shared library is missing or a tensor lives on the CPU.
"""
import ctypes
import os

import torch

from . import _lib
from ._lib import ConvEpilogue, ConvGeom, check


def make_geom(N, H, W, C, K, R, S, stride, pad_t, pad_l, P=None, Q=None):
    """Geometry of y[n,p,q,k] = sum x[n, p*stride - pad_t + r, q*stride - pad_l + s, c] w[k,r,s,c].
    P/Q default to the F.conv2d rule with symmetric padding (pad_t on both sides)."""
    if P is None:
        P = (H + 2 * pad_t - R) // stride + 1
    if Q is None:
        Q = (W + 2 * pad_l - S) // stride + 1
    return ConvGeom(N, H, W, C, K, R, S, P, Q, stride, pad_t, pad_l)


PRECISIONS = ("tf32", "fp32")


def parse_precision(value):
    """``SAE_PRECISION`` / ``CudaKernels.precision`` value -> "tf32" (unset or empty: the default) or "fp32"; anything else
    raises ValueError"""
    v = "" if value is None else str(value).strip().lower()
    if v == "":
        return "tf32"
    if v not in PRECISIONS:
        raise ValueError("unknown precision %r (SAE_PRECISION): expected one of %s" % (value, ", ".join(PRECISIONS)))
    return v


def parse_deterministic(value):
    """``SAE_DETERMINISTIC`` value -> bool: unset, "" or "0" off, "1" on; anything else raises ValueError"""
    v = "" if value is None else str(value).strip()
    if v not in ("", "0", "1"):
        raise ValueError("unknown SAE_DETERMINISTIC value %r: expected 0 or 1" % (value,))
    return v == "1"


def nhwc(t):
    """logical NCHW tensor -> the physical NHWC storage the kernels take (contiguous [N, H, W, C])"""
    return t.permute(0, 2, 3, 1).contiguous()


def nchw(t):
    """physical NHWC tensor -> its logical NCHW view (no copy)"""
    return t.permute(0, 3, 1, 2)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _floats(v):
    """host float array (FIR tap lists)"""
    return (ctypes.c_float * len(v))(*v)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _need_cuda(*ts, strided=False):
    for t in ts:
        if t is None:
            continue
        if not t.is_cuda:
            raise _lib.SaeError("sae_b200 kernels need CUDA tensors (got a %s tensor); there is no CPU fallback"
                                % t.device.type)
        if t.dtype != torch.float32:
            raise _lib.SaeError("sae_b200 kernels are fp32-only (got %s)" % t.dtype)
        if not strided and not t.is_contiguous():
            raise _lib.SaeError("sae_b200 kernels need contiguous NHWC storage")


def _need_int64(t):
    """the 64-bit integer counters of the non-finite guard (unsigned long long in the C ABI)"""
    if not t.is_cuda or t.dtype != torch.int64 or not t.is_contiguous():
        raise _lib.SaeError("non-finite guard counters must be contiguous int64 CUDA tensors")


def _need_fp64(*ts):
    """the fp64 accumulators of the training statistics (None: an optional argument left out)"""
    for t in ts:
        if t is not None and (not t.is_cuda or t.dtype != torch.float64 or not t.is_contiguous()):
            raise _lib.SaeError("training-statistics accumulators must be contiguous fp64 CUDA tensors")


class PointerTables:
    """Device copies of host address lists (tuples of ``data_ptr()``), cached by content.  The pinned staging rows are
    allocated up front — a miss costs a device allocation and an async copy, so a miss inside a CUDA-graph capture is legal:
    the copy becomes a memcpy node that re-reads its pinned row on every replay.  Rows filled during a capture are therefore
    permanent; rows filled in eager execution (where the caching allocator may hand the gradients new addresses now and
    then) are recycled round-robin, each guarded by an event so a row is never rewritten before its copy has run."""

    def __init__(self, n, device, eager_rows=24, capture_rows=24):
        self.n, self.device = n, device
        self.eager_rows, self.capture_rows = eager_rows, capture_rows
        cuda = device.type == "cuda"
        self.pinned = torch.zeros(eager_rows + capture_rows, max(n, 1), dtype=torch.int64).pin_memory() if cuda else None
        self.eager, self.captured = {}, {}
        self.row_key, self.row_event = [None] * eager_rows, [None] * eager_rows
        self.next_row, self.next_capture = 0, 0

    def _upload(self, row, key):
        row[:len(key)].copy_(torch.tensor(key, dtype=torch.int64))
        dev = torch.empty(len(key), dtype=torch.int64, device=self.device)
        dev.copy_(row[:len(key)], non_blocking=True)
        return dev

    def get(self, key):
        hit = self.captured.get(key)
        if hit is None:
            hit = self.eager.get(key)
        if hit is not None:
            return hit
        if self.pinned is None:
            hit = torch.tensor(key, dtype=torch.int64)
            self.eager[key] = hit
            return hit
        if torch.cuda.is_current_stream_capturing():
            if self.next_capture >= self.capture_rows:
                raise _lib.SaeError("PointerTables: more than %d address lists captured into CUDA graphs" % self.capture_rows)
            hit = self._upload(self.pinned[self.eager_rows + self.next_capture], key)
            self.next_capture += 1
            self.captured[key] = hit
            return hit
        r = self.next_row
        self.next_row = (r + 1) % self.eager_rows
        if self.row_key[r] is not None:
            self.eager.pop(self.row_key[r], None)
            self.row_event[r].synchronize()
        hit = self._upload(self.pinned[r], key)
        ev = torch.cuda.Event()
        ev.record()
        self.row_key[r], self.row_event[r] = key, ev
        self.eager[key] = hit
        return hit


class CudaKernels:
    """The product path: every method is one (or two) launches of hand-written sm_90a kernels."""
    name = "cuda"

    def __init__(self):
        self.lib = _lib.load()
        self.conv_impl = 0       # 0 auto, 1 force generic (mma.sync), 2 force wgmma
        # Every activation / gradient / filter this library writes is rounded to the nearest TF32 value (still stored
        # as fp32): the tensor cores ignore the low 13 mantissa bits of their operands, so rounding in the producer
        # makes that truncation exact and unbiased.  Set False for bit-exact fp32 results from the pointwise kernels
        # (the convolutions stay TF32; precision = "fp32" below gives fp32-accurate convolutions).
        self.round_tf32 = True
        self.fused_fir_act = os.environ.get("SAE_FUSED_FIR_ACT", "1") != "0"
        # activation bit masks next to the tensor-core convs' / the FIR + activation kernel's outputs (A/B: SAE_ACT_MASK=0)
        self.act_masks = os.environ.get("SAE_ACT_MASK", "1") != "0"
        # "tf32" (default): convolutions and linears consume TF32 operands.  "fp32": they run the split-TF32 (3xTF32) kernels,
        # fp32-accurate products at about a third of the TF32 tensor-core rate, and nothing is rounded to TF32 on storage
        # (every round_tf32 argument is 0).  The torch flags (cudnn.allow_tf32, matmul.allow_tf32) are not consulted.
        self.precision = os.environ.get("SAE_PRECISION")
        # Deterministic mode: every gradient reduction runs through the _det twin of its entry point, which adds the CTAs'
        # partial sums in a fixed order instead of with fp32 atomics, so training steps are bitwise reproducible (run to run,
        # eager against CUDA-graph replay, on any H100).  torch.use_deterministic_algorithms(True) turns it on as well: see
        # deterministic_mode().
        self.deterministic = parse_deterministic(os.environ.get("SAE_DETERMINISTIC"))

    @property
    def precision(self):
        return self._precision

    @precision.setter
    def precision(self, value):
        self._precision = parse_precision(value)

    def deterministic_mode(self):
        """the effective mode: this object's flag or torch.use_deterministic_algorithms"""
        return bool(self.deterministic) or torch.are_deterministic_algorithms_enabled()

    def _launch(self, device, name, *args, refusable=False):
        """``name(*args, stream)`` on ``device`` and its current stream, raising SaeError on a failure code.  In deterministic
        mode an entry point with a _det twin runs the twin instead: a size query, then the call with a workspace from the
        caching allocator (stream-ordered: the memory is reused only by work queued after this call).  refusable: the
        wrapper handles SAE_E_UNSUPPORTED (a shape the kernel does not take), which is returned instead of raised."""
        with torch.cuda.device(device):
            if self.deterministic_mode() and name + "_det" in _lib.DET_ENTRY_POINTS:
                fn = getattr(self.lib, name + "_det")
                size = ctypes.c_int64(0)
                rc = fn(*args, None, ctypes.byref(size), None)
                if rc == 0:
                    ws = torch.empty(max(size.value, 1), dtype=torch.uint8, device=device)
                    rc = fn(*args, _ptr(ws), ctypes.byref(size), _stream())
            else:
                rc = getattr(self.lib, name)(*args, _stream())
        if not (refusable and rc == _lib.SAE_E_UNSUPPORTED):
            check(rc, name)
        return rc

    def _conv(self, device, name, *args, filt=None):
        """``_launch`` of a convolution entry point; ``args[filt]``: its filter, a tensor.  In fp32 mode the split-TF32 twin
        (``name + "_3xtf32"``) runs instead, and the filter travels as the pair (hi, lo) = split_tf32(filter)."""
        args = list(args)
        if self._precision == "fp32":
            name += "_3xtf32"
            if filt is not None:
                hi, lo = self.split_tf32(args[filt])
                args[filt:filt + 1] = _ptr(hi), _ptr(lo)
        elif filt is not None:
            args[filt] = _ptr(args[filt])
        self._launch(device, name, *args)

    def _round(self, flag=None):
        """the round_tf32 argument of a kernel call: the policy flag (or an explicit per-call value), always 0 in fp32 mode"""
        if self._precision == "fp32":
            return 0
        return int(self.round_tf32 if flag is None else flag)

    def split_tf32(self, w):
        """(hi, lo) = (rna_tf32(w), rna_tf32(w - hi)): the filter pair of the split-TF32 conv entry points"""
        w = w.contiguous()
        hi, lo = torch.empty_like(w), torch.empty_like(w)
        self._launch(w.device, "sae_split_tf32", _ptr(w), _ptr(hi), _ptr(lo), w.numel())
        return hi, lo

    # ------------------------------------------------------------------ FIR
    def upfirdn2d(self, x, kernel, up_x, up_y, down_x, down_y, pad_x0, pad_x1, pad_y0, pad_y1, taps=None, round_tf32=None):
        """taps: optional host-side 1-D factors (taps_y, taps_x) with kernel == outer(taps_y, taps_x); supplied by
        the Blur modules, which build their kernels from 1-D tap lists — selects the separable fast path wherever that
        kernel takes the shape.  round_tf32: override of the rounding policy (the augmentation passes False)."""
        _need_cuda(x, kernel)
        n, h, w, c = x.shape
        kh, kw = kernel.shape
        oh = (h * up_y + pad_y0 + pad_y1 - kh) // down_y + 1
        ow = (w * up_x + pad_x0 + pad_x1 - kw) // down_x + 1
        out = torch.empty((n, oh, ow, c), device=x.device, dtype=x.dtype)
        pads = (pad_x0, pad_x1, pad_y0, pad_y1)
        if taps is not None and up_x == up_y and down_x == down_y and (len(taps[0]), len(taps[1])) == (kh, kw):
            if self._launch(x.device, "sae_upfirdn2d_separable", _ptr(x), _floats(taps[0]), _floats(taps[1]), _ptr(out), n, h, w,
                            c, kh, kw, up_x, down_x, *pads, self._round(round_tf32), refusable=True) != _lib.SAE_E_UNSUPPORTED:
                return out
        self._launch(x.device, "sae_upfirdn2d", _ptr(x), _ptr(kernel), _ptr(out), n, h, w, c, kh, kw, up_x, up_y, down_x, down_y,
                     *pads, self._round(round_tf32))
        return out

    # ------------------------------------------------------------- bias/act
    def bias_act(self, x, bias, ref, act, grad, alpha, scale, noise=None, noise_weight=None):
        """x: [..., C] channels innermost.  noise: one value per pixel (numel = x.numel() / C)."""
        _need_cuda(x, bias, ref, noise, noise_weight)
        out = torch.empty_like(x)
        c = x.shape[-1]
        self._launch(x.device, "sae_fused_bias_act", _ptr(x), _ptr(bias), _ptr(ref), _ptr(out), x.numel(), 1,
                     bias.numel() if bias is not None else 1, act, grad, alpha, scale, _ptr(noise), _ptr(noise_weight), c,
                     self._round())
        return out

    def bias_act_backward(self, grad_out, out, alpha, scale, want_bias=True, noise=None, mask=None):
        """mask: the activation bit mask a forward kernel wrote for ``out`` (``act_mask_of(out)``) — read instead of ``out``"""
        _need_cuda(grad_out, out, noise)
        c = out.shape[-1]
        gi = torch.empty_like(out)
        gb = torch.zeros(c, device=out.device, dtype=out.dtype) if want_bias else None
        gnw = torch.zeros(1, device=out.device, dtype=out.dtype) if noise is not None else None
        self._launch(out.device, "sae_bias_act_backward", _ptr(grad_out), _ptr(out), _ptr(gi), _ptr(gb), out.numel(), c, alpha,
                     scale, _ptr(noise), c, _ptr(gnw), self._round(), _ptr(mask))
        return gi, gb, gnw

    def fir_act_backward(self, grad, taps, act_out, pad, alpha, scale, want_bias=True, mask=None):
        """(FIR(grad) masked by the activation saved in ``act_out``, bias gradient) in one pass, or None when the shape is
        outside the fused kernel's configuration (the caller then runs upfirdn2d + bias_act_backward).
        grad [N,h,w,C]; act_out [N,oh,ow,C]; taps = (taps_y, taps_x) host factors; pad = (x0, x1, y0, y1)."""
        _need_cuda(grad, act_out)
        n, h, w, c = grad.shape
        kh, kw = len(taps[0]), len(taps[1])
        px0, px1, py0, py1 = pad
        oh, ow = h + py0 + py1 - kh + 1, w + px0 + px1 - kw + 1
        # the deterministic twin also takes outputs under 8 x 8, which the fused kernel refuses: those stay on the two-launch
        # path in both modes
        if tuple(act_out.shape) != (n, oh, ow, c) or oh < 8 or ow < 8 or not self.fused_fir_act:
            return None
        gi = torch.empty_like(act_out)
        gb = torch.zeros(c, device=grad.device, dtype=grad.dtype) if want_bias else None
        if self._launch(grad.device, "sae_fir_act_backward", _ptr(grad), _floats(taps[0]), _floats(taps[1]), _ptr(act_out),
                        _ptr(gi), _ptr(gb), n, h, w, c, kh, kw, px0, px1, py0, py1, alpha, scale, self._round(), _ptr(mask),
                        refusable=True) == _lib.SAE_E_UNSUPPORTED:
            return None
        return gi, gb

    def fir_bias_act(self, x, taps, pad, bias, noise, noise_weight, alpha, scale):
        """lrelu(FIR(x) + noise_weight * noise + bias) * scale in one pass, or None when the shape is outside the fused kernel's
        configuration (the caller then runs upfirdn2d + bias_act).  x [N,h,w,C]; taps = (taps_y, taps_x) host factors;
        pad = (x0, x1, y0, y1); noise: one value per output pixel or None."""
        _need_cuda(x, bias, noise, noise_weight)
        n, h, w, c = x.shape
        kh, kw = len(taps[0]), len(taps[1])
        px0, px1, py0, py1 = pad
        out = torch.empty((n, h + py0 + py1 - kh + 1, w + px0 + px1 - kw + 1, c), device=x.device, dtype=x.dtype)
        mask = self._new_act_mask(out, 3, True)
        if self._launch(x.device, "sae_fir_bias_act", _ptr(x), _floats(taps[0]), _floats(taps[1]), _ptr(bias), _ptr(noise),
                        _ptr(noise_weight), _ptr(out), n, h, w, c, kh, kw, px0, px1, py0, py1, alpha, scale, self._round(),
                        _ptr(mask), refusable=True) == _lib.SAE_E_UNSUPPORTED:
            return None
        if mask is not None:
            out._sae_act_mask = mask
        return out

    # ------------------------------------------------------------- modulate
    def modulate(self, x, s):
        _need_cuda(x, s)
        n, h, w, c = x.shape
        out = torch.empty_like(x)
        self._launch(x.device, "sae_modulate", _ptr(x), _ptr(s), _ptr(out), n, h * w, c, self._round())
        return out

    def modulate_backward(self, dy, x, s):
        _need_cuda(dy, x, s)
        n, h, w, c = x.shape
        dx = torch.empty_like(x)
        ds = torch.zeros_like(s)
        self._launch(x.device, "sae_modulate_backward", _ptr(dy), _ptr(x), _ptr(s), _ptr(dx), _ptr(ds), n, h * w, c, self._round())
        return dx, ds

    # ------------------------------------------------------- residual merge
    def add_scale(self, a, b, scale):
        """(a + b) * scale, or a * scale when b is None; any shape, a and b contiguous with identical layout"""
        _need_cuda(a, b)
        out = torch.empty_like(a)
        self._launch(a.device, "sae_add_scale", _ptr(a), _ptr(b), _ptr(out), a.numel(), scale, self._round())
        return out

    def upsample2x_add_scale(self, skip, res, scale):
        """(bilinear_x2(skip) + res) * scale;  skip [N,h,w,C], res [N,2h,2w,C]"""
        _need_cuda(skip, res)
        n, h, w, c = skip.shape
        assert tuple(res.shape) == (n, 2 * h, 2 * w, c)
        out = torch.empty_like(res)
        self._launch(res.device, "sae_upsample2x_add_scale", _ptr(skip), _ptr(res), _ptr(out), n, h, w, c, scale, self._round())
        return out

    def upsample2x_backward(self, dy, scale):
        """adjoint of the x2 bilinear interpolation times scale: dy [N,2h,2w,C] -> [N,h,w,C]"""
        _need_cuda(dy)
        n, oh, ow, c = dy.shape
        out = torch.empty((n, oh // 2, ow // 2, c), device=dy.device, dtype=dy.dtype)
        self._launch(dy.device, "sae_upsample2x_backward", _ptr(dy), _ptr(out), n, oh // 2, ow // 2, c, scale, self._round())
        return out

    def pad_channels(self, x, c_out):
        """x: logical [N, c_in, H, W] with any (n, c) strides and a flattenable pixel plane -> NHWC [N, H, W, c_out],
        channels c_in.. zero (one kernel instead of F.pad + a layout copy)"""
        _need_cuda(x, strided=True)          # the kernel addresses x through (n, c, pixel) element strides
        n, c, h, w = x.shape
        if h > 1 and x.stride(2) != w * x.stride(3):
            x = x.contiguous()
        out = torch.empty((n, h, w, c_out), device=x.device, dtype=x.dtype)
        self._launch(x.device, "sae_pad_channels", _ptr(x), _ptr(out), n, h * w, c, c_out, x.stride(0), x.stride(1), x.stride(3),
                     self._round())
        return out

    def reflect_pad(self, x, pads):
        """x [N,H,W,C] -> [N, H+pt+pb, W+pl+pr, C]; pads = (left, right, top, bottom)"""
        _need_cuda(x)
        n, h, w, c = x.shape
        pl, pr, pt, pb = pads
        out = torch.empty((n, h + pt + pb, w + pl + pr, c), device=x.device, dtype=x.dtype)
        self._launch(x.device, "sae_reflect_pad", _ptr(x), _ptr(out), n, h, w, c, pl, pr, pt, pb)
        return out

    def reflect_pad_backward(self, dy, pads):
        _need_cuda(dy)
        n, oh, ow, c = dy.shape
        pl, pr, pt, pb = pads
        dx = torch.empty((n, oh - pt - pb, ow - pl - pr, c), device=dy.device, dtype=dy.dtype)
        self._launch(dy.device, "sae_reflect_pad_backward", _ptr(dy), _ptr(dx), n, oh - pt - pb, ow - pl - pr, c, pl, pr, pt, pb)
        return dx

    def filter_prep(self, w_oihw, scale, want_crsk=True):
        """[K,C,R,S] parameter -> ([K,R,S,C], [C,R,S,K] or None), scaled and TF32-rounded, in one kernel"""
        _need_cuda(w_oihw)
        k, c, r, s = w_oihw.shape
        krsc = torch.empty((k, r, s, c), device=w_oihw.device, dtype=w_oihw.dtype)
        crsk = torch.empty((c, r, s, k), device=w_oihw.device, dtype=w_oihw.dtype) if want_crsk else None
        self._launch(w_oihw.device, "sae_filter_prep", _ptr(w_oihw), _ptr(krsc), _ptr(crsk), k, c, r, s, scale, self._round())
        return krsc, crsk

    def filter_unprep(self, d_krsc, scale):
        """adjoint of filter_prep: [K,R,S,C] gradient -> [K,C,R,S] * scale"""
        _need_cuda(d_krsc)
        k, r, s, c = d_krsc.shape
        out = torch.empty((k, c, r, s), device=d_krsc.device, dtype=d_krsc.dtype)
        self._launch(d_krsc.device, "sae_filter_unprep", _ptr(d_krsc), _ptr(out), k, c, r, s, scale)
        return out

    def _filter(self, w):
        """contiguous copy of a (small) filter tensor, rounded to TF32 when the policy says so"""
        w = w.contiguous()
        if not self._round():
            return w
        out = torch.empty_like(w)
        self._launch(w.device, "sae_round_tf32", _ptr(w), _ptr(out), w.numel())
        return out

    # ----------------------------------------------------------------- conv
    def _new_act_mask(self, y, act, tensor_core_kernel):
        """1 bit per element of an activation output ``y`` [..., C] (C % 32 == 0), written by the kernel that produces y and read
        by the activation's backward instead of y itself (sae_conv_epilogue.act_mask); None where no kernel would write it"""
        if act != 3 or not tensor_core_kernel or not self.act_masks or y.shape[-1] % 32 != 0 or y.numel() == 0:
            return None
        return torch.empty(y.numel() // 32, device=y.device, dtype=torch.int32)

    def _epi(self, bias=None, act=1, alpha=0.2, gain=1.0, noise=None, noise_weight=None, residual=None,
             res_scale=1.0, round_tf32=None, act_mask=None):
        _need_cuda(bias, noise, noise_weight, residual)
        e = ConvEpilogue()
        e.bias = bias.data_ptr() if bias is not None else None
        e.noise = noise.data_ptr() if noise is not None else None
        e.noise_weight = noise_weight.data_ptr() if noise_weight is not None else None
        e.residual = residual.data_ptr() if residual is not None else None
        e.alpha, e.gain, e.res_scale, e.act = alpha, gain, res_scale, act
        e.round_tf32 = self._round(round_tf32)
        e.act_mask = act_mask.data_ptr() if act_mask is not None else None
        return e

    def conv_fprop(self, x, w_krsc, g, impl=None, prepared=False, **epi):
        """x [N,H,W,C], w [K,R,S,C] -> y [N,P,Q,K].  prepared: w is already contiguous and TF32-rounded (filter_prep)"""
        _need_cuda(x, w_krsc if prepared else None)
        if not prepared:
            w_krsc = self._filter(w_krsc)
        assert tuple(x.shape) == (g.N, g.H, g.W, g.C) and tuple(w_krsc.shape) == (g.K, g.R, g.S, g.C), \
            (tuple(x.shape), tuple(w_krsc.shape), g.key())
        y = torch.empty((g.N, g.P, g.Q, g.K), device=x.device, dtype=x.dtype)
        impl = self.conv_impl if impl is None else impl
        mask = None
        if epi.get("act", 1) == 3 and self.act_masks:
            mask = self._new_act_mask(y, 3, impl == 2 or (impl == 0 and self.conv_impl_for(g, 0) == 2))
        e = self._epi(act_mask=mask, **epi)
        self._conv(x.device, "sae_conv2d_fprop", _ptr(x), w_krsc, _ptr(y), ctypes.byref(g), ctypes.byref(e), impl, filt=1)
        if mask is not None:
            y._sae_act_mask = mask
        return y

    def conv_dgrad(self, dy, w_krsc, g, impl=None, w_crsk=None, **epi):
        """dy [N,P,Q,K], w [K,R,S,C] -> dx [N,H,W,C] (also the forward of the transposed convolution).
        w_crsk: the same filter already transposed to [C,R,S,K] and rounded (filter_prep), if the caller has it."""
        _need_cuda(dy)
        assert tuple(dy.shape) == (g.N, g.P, g.Q, g.K) and tuple(w_krsc.shape) == (g.K, g.R, g.S, g.C), \
            (tuple(dy.shape), tuple(w_krsc.shape), g.key())
        wt = w_crsk if w_crsk is not None else self._filter(w_krsc.permute(3, 1, 2, 0))     # [C,R,S,K]
        dx = torch.empty((g.N, g.H, g.W, g.C), device=dy.device, dtype=dy.dtype)
        e = self._epi(**epi)
        impl = self.conv_impl if impl is None else impl
        self._conv(dy.device, "sae_conv2d_dgrad", _ptr(dy), wt, _ptr(dx), ctypes.byref(g), ctypes.byref(e), impl, filt=1)
        return dx

    def conv_wgrad(self, dy, x, g, impl=None):
        """dy [N,P,Q,K], x [N,H,W,C] -> dw [K,R,S,C]"""
        _need_cuda(dy, x)
        assert tuple(dy.shape) == (g.N, g.P, g.Q, g.K) and tuple(x.shape) == (g.N, g.H, g.W, g.C), \
            (tuple(dy.shape), tuple(x.shape), g.key())
        dw = torch.zeros((g.K, g.R, g.S, g.C), device=dy.device, dtype=dy.dtype)
        self._conv(dy.device, "sae_conv2d_wgrad", _ptr(dy), _ptr(x), _ptr(dw), ctypes.byref(g),
                   self.conv_impl if impl is None else impl)
        return dw

    # ------------------------------------------------ style-modulated conv, per-sample filters
    def conv_modulated_ok(self, g):
        """True when the per-sample-filter kernels (fprop, dgrad, modulated wgrad) all take this geometry"""
        return bool(self.lib.sae_conv2d_query_modulated(ctypes.byref(g)))

    def filter_modulate(self, w_krsc, s, want_krsc=True, want_crsk=False):
        """prepared filter [K,R,S,C] x per-sample scale [N,C] -> ([N,K,R,S,C] or None, [N,C,R,S,K] or None)"""
        _need_cuda(w_krsc, s)
        k, r, s_, c = w_krsc.shape
        n = s.shape[0]
        a = torch.empty((n, k, r, s_, c), device=s.device, dtype=s.dtype) if want_krsc else None
        b = torch.empty((n, c, r, s_, k), device=s.device, dtype=s.dtype) if want_crsk else None
        self._launch(s.device, "sae_filter_modulate", _ptr(w_krsc), _ptr(s), _ptr(a), _ptr(b), n, k, c, r, s_, self._round())
        return a, b

    def conv_fprop_per_sample(self, x, w_nkrsc, g, **epi):
        """x [N,H,W,C], per-sample filters [N,K,R,S,C] -> y [N,P,Q,K]"""
        _need_cuda(x, w_nkrsc)
        y = torch.empty((g.N, g.P, g.Q, g.K), device=x.device, dtype=x.dtype)
        mask = self._new_act_mask(y, epi.get("act", 1), True)          # only the wgmma kernel implements per-sample filters
        e = self._epi(act_mask=mask, **epi)
        self._conv(x.device, "sae_conv2d_fprop_per_sample", _ptr(x), w_nkrsc, _ptr(y), ctypes.byref(g), ctypes.byref(e), filt=1)
        if mask is not None:
            y._sae_act_mask = mask
        return y

    def conv_dgrad_per_sample(self, dy, w_ncrsk, g, **epi):
        """dy [N,P,Q,K], per-sample transposed filters [N,C,R,S,K] -> dx [N,H,W,C]"""
        _need_cuda(dy, w_ncrsk)
        dx = torch.empty((g.N, g.H, g.W, g.C), device=dy.device, dtype=dy.dtype)
        e = self._epi(**epi)
        self._conv(dy.device, "sae_conv2d_dgrad_per_sample", _ptr(dy), w_ncrsk, _ptr(dx), ctypes.byref(g), ctypes.byref(e), filt=1)
        return dx

    def conv_wgrad_modulated(self, dy, x, s, w_krsc, g):
        """dy [N,P,Q,K], UNSCALED x [N,H,W,C], s [N,C], forward filter [K,R,S,C] -> (dw [K,R,S,C], ds [N,C])"""
        _need_cuda(dy, x, s, w_krsc)
        dw = torch.zeros((g.K, g.R, g.S, g.C), device=dy.device, dtype=dy.dtype)
        ds = torch.zeros((g.N, g.C), device=dy.device, dtype=dy.dtype)
        self._conv(dy.device, "sae_conv2d_wgrad_modulated", _ptr(dy), _ptr(x), _ptr(s), _ptr(w_krsc), _ptr(dw), _ptr(ds),
                   ctypes.byref(g))
        return dw, ds

    def conv_impl_for(self, g, direction):
        return int(self.lib.sae_conv2d_query_impl(ctypes.byref(g), direction))

    # --------------------------------------------------------------- bucket
    def bucket_pack(self, ptrs, offsets, sizes, n, bucket):
        self._launch(bucket.device, "sae_bucket_pack", _ptr(ptrs), _ptr(offsets), _ptr(sizes), n, _ptr(bucket), bucket.numel())

    def bucket_unpack(self, ptrs, offsets, sizes, n, bucket, scale):
        self._launch(bucket.device, "sae_bucket_unpack", _ptr(ptrs), _ptr(offsets), _ptr(sizes), n, _ptr(bucket), bucket.numel(),
                     scale)

    def bucket_accumulate(self, ptrs, offsets, sizes, n, bucket):
        """bucket[offsets[t] + i] += tensor t of the pointer table ``ptrs`` (the layout of ``bucket_pack``; NULL: skipped)"""
        self._launch(bucket.device, "sae_bucket_accumulate", _ptr(ptrs), _ptr(offsets), _ptr(sizes), n, _ptr(bucket),
                     bucket.numel())


    # ----------------------------------------------------------------- Adam
    def adam_step(self, params, grads, offsets, sizes, exp_avg, exp_avg_sq, steps, lr, beta1, beta2, eps, grad_scale, cache,
                  skip=None):
        """One multi-tensor Adam update (torch.optim.Adam semantics) of ``params`` (list of tensors).  grads: list aligned with
        params — a tensor (the parameter's own gradient, or a view into the flat all-reduce bucket) or None (parameter
        skipped, its step count untouched).  offsets / sizes: device int64 tensors locating each parameter's moments in
        the flat ``exp_avg`` / ``exp_avg_sq``; steps: device float tensor, one count per parameter.  cache: the caller's
        ``PointerTables`` (device copies of the address lists).  skip: optional one-element device int64 tensor (the total of
        ``nonfinite_count``); the kernels drop the whole update when it is non-zero (sae_adam_step_guarded)."""
        p_tab = cache.get(tuple(p.data_ptr() for p in params))
        g_tab = cache.get(tuple(0 if g is None else g.data_ptr() for g in grads))
        for g in grads:
            if g is not None and (not g.is_cuda or g.dtype != torch.float32 or not g.is_contiguous()):
                raise _lib.SaeError("adam_step: gradients must be contiguous fp32 CUDA tensors")
        args = (_ptr(p_tab), _ptr(g_tab), _ptr(offsets), _ptr(sizes), len(params), _ptr(exp_avg), _ptr(exp_avg_sq), _ptr(steps), lr,
                beta1, beta2, eps, grad_scale)
        if skip is None:
            self._launch(exp_avg.device, "sae_adam_step", *args)
        else:
            _need_int64(skip)
            self._launch(exp_avg.device, "sae_adam_step_guarded", *args, _ptr(skip))

    def nonfinite_count(self, tensors, sizes, counts, cache):
        """counts[i] += number of NaN / +-Inf elements of tensors[i] (None: skipped), counts[n] += their sum; one launch.
        tensors: contiguous fp32 CUDA tensors; sizes: device int64 tensor of their element counts (the parameters' sizes);
        counts: device int64 tensor of n + 1 entries, zero-filled by the caller; cache: ``PointerTables``."""
        _need_int64(counts)
        for t in tensors:
            _need_cuda(t)
        if counts.numel() != len(tensors) + 1 or sizes.numel() != len(tensors):
            raise _lib.SaeError("nonfinite_count: counts needs n + 1 entries and sizes n")
        tab = cache.get(tuple(0 if t is None else t.data_ptr() for t in tensors))
        self._launch(counts.device, "sae_nonfinite_count", _ptr(tab), _ptr(sizes), len(tensors), _ptr(counts))

    def ema_update(self, params, offsets, sizes, shadow, updates, batch_images, half_life_images, rampup, cache, skip=None):
        """One averaging update of the flat ``shadow`` towards ``params`` (sae_ema_update; INTEGRATION §2f), then
        ``updates += 1``.  offsets / sizes: device int64 tensors locating each parameter's segment of ``shadow`` (the layout of
        ``adam_step``'s moments); updates: one-element device int64 tensor, the averaging updates already made, from which the
        kernel forms beta; cache: the caller's ``PointerTables``.  skip: optional one-element device int64 tensor; a non-zero
        value leaves shadow and updates unchanged."""
        _need_cuda(shadow, *params)
        _need_int64(updates)
        if skip is not None:
            _need_int64(skip)
        p_tab = cache.get(tuple(p.data_ptr() for p in params))
        self._launch(shadow.device, "sae_ema_update", _ptr(p_tab), _ptr(offsets), _ptr(sizes), len(params), _ptr(shadow),
                     shadow.numel(), _ptr(updates), float(batch_images), float(half_life_images), float(rampup), _ptr(skip))

    # ----------------------------------------------------------------- training statistics (INTEGRATION §2g)
    def sumsq(self, tensors, sizes, out, partials, cache, scale=1.0, skip=None):
        """out[i] += scale^2 * sum of squares of tensors[i] (None: skipped), in fp64 (sae_sumsq).  tensors: contiguous fp32 CUDA
        tensors; sizes: device int64 tensor of their element counts; out: device fp64 tensor of n entries; partials: device
        fp64 workspace of at least n * _lib.SAE_STATS_BLOCKS entries; cache: ``PointerTables``.  skip: optional one-element
        device int64 tensor; a non-zero value adds nothing."""
        for t in tensors:
            _need_cuda(t)
        _need_fp64(out, partials)
        if skip is not None:
            _need_int64(skip)
        if out.numel() < len(tensors) or partials.numel() < len(tensors) * _lib.SAE_STATS_BLOCKS:
            raise _lib.SaeError("sumsq: out needs n entries and partials n * SAE_STATS_BLOCKS")
        tab = cache.get(tuple(0 if t is None else t.data_ptr() for t in tensors))
        self._launch(out.device, "sae_sumsq", _ptr(tab), _ptr(sizes), len(tensors), float(scale), _ptr(out), _ptr(partials),
                     _ptr(skip))

    def adam_norms(self, params, grads, offsets, sizes, exp_avg, exp_avg_sq, steps, lr, beta1, beta2, eps, weight_out,
                   update_out, updates, partials, cache, skip=None):
        """After ``adam_step`` with the same arguments: weight_out[i] += |params[i]|^2 and update_out[i] += |Adam's step|^2
        (0 where grads[i] is None), the step recomputed from the moments and step counts; updates += 1 (sae_adam_norms).
        weight_out / update_out: device fp64 tensors of n entries; updates: one-element device fp64 tensor or None; partials:
        device fp64 workspace of at least 2 * n * _lib.SAE_STATS_BLOCKS entries.  skip: as for ``adam_step``; a non-zero value
        adds nothing, to the counter included."""
        _need_cuda(exp_avg, exp_avg_sq, steps, *params)
        _need_fp64(weight_out, update_out, updates, partials)
        if skip is not None:
            _need_int64(skip)
        n = len(params)
        if weight_out.numel() < n or update_out.numel() < n or partials.numel() < 2 * n * _lib.SAE_STATS_BLOCKS:
            raise _lib.SaeError("adam_norms: outputs need n entries and partials 2 * n * SAE_STATS_BLOCKS")
        p_tab = cache.get(tuple(p.data_ptr() for p in params))
        g_tab = cache.get(tuple(0 if g is None else g.data_ptr() for g in grads))
        self._launch(exp_avg.device, "sae_adam_norms", _ptr(p_tab), _ptr(g_tab), _ptr(offsets), _ptr(sizes), n, _ptr(exp_avg),
                     _ptr(exp_avg_sq), _ptr(steps), float(lr), float(beta1), float(beta2), float(eps), _ptr(weight_out),
                     _ptr(update_out), _ptr(updates), _ptr(partials), _ptr(skip))

    def score_stats(self, x, acc):
        """acc[0:4] += (sum, sum of signs, count) of the finite elements of x and the count of its NaN / +-Inf elements
        (sae_score_stats).  x: fp32 CUDA tensor of 1 to 4 dimensions, any non-negative strides; acc: device fp64 tensor."""
        _need_cuda(x, strided=True)
        _need_fp64(acc)
        if acc.numel() < 4 or not 1 <= x.dim() <= 4:
            raise _lib.SaeError("score_stats: needs a 1- to 4-dimensional tensor and 4 accumulators")
        shape = (ctypes.c_int64 * x.dim())(*x.shape)
        strides = (ctypes.c_int64 * x.dim())(*x.stride())
        self._launch(acc.device, "sae_score_stats", _ptr(x), x.dim(), shape, strides, _ptr(acc))

    # ----------------------------------------------------------------- augmentation (INTEGRATION §2h)
    def augment_params(self, u, z, p, h, w):
        """per-image records [N, SAE_AUG_RECORD] (G_inv, then C) from the draws u [N, SAE_AUG_UNIFORMS], z [N, SAE_AUG_NORMALS]
        and the one-element device probability p, for images of h x w (sae_augment_params)"""
        _need_cuda(u, z, p)
        n = u.shape[0]
        if tuple(u.shape) != (n, _lib.SAE_AUG_UNIFORMS) or tuple(z.shape) != (n, _lib.SAE_AUG_NORMALS):
            raise _lib.SaeError("augment_params: draws must be [N, %d] and [N, %d]" % (_lib.SAE_AUG_UNIFORMS, _lib.SAE_AUG_NORMALS))
        rec = torch.empty((n, _lib.SAE_AUG_RECORD), device=u.device, dtype=u.dtype)
        self._launch(u.device, "sae_augment_params", _ptr(u), _ptr(z), _ptr(p), _ptr(rec), n, h, w)
        return rec

    def _need_rec(self, rec, n):
        _need_cuda(rec)
        if tuple(rec.shape) != (n, _lib.SAE_AUG_RECORD):
            raise _lib.SaeError("augmentation records must be [N, %d]" % _lib.SAE_AUG_RECORD)

    def augment_sample(self, x, rec, copy_identity=True):
        """x: logical [N, 3, H, W] (any strides) -> NHWC [N, 2(H + 6), 2(W + 6), 4] (channel 3 zero): the transformed sample
        grid of the reflect-padded, 2x upsampled image (sae_augment_sample)"""
        _need_cuda(x, strided=True)
        n, c, h, w = x.shape
        if c != 3:
            raise _lib.SaeError("augment_sample: images must have 3 channels")
        self._need_rec(rec, n)
        s = torch.empty((n, 2 * (h + 6), 2 * (w + 6), 4), device=x.device, dtype=x.dtype)
        self._launch(x.device, "sae_augment_sample", _ptr(x), _ptr(rec), _ptr(s), n, h, w, *x.stride(), int(copy_identity))
        return s

    def augment_sample_adjoint(self, ds, gc, rec, h, w, copy_identity=True):
        """adjoint of ``augment_sample``: ds NHWC [N, 2(h + 6), 2(w + 6), 4] -> NHWC [N, h, w, 3]; an image whose G_inv is I
        copies channels 0..2 of gc NHWC [N, h, w, 4] instead (copy_identity)"""
        _need_cuda(ds, gc)
        n = ds.shape[0]
        if tuple(ds.shape) != (n, 2 * (h + 6), 2 * (w + 6), 4) or (gc is not None and tuple(gc.shape) != (n, h, w, 4)):
            raise _lib.SaeError("augment_sample_adjoint: shape mismatch")
        self._need_rec(rec, n)
        dx = torch.empty((n, h, w, 3), device=ds.device, dtype=ds.dtype)
        self._launch(ds.device, "sae_augment_sample_adjoint", _ptr(ds), _ptr(gc), _ptr(rec), _ptr(dx), n, h, w, int(copy_identity))
        return dx

    def augment_color(self, a, b, rec, offset=True, copy_identity=True):
        """NHWC [N, H, W, 3] = C[:3, :3] v (+ C[:3, 3] with offset), v = a (logical [N, 3, H, W], any strides) for an image whose
        G_inv is I (copy_identity), else channels 0..2 of b (NHWC [N, H, W, 4]) (sae_augment_color)"""
        _need_cuda(a, strided=True)
        _need_cuda(b)
        n, h, w, c = b.shape
        if c != 4 or tuple(a.shape) != (n, 3, h, w):
            raise _lib.SaeError("augment_color: shape mismatch")
        self._need_rec(rec, n)
        out = torch.empty((n, h, w, 3), device=b.device, dtype=b.dtype)
        self._launch(b.device, "sae_augment_color", _ptr(a), _ptr(b), _ptr(rec), _ptr(out), n, h, w, *a.stride(), int(offset),
                     int(copy_identity))
        return out

    def augment_color_adjoint(self, dy, rec):
        """dy: logical [N, 3, H, W] (any strides) -> NHWC [N, H, W, 4] = C[:3, :3]^T dy, channel 3 zero
        (sae_augment_color_adjoint)"""
        _need_cuda(dy, strided=True)
        n, c, h, w = dy.shape
        if c != 3:
            raise _lib.SaeError("augment_color_adjoint: images must have 3 channels")
        self._need_rec(rec, n)
        gc = torch.empty((n, h, w, 4), device=dy.device, dtype=dy.dtype)
        self._launch(dy.device, "sae_augment_color_adjoint", _ptr(dy), _ptr(rec), _ptr(gc), n, h, w, *dy.stride())
        return gc

    def ada_adjust(self, p, acc, step, target):
        """p = max(0, p + (float)(sign(acc[1] / acc[2] - target) * step)) when acc[2] > 0, then acc = 0 (sae_ada_adjust).
        p: one-element fp32 device tensor; acc: the four fp64 sums of ``score_stats``"""
        _need_cuda(p)
        _need_fp64(acc)
        if p.numel() != 1 or acc.numel() != 4:
            raise _lib.SaeError("ada_adjust: p needs one element and acc four")
        self._launch(p.device, "sae_ada_adjust", _ptr(p), _ptr(acc), float(step), float(target))

    # ----------------------------------------------------------------- ToRGB
    def torgb_forward(self, x, s, w, bias, wscale):
        """x [N,H,W,C], s [N,C], w [3,C], bias [3] or None -> y [N,H,W,4] (channel 3 zero)"""
        _need_cuda(x, s, w, bias)
        n, h, wd, c = x.shape
        y = torch.empty((n, h, wd, 4), device=x.device, dtype=x.dtype)
        self._launch(x.device, "sae_torgb_forward", _ptr(x), _ptr(s), _ptr(w), _ptr(bias), _ptr(y), n, h, wd, c, wscale,
                     self._round())
        return y

    def torgb_backward(self, dy, x, s, w, wscale, want_dx=True, want_gw=True):
        """dy: logical [N,3,H,W] (any strides) -> (dx [N,H,W,C] or None, gw [N,3,C] = sum_p dy (x) x or None)"""
        _need_cuda(x, s, w)
        _need_cuda(dy, strided=True)
        n, h, wd, c = x.shape
        dx = torch.empty_like(x) if want_dx else None
        gw = torch.zeros((n, 3, c), device=x.device, dtype=x.dtype) if want_gw else None
        self._launch(x.device, "sae_torgb_backward", _ptr(dy), _ptr(x), _ptr(s), _ptr(w), _ptr(dx), _ptr(gw), n, h, wd, c, wscale,
                     dy.stride(0), dy.stride(1), dy.stride(2), dy.stride(3), self._round())
        return dx, gw

    # ----------------------------------------------------------------- crops
    def crop_gather(self, x, flip, scale, offset, num_crops, size, c_pad, out=None):
        """x: logical [B, C, H, W] (any strides); flip [Q], scale / offset [Q, 2] -> NHWC [Q, size, size, c_pad], channels
        C.. zero.  out: optional destination (a [Q, size, size, c_pad] slice of a larger batch buffer)"""
        _need_cuda(x, flip, scale, offset, strided=True)
        b, c, h, w = x.shape
        q = flip.numel()
        if out is None:
            out = torch.empty((q, size, size, c_pad), device=x.device, dtype=x.dtype)
        assert tuple(out.shape) == (q, size, size, c_pad) and out.is_contiguous()
        self._launch(x.device, "sae_crop_gather", _ptr(x), _ptr(flip), _ptr(scale), _ptr(offset), _ptr(out), q, num_crops, c, h, w,
                     size, c_pad, x.stride(0), x.stride(1), x.stride(2), x.stride(3), self._round())
        return out

    def crop_gather_backward(self, dy, flip, scale, offset, num_crops, c, h, w):
        """dy: logical [Q, C', S, S] (any strides, C' >= c) -> dx [Q / num_crops, c, h, w] contiguous"""
        _need_cuda(dy, flip, scale, offset, strided=True)
        q, s = dy.shape[0], dy.shape[2]
        dx = torch.empty((q // num_crops, c, h, w), device=dy.device, dtype=dy.dtype)
        self._launch(dy.device, "sae_crop_gather_backward", _ptr(dy), _ptr(flip), _ptr(scale), _ptr(offset), _ptr(dx), q, num_crops,
                     c, h, w, s, dy.stride(0), dy.stride(1), dy.stride(2), dy.stride(3))
        return dx



_kernels = None


def act_mask_of(t):
    """the activation bit mask the producing kernel left next to ``t`` (None: the backward reads ``t`` itself).  The mask is a
    Python attribute of the tensor object the kernel wrapper returned: callers that hand ``t`` to autograd (outputs of a
    Function come back as new objects) read it right after the forward call and keep it in their ctx."""
    return getattr(t, "_sae_act_mask", None) if t is not None else None


def kernels():
    """The active kernel set; instantiates ``CudaKernels`` (loading the .so) on first use."""
    global _kernels
    if _kernels is None:
        _kernels = CudaKernels()
    return _kernels


def set_kernels(k):
    """Test hook (tests/ only): install an object with the ``CudaKernels`` interface."""
    global _kernels
    prev = _kernels
    _kernels = k
    return prev
