"""GPU (H100): every parameter gradient of the D, R1 and G half-steps at the 256² default nets against fp64.

What Adam consumes is the gradient the hand-written autograd layer (the ``Function`` classes of ``stylegan2_op/`` and
``util.py``) hands back.  A wrong argument passed to a correct kernel — a gain, ``wscale``, a mask, a noise map — is invisible
to the per-kernel tests, so this file checks the product of the layer at network level: the trainer's own bodies
(``_discriminator_body`` / ``_r1_body`` / ``_generator_body`` with ``step=False``) against the oracle's fp64 gradient of the
same half-step (``OracleTrainer``'s definition: the sum of the loss means, times ``R1_once_every`` for R1), on the same seeded
parameters (``perturbed_state_dict``: non-zero biases, noise weights 0.05), images, crops and generator noise.

Comparison, per parameter tensor of the half-step's group, matched by ``state_dict`` key (a key missing on either side fails):
* where the fp64 gradient is exactly zero or absent (the R1 gradients of the biases), the product's must be too;
* otherwise relative L2, asserted against one bound per precision and half-step kind (DESIGN.md §2); max-norm relative error
  is recorded beside it.  The noise weights, whose gradients cancel, are judged against a natural scale (NATURAL_SCALE).
  Both go to the JSON file ``SAE_PARITY_RECORD`` names, one entry per (variant, half-step, tensor).

The coverage table ``BACKWARD_REACHED`` lists, for every ``Function`` subclass of the package, the variants whose half-steps
run its backward; the test wraps every ``backward`` and requires the table to be exactly what ran.  ``NOT_DIFFERENTIATED``
gives the reason for each one training never differentiates.  ``tests/test_gradient_function_table.py`` (CPU) fails when a
``Function`` has no row."""
import json
import os
import time

import pytest
import torch

from oracle import sae_oracle as O
from oracle.fixtures import perturbed_state_dict, rel_err, rel_l2, rnd
from tests.test_gpu_parity_full import _CropDraws

pytestmark = pytest.mark.gpu
DEV = "cuda"

OPTS_256 = dict(crop_size=256, batch_size=2)
# the ffhq1024 launcher's channel set at 256²: 409 / 204 / 102-channel generator layers take the _pad32 route
OPTS_FFHQ_256 = dict(crop_size=256, batch_size=2, netG_scale_capacity=0.8, netE_scale_capacity=0.4, global_code_ch=1536,
                     netE_num_downsampling_sp=5)
# crop draws of each half-step, per configuration: seeds whose fp64 truth passes the head-margin check below
CROP_SEED = {"256": {"D": 2, "R1": 3, "G": 2}, "ffhq": {"G": 10}}
# A leaky-ReLU mask bit is decided by the sign of a pre-activation; fp32 evaluation moves a pre-activation by ~1e-6 of its
# layer's RMS.  In the dense head layers (16 rows in Dpatch's pair linears, 2-6 in D's final linear) one flipped bit moves
# every upstream gradient of the network by ~1e-3, so the fp64 truth requires every head pre-activation to be at least
# HEAD_MARGIN x its layer's RMS away from zero.  The conv layers' flips are diluted over 10^5-10^6 elements each.
HEAD_MARGIN = 5e-6

# relative-L2 bounds per (precision, half-step kind), measured worst in DESIGN.md §2.  TF32: the documented spread of
# leaky-ReLU mask flips, which in TF32 mode also reach the 16-row head layers (no input margin decides a sign at TF32's
# 2^-11), and for the noise weights (judged at their natural scale, below) the spread of a sum of ~10^5 TF32-rounded terms.
# fp32 mode: one constant per kind, 2x / 5x the worst tensor measured on an H100.
TOL = {("tf32", "first"): 4e-2, ("tf32", "R1"): 2.5e-2, ("tf32", "noise"): 1e-1,
       ("fp32", "first"): 1.5e-3, ("fp32", "R1"): 5e-4, ("fp32", "noise"): 5e-3}

# variant -> (precision, deterministic, fused blocks, R1 through the general path, half-steps)
VARIANTS = {
    "tf32": ("tf32", False, True, False, ("D", "R1", "G")),
    "fp32": ("fp32", False, True, False, ("D", "R1", "G")),
    "fp32_det": ("fp32", True, True, False, ("D", "R1", "G")),
    "fp32_unfused": ("fp32", False, False, False, ("D", "R1")),
    "fp32_r1_general": ("fp32", False, False, True, ("R1",)),
    "fp32_r1_general_fused": ("fp32", False, True, True, ("R1",)),
}

# (half-step, key prefix or suffix) -> why that gradient is judged against its natural scale, max(||fp64||, scale), instead of
# its own norm.  Both figures are recorded for every tensor that has a natural scale.
NATURAL_SCALE = {
    ("G", ".noise.weight"): "a sum over every pixel of gradient x zero-mean noise, which cancels to 1/12-1/15 of the L2 norm "
                            "of the per-pixel terms at the 256² nets; scale: that L2 norm",
}


def _natural_scale_reason(kind, key):
    return next((why for (k, pattern), why in NATURAL_SCALE.items()
                 if k == kind and (key.startswith(pattern) or key.endswith(pattern))), None)


FFHQ = "fp32_ffhq_channels"

_ALL = tuple(VARIANTS) + (FFHQ,)
_WITH_R1 = tuple(VARIANTS)                 # every variant but the ffhq channel set runs an R1 half-step
_FIRST = ("tf32", "fp32", "fp32_det")      # the shipping path of all three half-steps
_GENERAL = ("fp32_unfused", "fp32_r1_general", "fp32_r1_general_fused")
# Function -> the variants whose half-steps run its backward
BACKWARD_REACHED = {
    "_PrepFilter": _ALL,
    "_UnprepFilter": (),
    "_ConvFprop": _ALL,
    "_ConvDgrad": _ALL,
    "_ConvWgrad": (),
    "_ConvBiasAct": _ALL,
    "_ConvNoiseBiasAct": _FIRST + (FFHQ,),
    "_ConvResidual": _ALL,                 # always with scale 1: the merge factor is folded into the gains and wscale
    "_PadChannels": _ALL,
    "_ViewAsPadded": _FIRST + (FFHQ,),
    "_Modulate": _FIRST + (FFHQ,),
    "_ModulatedConv": _FIRST,              # needs channel counts that are multiples of 32: not the ffhq set
    "_ToRGB": _FIRST,                      # the ffhq set's 102-channel ToRGB takes the general modulated conv
    "_AddScale": (FFHQ,),                  # the 409-channel head block's skip
    "_ReflectPad": _FIRST,                 # the ffhq set's encoder has channel counts that are not multiples of 4
    "_ReflectPadAdjoint": (),
    "_Upsample2xAddScale": _FIRST + (FFHQ,),
    "_FirNoiseBiasAct": _FIRST + (FFHQ,),
    "_ResBlockDataGrad": _FIRST,
    "_ResBlockFused": _FIRST + ("fp32_r1_general_fused", FFHQ),
    "FusedLeakyReLUFunctionBackward": _WITH_R1,
    "FusedLeakyReLUFunction": _ALL,
    "_NoiseBiasLeakyReLU": (FFHQ,),
    "UpFirDn2dBackward": _GENERAL,
    "UpFirDn2d": _ALL,
    "_CropGather": _FIRST + (FFHQ,),
    "_CropGatherMulti": (),
}
# Function -> why no training half-step runs its backward
NOT_DIFFERENTIATED = {
    "_UnprepFilter": "the backward of a weight gradient's filter layout change: no loss differentiates a weight gradient",
    "_ConvWgrad": "its output is a weight gradient, and no loss differentiates a weight gradient again",
    "_ReflectPadAdjoint": "the backward of the encoder's reflection-pad gradient: second order through E, never asked for",
    "_CropGatherMulti": "the batched D-step crops read real images and G's output while G is frozen: no input requires grad",
}


def _cuda(t):
    return t.detach().float().to(DEV)


def _noise_maps(copt, seed0=950):
    """the generator noise of one loss command: [rec call, mix call], each {"<block>.<conv>": [B,1,H,W]} with B the call's
    batch, so the product takes its fused per-image noise paths"""
    res = copt.crop_size // 2 ** copt.netE_num_downsampling_sp
    layers = [("HeadResnetBlock%d.conv%d" % (i, c), res) for i in range(copt.netG_num_base_resnet_layers) for c in (1, 2)]
    for j in range(copt.netE_num_downsampling_sp):
        layers += [("UpsamplingResBlock%d.conv%d" % (2 ** (4 + j), c), res * 2 ** (j + 1)) for c in (1, 2)]
    b = copt.batch_size
    return [{name: rnd(seed0 + 100 * call + i, n, 1, r, r) for i, (name, r) in enumerate(layers)}
            for call, n in enumerate((b // 2, b))]


def _norm(t):
    return float(t.norm()) if t is not None else 0.0


def _f32(t):
    return t.float().double()


def _kernel_coordinate_crops(x, opt, flip, scale, offset):
    """``O.random_crops`` sampled at the coordinates the crop kernel computes in fp32 (csrc/train_ops.cu, crop_gather_kernel:
    linspace, then one fused multiply-add per normalised coordinate, then the un-normalisation), so that both sides read
    the images at the same points.  The grid passed to grid_sample un-normalises to exactly those fp32 values (W, H are powers
    of two)."""
    n, S = opt.patch_num_crops, opt.patch_size
    B, H, W = x.size(0) * n, x.shape[2], x.shape[3]
    step = float(torch.tensor(2.0 / (S - 1)).float())
    k = torch.arange(S, dtype=torch.float64)
    lin = _f32(torch.where(k < S // 2, -1.0 + step * k, 1.0 - step * (S - 1 - k)))
    sx, sy, ox, oy = (t.reshape(B, 1, 1) for t in (scale[..., 0], scale[..., 1], offset[..., 0], offset[..., 1]))
    gx = _f32(lin.view(1, 1, S) * flip.reshape(B, 1, 1) * sx + ox).expand(B, S, S)
    gy = _f32(lin.view(1, S, 1) * sy + oy).expand(B, S, S)
    ix, iy = _f32(_f32(gx + 1) * W - 1) * 0.5, _f32(_f32(gy + 1) * H - 1) * 0.5
    grid = torch.stack([(2 * ix + 1) / W - 1, (2 * iy + 1) / H - 1], dim=3)
    crop = torch.nn.functional.grid_sample(x.unsqueeze(1).expand(-1, n, -1, -1, -1).flatten(0, 1), grid, align_corners=False)
    return crop.view(B // n, n, crop.size(1), S, S)


def _fp64_truth(copt, sd64, real, noises, kinds, crop_seed):
    """losses, the gradient of every parameter of the half-step's group keyed by state_dict key (None: unused), the natural
    scale of the gradients listed in NATURAL_SCALE, and the smallest head pre-activation relative to its layer's RMS"""
    m = O.OracleModel(copt, sd64)
    groups = {"generator": {"G": m.G, "E": m.E}, "discriminator": {"D": m.D, "Dpatch": m.Dp}}
    draws = _CropDraws()
    margins = []
    fused_leaky_relu = O.fused_leaky_relu

    def crops(x, opt):
        params = (_f32(t) for t in draws.draw(x.size(0) * opt.patch_num_crops, opt.patch_min_scale, opt.patch_max_scale))
        return _kernel_coordinate_crops(x, opt, *params)

    def head_margin_recorder(x, bias, negative_slope=0.2, scale=O.SQRT2):
        if x.dim() == 2:
            z = (x + bias if bias is not None else x).detach()
            margins.append(float(z.abs().min() / z.pow(2).mean().sqrt()))
        return fused_leaky_relu(x, bias, negative_slope, scale)

    out = {}
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(O, "random_crops", crops)
        mp.setattr(O, "fused_leaky_relu", head_margin_recorder)
        for kind in kinds:
            mode = "generator" if kind == "G" else "discriminator"
            keys, params = [], []
            for group, nets in groups.items():
                for pre, P in nets.items():
                    for k, v in P.items():
                        if k.endswith(".kernel"):
                            continue
                        v.requires_grad_(group == mode)
                        if group == mode:
                            keys.append(pre + "." + k)
                            params.append(v)
            draws.reseed(crop_seed[kind])
            scale = {}
            margins.clear()
            if kind == "D":
                L = m.discriminator_losses(real, noises)
                total = sum(v.mean() for v in L.values())
                grads = torch.autograd.grad(total, params, allow_unused=True)
            elif kind == "R1":
                L = m.r1_loss(real)
                total = sum(v.mean() for v in L.values()) * copt.R1_once_every
                grads = torch.autograd.grad(total, params, allow_unused=True)
            else:
                maps = [{k: v.clone().requires_grad_() for k, v in d.items()} for d in noises]
                L = m.generator_losses(real, maps)
                total = sum(v.mean() for v in L.values())
                names = sorted(maps[0])
                got = torch.autograd.grad(total, params + [d[n] for d in maps for n in names], allow_unused=True)
                grads, g_maps = got[:len(params)], got[len(params):]
                # d total / d nw = sum over pixels of z * (d total / d z) / nw: the L2 norm of those per-pixel terms
                for i, n in enumerate(names):
                    nw = float(m.G[n + ".noise.weight"].detach())
                    terms = [maps[c][n].detach() * g_maps[c * len(names) + i] / nw for c in range(len(maps))]
                    scale["G.%s.noise.weight" % n] = sum(float(t.pow(2).sum()) for t in terms) ** 0.5
            out[kind] = {"losses": {k: v.detach() for k, v in L.items()}, "grads": dict(zip(keys, grads)), "scale": scale,
                         "head_margin": min(margins)}
    for P in (m.G, m.E, m.D, m.Dp):
        for v in P.values():
            v.requires_grad_(False)
    return out


class _Setup:
    """one configuration: seeded parameters, images, noise, the fp64 truth and the product's model + trainer"""

    def __init__(self, opt_kw, kinds, crop_seed):
        import swapping_autoencoder_pytorch_b200 as S
        from swapping_autoencoder_pytorch_b200 import default_options
        copt = default_options(**dict(opt_kw, num_gpus=0))
        self.sd64 = perturbed_state_dict(copt)
        self.real = rnd(900, copt.batch_size, 3, copt.crop_size, copt.crop_size).clamp(-1, 1)
        self.noises = _noise_maps(copt)
        t0 = time.time()
        self.crop_seed = crop_seed
        self.truth = _fp64_truth(copt, self.sd64, self.real, self.noises, kinds, crop_seed)
        self.truth_seconds = time.time() - t0
        opt = default_options(**dict(opt_kw, num_gpus=1))
        assert opt.batch_discriminator_passes
        torch.manual_seed(0)
        model = S.create_model(opt)
        self.inner = model.singlegpu_model
        missing, unexpected = self.inner.load_state_dict({k: _cuda(v) for k, v in self.sd64.items()}, strict=False)
        assert not unexpected, unexpected
        assert all(k.endswith(".kernel") or k == "num_discriminator_iters" for k in missing), missing
        self.trainer = S.create_optimizer(opt, model)
        self.names = {id(p): n for n, p in self.inner.named_parameters()}


@pytest.fixture(scope="module")
def nets_256():
    return _Setup(OPTS_256, ("D", "R1", "G"), CROP_SEED["256"])


RECORD = {}
RAN = set()


@pytest.fixture(scope="module", autouse=True)
def _write_record():
    yield
    path = os.environ.get("SAE_PARITY_RECORD")
    if RECORD and path:
        old = {}
        if os.path.exists(path):
            try:
                with open(path) as f:
                    old = json.load(f)
            except ValueError:
                old = {}
        old.update(RECORD)
        with open(path, "w") as f:
            json.dump(old, f, indent=1, sort_keys=True)


def _function_classes():
    import importlib
    from torch.autograd import Function
    out = {}
    # by module path: the package re-exports a function named upfirdn2d over its submodule's name
    for name in ("stylegan2_op.conv", "stylegan2_op.blocks", "stylegan2_op.fused_act", "stylegan2_op.upfirdn2d", "util"):
        mod = importlib.import_module("swapping_autoencoder_pytorch_b200." + name)
        for obj in vars(mod).values():
            if isinstance(obj, type) and issubclass(obj, Function) and obj.__module__ == mod.__name__:
                out[obj.__name__] = obj
    return out


@pytest.fixture
def backward_spy():
    """wraps every Function's backward so that RAN collects the names of those that ran"""
    saved = {}
    for name, cls in _function_classes().items():
        orig = cls.__dict__["backward"]
        saved[cls] = orig

        def spy(ctx, *grads, _fn=orig.__func__, _name=name):
            RAN.add(_name)
            return _fn(ctx, *grads)
        cls.backward = staticmethod(spy)
    RAN.clear()
    yield RAN
    for cls, orig in saved.items():
        cls.backward = orig


@pytest.fixture
def served_inputs(monkeypatch):
    """the crop draws and generator noise of the fp64 truth, served to the product: returns a function that installs them for
    one configuration and returns (crop draws, noise server)"""
    from swapping_autoencoder_pytorch_b200 import util
    from swapping_autoencoder_pytorch_b200.stylegan2_layers import NoiseInjection

    draws = _CropDraws()
    monkeypatch.setattr(util, "draw_crop_parameters",
                        lambda b, sr, device: tuple(t.float().to(device) for t in draws.draw(b, sr[0], sr[1])))

    class Server:
        def __init__(self, setup):
            self.names = {id(m): n[:-len(".noise")] for n, m in setup.inner.G.named_modules() if isinstance(m, NoiseInjection)}
            self.maps = [{k: _cuda(v) for k, v in d.items()} for d in setup.noises]
            assert set(self.names.values()) == set(self.maps[0]), (sorted(self.names.values()), sorted(self.maps[0]))
            self.calls = {}

        def resolve(self, module, image, noise=None):
            assert noise is None and module.fixed_noise is None
            if module.image_size is None:
                module.image_size = image.shape
            name = self.names[id(module)]
            i = self.calls.get(name, 0)
            self.calls[name] = i + 1
            z = self.maps[i][name]
            assert tuple(z.shape) == (image.shape[0], 1) + tuple(image.shape[2:]), (name, i, tuple(z.shape), tuple(image.shape))
            return z

    current = []

    def install(setup):
        server = Server(setup)
        current[:] = [server]
        return draws, server
    monkeypatch.setattr(NoiseInjection, "resolve_noise", lambda self, image, noise=None: current[0].resolve(self, image, noise))
    return install


def _run_half_step(setup, kind, general_r1):
    from swapping_autoencoder_pytorch_b200.stylegan2_op import conv as C
    tr = setup.trainer
    images = _cuda(setup.real)
    if kind == "D":
        losses, params = tr._discriminator_body(images, step=False), tr.Dparams
    elif kind == "G":
        losses, params = tr._generator_body(images, step=False), tr.Gparams
    elif not general_r1:
        losses, params = tr._r1_body(images, step=False), tr.Dparams
    else:
        # the route the reference's unchanged model file takes: the recorded backward computes every gradient.  With fused
        # blocks off (per_operator_blocks) it records per-operator nodes; with them on, _ResBlockFused re-evaluates the block
        # per operator inside its recorded backward.
        tr.set_requires_grad(tr.Dparams, True)
        tr.set_requires_grad(tr.Gparams, False)
        tr.optimizer_D.zero_grad()
        prev = C.set_data_gradients_only(False)
        try:
            losses = setup.inner._compute_R1_loss(images)
        finally:
            C.set_data_gradients_only(prev)
        (sum(v.mean() for v in losses.values()) * tr.opt.R1_once_every).backward()
        params = tr.Dparams
    torch.cuda.synchronize()
    grads = {setup.names[id(p)]: p.grad for p in params}
    return {k: v for k, v in losses.items() if not k.startswith("_")}, grads


def _compare(variant, kind, precision, losses, grads, truth):
    """one half-step against its fp64 truth; returns the failures"""
    bound = TOL[(precision, "R1" if kind == "R1" else "first")]
    rec = RECORD.setdefault("training_gradients", {}).setdefault(variant, {}).setdefault(kind, {})
    bad = []
    rec["_head_margin"] = truth["head_margin"]
    if truth["head_margin"] < HEAD_MARGIN:
        bad.append(("fp64 truth: a head pre-activation at %.1e of its layer's RMS; choose another crop seed"
                    % truth["head_margin"],))
    missing, extra = set(truth["grads"]) - set(grads), set(grads) - set(truth["grads"])
    if missing or extra:
        bad.append(("parameter keys differ", sorted(missing), sorted(extra)))
    for name, ref in truth["losses"].items():
        e = rel_err(losses[name], ref)
        rec["loss." + name] = {"rel_max": e}
        if e >= bound:
            bad.append(("loss." + name, e))
    worst = (0.0, None)
    for key in sorted(set(truth["grads"]) & set(grads)):
        ref, got = truth["grads"][key], grads[key]
        if ref is None or not bool(ref.any()):
            zero = got is None or not bool(got.any())
            rec[key] = {"fp64_exact_zero": True, "product_zero": zero}
            if not zero:
                bad.append((key, "fp64 gradient is exactly zero, product's max |g| = %.3e" % float(got.abs().max())))
            continue
        if got is None:
            bad.append((key, "no gradient"))
            continue
        if tuple(got.shape) != tuple(ref.shape):
            bad.append((key, "shape", tuple(got.shape), tuple(ref.shape)))
            continue
        l2, mx = rel_l2(got, ref), rel_err(got, ref)
        rec[key] = entry = {"rel_l2": l2, "rel_max": mx}
        e, b = l2, bound
        if key in truth["scale"]:
            scale = truth["scale"][key]
            entry["natural_scale_over_norm"] = scale / _norm(ref)
            entry["rel_l2_natural_scale"] = float((got.detach().double().cpu() - ref).norm()) / max(_norm(ref), scale)
            if _natural_scale_reason(kind, key):
                e = entry["rel_l2_natural_scale"]
                b = TOL[(precision, "noise")]
        worst = max(worst, (e, key))
        if not e < b:
            bad.append((key, l2, mx, entry.get("rel_l2_natural_scale")))
    rec["_worst_rel_l2"] = {"tensor": worst[1], "rel_l2": worst[0], "bound": bound}
    return bad


def _measure_variant(setup, variant, precision, det, fused, general_r1, kinds, served_inputs, spy):
    """runs the variant's half-steps; returns (failures, names of the Functions whose backward ran)"""
    from swapping_autoencoder_pytorch_b200 import backend
    from swapping_autoencoder_pytorch_b200.stylegan2_op import blocks
    draws, server = served_inputs(setup)
    kern = backend.kernels()
    prev = (kern.precision, kern.deterministic, blocks.set_fused_blocks(fused))
    kern.precision, kern.deterministic = precision, det
    bad, ran = [], set()
    try:
        for kind in kinds:
            server.calls = {}
            spy.clear()
            draws.reseed(setup.crop_seed[kind])
            losses, grads = _run_half_step(setup, kind, general_r1)
            ran |= spy
            if kind != "R1":        # every noise map of both G calls was served, once
                assert server.calls == {n: 2 for n in server.maps[0]}, server.calls
            bad += [(kind,) + b for b in _compare(variant, kind, precision, losses, grads, setup.truth[kind])]
    finally:
        kern.precision, kern.deterministic = prev[0], prev[1]
        blocks.set_fused_blocks(prev[2])
    RECORD.setdefault("backward_ran", {})[variant] = sorted(ran)
    return bad, ran


def _run_variant(setup, variant, *args):
    bad, ran = _measure_variant(setup, variant, *args)
    assert not bad, (variant, bad)
    expected = {name for name, vs in BACKWARD_REACHED.items() if variant in vs}
    assert ran == expected, (variant, "ran but not in the table:", sorted(ran - expected),
                             "in the table but did not run:", sorted(expected - ran))


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_half_step_gradients_256(variant, nets_256, served_inputs, backward_spy):
    RECORD.setdefault("training_gradients_timing", {})["fp64_truth_256_seconds"] = nets_256.truth_seconds
    _run_variant(nets_256, variant, *VARIANTS[variant], served_inputs, backward_spy)


def test_generator_gradients_ffhq_channels(served_inputs, backward_spy):
    """G step in fp32 mode with the ffhq1024 channel set at 256²: 409 / 204 / 102 channels through the channel-pad kernel, the
    memoised padded filter and the slice back"""
    setup = _Setup(OPTS_FFHQ_256, ("G",), CROP_SEED["ffhq"])
    RECORD.setdefault("training_gradients_timing", {})["fp64_truth_ffhq_G_seconds"] = setup.truth_seconds
    _run_variant(setup, FFHQ, "fp32", False, True, False, ("G",), served_inputs, backward_spy)
