"""GPU (H100): the adaptive discriminator augmentation's kernels (csrc/augment.cu) and its training-loop integration.

* the geometric operator against the fp64 restatement (tests/ada_oracle.py), given matrices: the identity forced through the
  resampler, each transform alone and random composites at p = 1, at 32², 64², 256² and 48 × 80, max-norm relative
  <= 2e-5 in both precision modes (nothing is rounded to TF32); the identity copy is bitwise;
* the adjoint: <A x, y> = <x, A^T y> to 1e-5 relative, A^T against the oracle's autograd backward to 2e-5;
* the colour operator and its transpose against the oracle to 1e-6; the matrices from the same draws to 1e-6, exactly I at
  p = 0; the p adjustment bitwise equal to the host formula;
* R1 through the augmentation on the tiny nets: the adjoint of D's input gradient, the gradient with respect to real and
  the penalty against fp64 in both modes, D's weight gradients in the fp32 mode;
* deterministic mode with tuning on: two runs bitwise equal, and eager execution bitwise equal to graph replay, in p, losses
  and parameters over 16 half-steps with a lazy R1 and two adjustments."""
import math

import numpy as np
import pytest
import torch

from oracle import sae_oracle as O
from oracle.fixtures import TINY, rel_err, rel_l2, rnd
from swapping_autoencoder_pytorch_b200 import _lib, augment, backend, default_options
from swapping_autoencoder_pytorch_b200.backend import nhwc
from tests import ada_oracle as A

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture
def kern():
    k = backend.kernels()
    prev = (k.precision, k.deterministic, k.round_tf32)
    yield k
    k.precision, k.deterministic, k.round_tf32 = prev


def _eye(n):
    return torch.eye(3, dtype=torch.float64).expand(n, 3, 3).clone()


def _rot(t):
    return torch.tensor([[math.cos(t), -math.sin(t), 0.0], [math.sin(t), math.cos(t), 0.0], [0.0, 0.0, 1.0]],
                        dtype=torch.float64)


def _single_transforms(h, w):
    """G_inv of each geometric transform alone, as aug_params_kernel composes it"""
    return {
        "xflip": torch.diag(torch.tensor([-1.0, 1.0, 1.0], dtype=torch.float64)),
        "rot90": _rot(math.pi / 2),
        "int_translation": torch.tensor([[1.0, 0, -round(0.1 * w)], [0, 1.0, round(0.07 * h)], [0, 0, 1.0]],
                                        dtype=torch.float64),
        "iso_scale": torch.diag(torch.tensor([1 / 1.2, 1 / 1.2, 1.0], dtype=torch.float64)),
        "rotation": _rot(0.7),
        "aniso_scale": torch.diag(torch.tensor([1 / 1.15, 1.15, 1.0], dtype=torch.float64)),
        "frac_translation": torch.tensor([[1.0, 0, -0.0625 * w], [0, 1.0, 0.031 * h], [0, 0, 1.0]], dtype=torch.float64),
    }


def _records(G, C=None):
    """fp32 device records and the fp64 matrices they hold (the oracle runs on the very values the kernels read)"""
    n = G.shape[0]
    if C is None:
        C = torch.eye(4, dtype=torch.float64).expand(n, 4, 4)
    rec = A.pack(G.float(), C.float()).to(DEV)
    g, c = A.unpack(rec.double())
    return rec, g, c


SIZES = [(32, 32), (64, 64), (256, 256), (48, 80)]


@pytest.mark.parametrize("precision", ["tf32", "fp32"])
@pytest.mark.parametrize("h,w", SIZES, ids=["%dx%d" % s for s in SIZES])
def test_geometric_against_fp64(kern, precision, h, w):
    kern.precision = precision
    n = 2 if h >= 256 else 3
    x = (rnd(960 + h, n, 3, h, w).clamp(-2, 2)).float().to(DEV)
    x64 = x.double()
    cases = {"identity": _eye(n)}
    cases.update({k: v.expand(n, 3, 3).clone() for k, v in _single_transforms(h, w).items()})
    gen = torch.Generator().manual_seed(h * 1000 + w)
    u, z = torch.rand(n, A.UNIFORMS, generator=gen, dtype=torch.float64), torch.randn(n, A.NORMALS, generator=gen,
                                                                                          dtype=torch.float64)
    cases["composite_p1"] = A.matrices(u.float(), z.float(), 1.0, h, w)[0]
    worst = {}
    for name, G in cases.items():
        rec, g, _ = _records(G)
        y = augment.augment(x, rec, copy_identity=False)
        ref = A.geometric(x64, g.to(DEV), copy_identity=False)
        worst[name] = rel_err(y, ref)
    bound = {"identity": 1e-5}
    bad = {k: v for k, v in worst.items() if not v <= bound.get(k, 2e-5)}
    assert not bad, (bad, worst)


def test_identity_is_copied_bitwise(kern):
    x = torch.randn(3, 3, 48, 80, device=DEV)
    rec, _, _ = _records(_eye(3))
    for precision in ("tf32", "fp32"):
        kern.precision = precision
        assert torch.equal(augment.augment(x, rec), x)
    # a view with other strides: the copy reads it through them
    xs = torch.randn(3, 48, 80, 3, device=DEV).permute(0, 3, 1, 2)
    assert torch.equal(augment.augment(xs, rec), xs)


@pytest.mark.parametrize("h,w", [(32, 32), (48, 80), (256, 256)], ids=["32x32", "48x80", "256x256"])
def test_adjoint(h, w):
    n = 2
    gen = torch.Generator().manual_seed(7 + h)
    u, z = torch.rand(n, A.UNIFORMS, generator=gen), torch.randn(n, A.NORMALS, generator=gen)
    G, C = A.matrices(u, z, 1.0, h, w)
    G[1] = _eye(1)[0]                                  # one identity image: its adjoint is the colour transpose alone
    rec, g, c = _records(G, C)
    x = torch.randn(n, 3, h, w, device=DEV)
    ax = augment.linear(x, rec)
    y = ax + torch.randn_like(ax)
    aty = augment.adjoint(y, rec)
    lhs, rhs = float((ax.double() * y.double()).sum()), float((x.double() * aty.double()).sum())
    assert abs(lhs - rhs) <= 1e-5 * abs(lhs), (lhs, rhs)
    # the reference runs on the CPU: on the device its backward would start cuBLAS on the autograd engine's device thread,
    # after which torch.profiler in the same process (tests/test_gpu_bandwidth_paths.py counts kernels with it) was seen to
    # miss a call's kernels now and then
    x64 = x.double().cpu().requires_grad_()
    ref, = torch.autograd.grad(A.augment(x64, g.cpu(), c.cpu()), x64, y.double().cpu())
    assert rel_err(aty, ref) <= 2e-5
    # the adjoint's backward is the operator's linear part
    yg = y.clone().requires_grad_()
    t = torch.randn_like(x)
    back, = torch.autograd.grad(augment.adjoint(yg, rec), yg, t)
    assert torch.equal(back, augment.linear(t, rec))


def test_color_and_transpose(kern):
    n, h, w = 4, 17, 29
    gen = torch.Generator().manual_seed(3)
    u, z = torch.rand(n, A.UNIFORMS, generator=gen), torch.randn(n, A.NORMALS, generator=gen)
    G, C = A.matrices(u, z, 1.0, h, w)
    G[0] = _eye(1)[0]
    C[3] = torch.eye(4, dtype=torch.float64)
    rec, g, c = _records(G, C)
    a = torch.randn(n, 3, h, w, device=DEV)
    b = torch.randn(n, 3, h, w, device=DEV)
    k = backend.kernels()
    for offset in (True, False):
        b4 = torch.cat([nhwc(b), torch.full_like(nhwc(b)[..., :1], float("nan"))], 3)          # channel 3 is never read
        out = k.augment_color(a, b4, rec, offset=offset, copy_identity=True).permute(0, 3, 1, 2)
        v = torch.where(A.is_identity(g).to(DEV).view(-1, 1, 1, 1), a, b).double()
        assert rel_err(out, A.color(v, c.to(DEV), offset)) <= 1e-6
        assert torch.equal(out[3], (a[3] if A.is_identity(g)[3] else b[3]))       # C = I: a copy
    dy = torch.randn(n, 3, h, w, device=DEV).permute(0, 1, 3, 2).contiguous().permute(0, 1, 3, 2)    # other strides
    gc4 = k.augment_color_adjoint(dy, rec)
    assert torch.equal(gc4[..., 3], torch.zeros_like(gc4[..., 3]))
    gc = gc4[..., :3].permute(0, 3, 1, 2)
    assert rel_err(gc, torch.einsum("nji,njhw->nihw", c.to(DEV)[:, :3, :3], dy.double())) <= 1e-6
    assert torch.equal(gc[3], dy[3])


@pytest.mark.parametrize("p", [0.0, 0.3, 1.0, 1.7])
def test_matrices_from_draws(p):
    n, h, w = 4096, 256, 192
    u, z = augment.draw(n, DEV)
    pd = torch.full((1,), p, device=DEV)
    rec = augment.params(u, z, pd, h, w)
    G, C = A.unpack(rec.double().cpu())
    Gr, Cr = A.matrices(u.cpu(), z.cpu(), float(pd), h, w)
    if p == 0.0:
        assert torch.equal(G, _eye(n)) and torch.equal(C, torch.eye(4, dtype=torch.float64).expand(n, 4, 4))
    for got, ref in ((G, Gr), (C, Cr)):
        err = ((got - ref).abs() / ref.abs().clamp_min(1.0)).max()
        assert float(err) <= 1e-6, float(err)
    assert torch.equal(rec[:, 25:].cpu(), torch.zeros(n, _lib.SAE_AUG_RECORD - 25))


def test_p_adjust_is_the_host_formula():
    k = backend.kernels()
    cases = [(0.25, [3.0, 10.0, 16.0, 0.0], 0.013, 0.6), (0.25, [3.0, 6.0, 16.0, 1.0], 0.013, 0.6),
             (0.004, [0.0, -7.0, 9.0, 0.0], 0.031, 0.6), (0.7, [0.0, 3.0, 5.0, 0.0], 1e-3, 0.6),
             (0.5, [0.0, 0.0, 0.0, 4.0], 0.2, 0.6), (0.1, [1.0, 5.0, 7.0, 0.0], 1.0 / 3.0, 0.6)]
    for p0, acc0, step, target in cases:
        p = torch.full((1,), p0, device=DEV)
        acc = torch.tensor(acc0, dtype=torch.float64, device=DEV)
        k.ada_adjust(p, acc, step, target)
        exp = np.float32(p0)
        if acc0[2] > 0:
            exp = max(np.float32(0), exp + np.float32(np.sign(acc0[1] / acc0[2] - target) * step))
        assert p.cpu().numpy().view(np.int32)[0] == np.array([exp], dtype=np.float32).view(np.int32)[0], (p0, acc0)
        assert acc.abs().sum().item() == 0.0


# ------------------------------------------------------------------------------------------------------------- R1
R1_TOL = {"tf32": 2.5e-2, "fp32": 5e-4}


@pytest.mark.parametrize("precision", ["tf32", "fp32"])
def test_r1_through_the_augmentation(kern, precision):
    import swapping_autoencoder_pytorch_b200 as S
    kern.precision = precision
    opt = default_options(**dict(TINY, num_gpus=1, augment_p=1.0, lambda_patch_R1=0.0, R1_once_every=4))
    torch.manual_seed(0)
    tr = S.create_optimizer(opt, S.create_model(opt))
    inner = tr.model.singlegpu_model
    real = rnd(970, 2, 3, 64, 64).clamp(-1, 1)
    # seed 9 would put one of D's leaky-ReLU pre-activations at the augmented image within fp32 rounding of zero: D's own
    # input gradient there is 1.9e-3 off fp64 in the fp32 mode, with or without the augmentation.  This seed does not.
    gen = torch.Generator().manual_seed(10)
    G, C = A.matrices(torch.rand(2, A.UNIFORMS, generator=gen), torch.randn(2, A.NORMALS, generator=gen), 1.0, 64, 64)
    rec, g, c = _records(G, C)
    g, c = g.cpu(), c.cpu()
    assert not A.is_identity(g).any()
    inner.augment_pipe = lambda x: augment.augment(x, rec)
    # the product: the R1 half-step body's loss and backward, and the gradient with respect to real
    x = real.float().to(DEV)
    tr.set_requires_grad(tr.Dparams, True)
    tr.set_requires_grad(tr.Gparams, False)
    tr.optimizer_D.zero_grad()
    r1 = inner(x.clone(), command="compute_R1_loss")
    (sum(v.mean() for v in r1.values()) * opt.R1_once_every).backward()
    xg = x.clone().requires_grad_()
    gx, = torch.autograd.grad(inner.D(inner.augment_pipe(xg)).sum(), xg)
    # the adjoint alone, on the gradient the product's D hands it
    a = augment.augment(x, rec).detach().requires_grad_()
    dy, = torch.autograd.grad(inner.D(a).sum(), a)
    x64 = real.clone().requires_grad_()
    ref, = torch.autograd.grad(A.augment(x64, g, c), x64, dy.double().cpu())
    assert rel_err(augment.adjoint(dy, rec), ref) <= 2e-5
    # fp64
    sd = {k: v.detach().double().cpu() for k, v in inner.state_dict().items()}
    D = {k[2:]: v for k, v in sd.items() if k.startswith("D.")}
    leaves = {k: v.requires_grad_() for k, v in D.items() if not k.endswith(".kernel")}
    x64 = real.clone().requires_grad_()
    pred = O.discriminator_forward(D, opt, A.augment(x64, g, c)).sum()
    g64, = torch.autograd.grad(pred, x64, create_graph=True)
    pen = g64.pow(2).sum(dim=(1, 2, 3)) * (opt.lambda_R1 * 0.5)
    names = list(leaves)
    grads = torch.autograd.grad(pen.mean() * opt.R1_once_every, [leaves[k] for k in names], allow_unused=True)
    assert rel_l2(gx, g64) <= R1_TOL[precision]
    assert rel_err(r1["D_R1"], pen) <= R1_TOL[precision]
    if precision == "tf32":
        # the tiny nets' deepest R1 weight gradients are 2.7-3.1e-2 off fp64 in TF32 mode (the bound is the 256² nets'); the
        # augmentation is the same fp32 operator in both modes, so its weight gradients are checked in the fp32 mode, where
        # the bound is sharp
        return
    params = dict(inner.named_parameters())
    bad = []
    for k, ref in zip(names, grads):
        got = params["D." + k].grad
        if ref is None or float(ref.abs().max()) == 0.0:
            assert got is None or float(got.abs().max()) == 0.0, k
            continue
        e = rel_l2(got, ref)
        if not e <= R1_TOL[precision]:
            bad.append((k, e))
    assert not bad, bad


# ------------------------------------------------------------------------------------------------------------- determinism
def _trainer(**over):
    import swapping_autoencoder_pytorch_b200 as S
    opt = default_options(**dict(TINY, num_gpus=1, R1_once_every=4, augment_p=0.5, ada_target=0.6, ada_kimg=0.1,
                                 ada_interval=4, **over))
    torch.manual_seed(0)
    return S.create_optimizer(opt, S.create_model(opt))


def _run(graphs, steps=16, **over):
    tr = _trainer(cuda_graphs=graphs, **over)
    torch.manual_seed(123)
    real = torch.randn(2, 3, 64, 64, device=DEV, generator=torch.Generator(DEV).manual_seed(5)).clamp(-1, 1)
    snaps = []
    for _ in range(steps):
        out = tr.train_one_step({"real_A": real}, 0)
        snaps.append((tr.augment.p.clone(), {k: float(v) for k, v in out.items()},
                      [p.detach().clone() for p in tr.model.singlegpu_model.parameters()]))
    if graphs:
        assert tr.graphs.disabled is None, (tr.graphs.disabled, tr.graphs.last_traceback)
        assert all(key[-1] == ("ada",) for key in tr.graphs.captured), sorted(tr.graphs.captured)
    return snaps


def _bitwise(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


def _same(a, b):
    for step, (sa, sb) in enumerate(zip(a, b)):
        assert _bitwise(sa[0], sb[0]), (step, sa[0], sb[0])
        assert sa[1] == sb[1], (step, sa[1], sb[1])
        assert all(_bitwise(x, y) for x, y in zip(sa[2], sb[2])), step


def test_deterministic_runs_are_bitwise_equal(kern):
    kern.deterministic = True
    a, b = _run(True), _run(True)
    _same(a, b)
    ps = [float(s[0]) for s in a]
    assert ps[0] == np.float32(0.5) and len(set(ps)) >= 2, ps          # tuned at least once
    assert sum("D_R1" in s[1] for s in a) == 2


def test_eager_equals_graph_replay_bitwise(kern, monkeypatch):
    """Without random draws eager and replayed trajectories must coincide: noise maps zero, no patch discriminator, and the
    augmentation's draws the same fixed numbers on every call (copied inside the graph, as its draws would be made there)."""
    from swapping_autoencoder_pytorch_b200.stylegan2_layers import NoiseInjection

    def zero_noise(self, image, noise=None):
        if self.image_size is None:
            self.image_size = image.shape
        b, _, h, w = image.shape
        return image.new_empty(b, 1, h, w).zero_()
    monkeypatch.setattr(NoiseInjection, "resolve_noise", zero_noise)
    gen = torch.Generator(DEV).manual_seed(17)
    fixed = (torch.rand(64, _lib.SAE_AUG_UNIFORMS, device=DEV, generator=gen),
             torch.randn(64, _lib.SAE_AUG_NORMALS, device=DEV, generator=gen))
    monkeypatch.setattr(augment, "draw", lambda n, device, dtype=torch.float32: (fixed[0][:n].clone(), fixed[1][:n].clone()))
    kern.deterministic = True
    over = dict(lambda_PatchGAN=0.0, lambda_patch_R1=0.0)
    eager, graph = _run(False, **over), _run(True, **over)
    _same(eager, graph)
    ps = [float(s[0]) for s in eager]
    assert len(set(ps)) >= 2, ps
