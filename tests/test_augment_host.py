"""CPU: the adaptive discriminator augmentation (opt.augment_p / opt.ada_target; augment.AugmentPipe) on the kernel emulation.

* the fp64 oracle: the identity chain reproduces the input, an integer translation shifts it exactly (reflecting at the
  border), the matrices are I at p = 0 and every gate is open at p = 1;
* the autograd Functions: forward against the oracle, the adjoint's dot-product identity, double backward;
* p tuning: a scripted sequence of real-logit signs gives, after 12 D updates at ada_interval 4, exactly the p of the
  formula in numpy float32, with one adjustment per update at micro_batches 2;
* per-sample identical D / G / R1 losses with batch_discriminator_passes on and off, augmentation on;
* off changes nothing: the same random draws consumed, graph keys and state_dict keys; on: the "ada" state round trip;
* two ranks over gloo with different local logits end with the same p."""
import os
import socket
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle.fixtures import TINY, rnd
from swapping_autoencoder_pytorch_b200 import augment, backend, default_options
from tests import ada_oracle as A
from tests.cpu_emulation import EmulatedKernels


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


class AugmentKernels(EmulatedKernels):
    """the emulation with the augmentation's entry points (include/sae_b200.h, ABI 20) restated on the oracle, plus
    score_stats; ``log`` records the augmentation and tuning calls"""

    def __init__(self):
        self.log = []

    def upfirdn2d(self, x, kernel, up_x, up_y, down_x, down_y, pad_x0, pad_x1, pad_y0, pad_y1, taps=None, round_tf32=None):
        return EmulatedKernels.upfirdn2d(self, x, kernel, up_x, up_y, down_x, down_y, pad_x0, pad_x1, pad_y0, pad_y1, taps)

    def score_stats(self, x, acc):
        self.log.append(("score_stats", tuple(x.shape)))
        fin = torch.isfinite(x)
        acc[0] += float(x[fin].double().sum())
        acc[1] += float(torch.sign(x[fin]).double().sum())
        acc[2] += int(fin.sum())
        acc[3] += int((~fin).sum())

    def augment_params(self, u, z, p, h, w):
        self.log.append(("augment_params", u.shape[0]))
        G, C = A.matrices(u, z, float(p.reshape(-1)[0]), h, w)
        return A.pack(G, C).to(u.dtype)

    def augment_sample(self, x, rec, copy_identity=True):
        G, _ = A.unpack(rec)
        s = A.sample(x, G)
        if copy_identity:
            s = torch.where(A.is_identity(G).view(-1, 1, 1, 1), torch.zeros_like(s), s)
        return _nhwc(torch.cat([s, torch.zeros_like(s[:, :1])], 1))

    def augment_sample_adjoint(self, ds, gc, rec, h, w, copy_identity=True):
        def vjp():
            x = torch.zeros(ds.shape[0], 3, h, w, dtype=ds.dtype, requires_grad=True)
            return torch.autograd.grad(A.sample(x, A.unpack(rec)[0]), x, _nchw(ds)[:, :3])[0]
        # the product calls this from inside a custom op, where autograd is dispatched past: the restatement's VJP runs on a
        # thread of its own, whose dispatch state is fresh
        with ThreadPoolExecutor(1) as pool:
            dx = _nhwc(pool.submit(vjp).result())
        if copy_identity:
            dx = torch.where(A.is_identity(A.unpack(rec)[0]).view(-1, 1, 1, 1), gc[..., :3], dx)
        return dx

    def augment_color(self, a, b, rec, offset=True, copy_identity=True):
        G, C = A.unpack(rec)
        v = _nchw(b)[:, :3]
        if copy_identity:
            v = torch.where(A.is_identity(G).view(-1, 1, 1, 1), a, v)
        return _nhwc(A.color(v, C, offset))

    def augment_color_adjoint(self, dy, rec):
        C = A.unpack(rec)[1]
        g = torch.einsum("nji,njhw->nihw", C[:, :3, :3], dy)
        return _nhwc(torch.cat([g, torch.zeros_like(g[:, :1])], 1))

    def ada_adjust(self, p, acc, step, target):
        self.log.append(("ada_adjust", float(step), float(target)))
        if float(acc[2]) > 0:
            rt = float(acc[1]) / float(acc[2])
            adjust = float(np.sign(rt - target)) * step
            p.copy_(torch.tensor([max(np.float32(0), np.float32(float(p[0])) + np.float32(adjust))], dtype=torch.float32))
        acc.zero_()


@pytest.fixture
def kern():
    prev = backend.set_kernels(AugmentKernels())
    yield backend.kernels()
    backend.set_kernels(prev)


def _trainer(**over):
    import swapping_autoencoder_pytorch_b200 as S
    opt = default_options(**dict(TINY, **over))
    torch.manual_seed(0)
    return S.create_optimizer(opt, S.create_model(opt))


# ------------------------------------------------------------------------------------------------------------- oracle
def test_oracle_identity_and_integer_translation():
    x = rnd(930, 2, 3, 16, 24)
    eye = torch.eye(3, dtype=torch.float64).expand(2, 3, 3).clone()
    assert (A.geometric(x, eye, copy_identity=False) - x).abs().max() <= 1e-10
    assert torch.equal(A.geometric(x, eye), x)
    for tx, ty in ((3, -2), (-5, 4), (7, 0)):
        G = eye.clone()
        G[:, 0, 2], G[:, 1, 2] = -tx, -ty                       # G_inv = translate2d(t)^-1: out[k] = x[k - t]
        ref = torch.nn.functional.pad(x, (23, 23, 15, 15), mode="reflect")
        exp = ref[:, :, 15 - ty:15 - ty + 16, 23 - tx:23 - tx + 24]
        assert (A.geometric(x, G) - exp).abs().max() <= 1e-10, (tx, ty)


def test_oracle_matrices_gates():
    torch.manual_seed(1)
    u, z = torch.rand(64, A.UNIFORMS, dtype=torch.float64), torch.randn(64, A.NORMALS, dtype=torch.float64)
    G, C = A.matrices(u, z, 0.0, 32, 32)
    assert torch.equal(G, torch.eye(3, dtype=torch.float64).expand(64, 3, 3))
    assert torch.equal(C, torch.eye(4, dtype=torch.float64).expand(64, 4, 4))
    # p = 1: every gate is open, so each factor depends on its draw; check two factors whose effect is visible alone
    G1, C1 = A.matrices(u, z, 1.0, 32, 32)
    assert not A.is_identity(G1).any()
    only_brightness = torch.zeros_like(u) + 0.99                  # every gate closed at p = 0.5 ...
    only_brightness[:, 14] = 0.0                                  # ... but brightness's
    _, Cb = A.matrices(only_brightness, z, 0.5, 32, 32)
    assert torch.allclose(Cb[:, 0, 3], 0.2 * z[:, 4]) and torch.equal(Cb[:, :3, :3], torch.eye(3, dtype=torch.float64).expand(64, 3, 3))
    ones = torch.zeros_like(u)                                    # u = 0 opens every gate for any p > 0
    G2, C2 = A.matrices(ones, z, 1e-6, 32, 32)
    G3, C3 = A.matrices(ones, z, 1.0, 32, 32)
    assert torch.equal(G2, G3) and torch.equal(C2, C3)
    assert not torch.equal(C3, torch.eye(4, dtype=torch.float64).expand(64, 4, 4))


# ------------------------------------------------------------------------------------------------------------- Functions
def test_functions_match_the_oracle_and_are_twice_differentiable(kern, fp64_default):
    torch.manual_seed(2)
    n, h, w = 4, 12, 16
    x = rnd(931, n, 3, h, w)
    u, z = torch.rand(n, A.UNIFORMS), torch.randn(n, A.NORMALS)
    u[0] = 0.999                                                  # image 0: every gate closed, so it is copied
    G, C = A.matrices(u, z, 0.7, h, w)
    rec = A.pack(G, C)
    y = augment.augment(x, rec)
    assert (y - A.augment(x, G, C)).abs().max() <= 1e-12
    assert torch.equal(y[0], x[0])
    # <A x, v> = <x, A^T v> for the linear part, and the double backward is the linear operator again
    xg = x.clone().requires_grad_()
    v = rnd(932, n, 3, h, w)
    lin = augment.linear(xg, rec)
    g, = torch.autograd.grad((lin * v).sum(), xg, create_graph=True)
    assert abs(float((lin * v).sum().detach()) - float((x * g).sum().detach())) <= 1e-10 * float(lin.detach().abs().sum())
    t = rnd(933, n, 3, h, w)
    vg = v.clone().requires_grad_()
    g2, = torch.autograd.grad(augment.adjoint(vg, rec), vg, t)
    assert (g2 - augment.linear(t, rec)).abs().max() <= 1e-12
    assert torch.autograd.gradcheck(lambda a: augment.augment(a, rec), (x[:, :, :6, :6].clone().requires_grad_(),))
    assert torch.autograd.gradgradcheck(lambda a: augment.augment(a, rec).pow(2).sum(), (x[:, :, :6, :6].clone().requires_grad_(),))


# ------------------------------------------------------------------------------------------------------------- tuning
def _scripted_real_logits(tr, signs):
    """make every D-step D(real) of ``tr`` be a tensor whose signs come, one update at a time, from ``signs``"""
    pipe = tr.augment
    orig = pipe.observe
    it = iter(signs)

    def observe(logits):
        s = next(it)
        orig(torch.tensor(s, dtype=logits.dtype).view(-1, 1))
    pipe.observe = observe


@pytest.mark.parametrize("micro_batches", [1, 2])
def test_p_tuning_follows_the_formula(kern, fp64_default, micro_batches):
    target, kimg, interval, batch = 0.6, 0.05, 4, 4
    tr = _trainer(ada_target=target, ada_kimg=kimg, ada_interval=interval, augment_p=0.1, micro_batches=micro_batches,
                  lambda_R1=0.0, lambda_patch_R1=0.0)
    rng = np.random.RandomState(3)
    per_update = [[rng.choice([-1.0, 1.0], size=batch // micro_batches, p=[q, 1 - q]).tolist() for _ in range(micro_batches)]
                  for q in rng.uniform(0.0, 0.6, size=12)]
    _scripted_real_logits(tr, [s for upd in per_update for s in upd])
    real = rnd(934, batch, 3, 64, 64).clamp(-1, 1)
    p = np.float32(0.1)
    for k in range(12):
        tr.train_discriminator_one_step(real)
        if (k + 1) % interval == 0:
            signs = [s for upd in per_update[k + 1 - interval:k + 1] for m in upd for s in m]
            rt = sum(signs) / len(signs)
            adjust = np.sign(rt - target) * batch * interval / (kimg * 1000)
            p = max(np.float32(0), p + np.float32(adjust))
    assert [e for e in kern.log if e[0] == "ada_adjust"] == [("ada_adjust", batch * interval / (kimg * 1000), target)] * 3
    assert tr.augment_p() == float(p) and p != np.float32(0.1)
    assert sum(1 for e in kern.log if e[0] == "augment_params") == 12 * micro_batches


# ------------------------------------------------------------------------------------------------------------- losses
def test_batched_and_three_pass_discriminators_agree(kern, fp64_default):
    real = rnd(935, 4, 3, 64, 64).clamp(-1, 1)
    out = []
    for batched in (True, False):
        tr = _trainer(augment_p=0.8, batch_discriminator_passes=batched, R1_once_every=1)
        model = tr.model.singlegpu_model
        torch.manual_seed(11)
        d, _, _, _ = model(real, command="compute_discriminator_losses")
        torch.manual_seed(12)
        g, _ = model(real, command="compute_generator_losses")
        torch.manual_seed(13)
        r1 = model(real.clone(), command="compute_R1_loss")
        out.append({**{k: v.detach() for k, v in d.items()}, **{k: v.detach() for k, v in g.items()},
                    "D_R1": r1["D_R1"].detach()})
    a, b = out
    assert sorted(a) == sorted(b)
    for k in a:
        assert a[k].shape == b[k].shape and (a[k] - b[k]).abs().max() <= 1e-10 * max(1.0, float(a[k].abs().max())), k


def test_r1_gradient_is_taken_through_the_augmentation(kern, fp64_default):
    tr = _trainer(augment_p=1.0, lambda_patch_R1=0.0)
    model = tr.model.singlegpu_model
    real = rnd(936, 2, 3, 64, 64).clamp(-1, 1)
    torch.manual_seed(4)
    r1 = model(real.clone(), command="compute_R1_loss")["D_R1"]
    torch.manual_seed(4)
    u, z = augment.draw(2, real.device, real.dtype)
    G, C = A.matrices(u, z, 1.0, 64, 64)
    x = real.clone().requires_grad_()
    model.augment_pipe = None
    g, = torch.autograd.grad(model.D(A.augment(x, G, C)).sum(), x)
    exp = g.pow(2).sum([1, 2, 3]) * (tr.opt.lambda_R1 * 0.5)
    assert r1.shape == exp.shape and float((r1 - exp).abs().max()) <= 1e-10 * float(exp.abs().max())
    assert float((A.augment(real, G, C) - real).abs().max()) > 0.1                 # p = 1: the images did change


# ------------------------------------------------------------------------------------------------------------- off / state
def test_off_changes_nothing(kern, fp64_default, monkeypatch):
    tr = _trainer(R1_once_every=1)
    assert tr.augment is None and tr.augment_key() == () and tr.model.singlegpu_model.augment_pipe is None
    real = rnd(937, 2, 3, 64, 64).clamp(-1, 1)

    def no_draw(*a, **k):
        raise AssertionError("the augmentation drew with the option off")
    monkeypatch.setattr(augment, "draw", no_draw)
    torch.manual_seed(5)
    tr.train_one_step({"real_A": real}, 0)                        # D + R1
    tr.train_one_step({"real_A": real}, 0)                        # G
    after = torch.rand(4)
    assert kern.log == []
    monkeypatch.undo()
    assert sorted(tr.state_dict()) == ["discriminator_iter_counter", "optimizer_D", "optimizer_G", "train_mode_counter"]
    with pytest.raises(RuntimeError):
        tr.augment_p()
    on = _trainer(augment_p=0.3)
    assert on.augment_key() == (("ada",),)
    assert sorted(on.state_dict()) == sorted(tr.state_dict() | {"ada": None})
    assert list(tr.model.singlegpu_model.state_dict()) == list(on.model.singlegpu_model.state_dict())
    # the augmentation consumes its draws only when on
    torch.manual_seed(5)
    on.train_one_step({"real_A": real}, 0)
    on.train_one_step({"real_A": real}, 0)
    assert not torch.equal(torch.rand(4), after)


@pytest.mark.parametrize("bad", [dict(augment_p=-0.1), dict(augment_p=float("nan")), dict(ada_target=1.0),
                                 dict(ada_target=-0.5), dict(ada_kimg=0.0), dict(ada_interval=0), dict(ada_interval=2.5)])
def test_out_of_range_options_raise(kern, bad):
    with pytest.raises(ValueError):
        _trainer(**bad)


def test_state_dict_round_trip(kern, fp64_default):
    tr = _trainer(ada_target=0.6, augment_p=0.25)
    with torch.no_grad():
        tr.augment.p.fill_(0.375)
        tr.augment.acc.copy_(torch.tensor([1.5, -2.0, 6.0, 1.0], dtype=torch.float64))
    sd = tr.state_dict()
    assert sorted(sd["ada"]) == ["acc", "p"]
    fresh = _trainer(ada_target=0.6, augment_p=0.25)
    p_obj, acc_obj = fresh.augment.p, fresh.augment.acc
    fresh.load_state_dict(sd)
    assert fresh.augment.p is p_obj and fresh.augment.acc is acc_obj           # in place
    assert fresh.augment_p() == 0.375 and fresh.augment.acc.tolist() == [1.5, -2.0, 6.0, 1.0]


# ------------------------------------------------------------------------------------------------------------- two ranks
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out):
    import swapping_autoencoder_pytorch_b200 as S
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    backend.set_kernels(AugmentKernels())
    torch.set_default_dtype(torch.float64)
    opt = default_options(**dict(TINY, ada_target=0.6, ada_kimg=0.1, ada_interval=2, augment_p=0.2, lambda_R1=0.0,
                                 lambda_patch_R1=0.0))
    torch.manual_seed(100 + rank)
    model = S.create_model(opt)
    trainer = S.create_optimizer(opt, model)
    pipe = trainer.augment
    orig = pipe.observe
    # rank 0 sees mostly positive real logits, rank 1 mostly negative ones: only their sum decides the direction
    pipe.observe = lambda logits: orig(torch.full((3, 1), 1.0 if rank == 0 else -0.5))
    x = model.shard(rnd(938, 4, 3, 64, 64).clamp(-1, 1))
    torch.manual_seed(7 + rank)
    ps = []
    for _ in range(4):
        trainer.train_discriminator_one_step(x)
        ps.append(trainer.augment_p())
    torch.save({"p": ps, "acc": pipe.acc.clone()}, os.path.join(out, "a%d.pt" % rank))
    dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_two_ranks_end_with_the_same_p(tmp_path):
    world = 2
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    a0 = torch.load(os.path.join(tmp_path, "a0.pt"))
    a1 = torch.load(os.path.join(tmp_path, "a1.pt"))
    assert a0["p"] == a1["p"]
    # over both ranks r_t = (3 * 1 + 3 * -1) / 6 = 0 < 0.6 (rank 0 alone would have 1 > 0.6): p falls by
    # B * interval / (kimg * 1000) = (2 * 2) * 2 / 100 per adjustment
    step = np.float32(-(2 * 2) * 2 / 100.0)
    p0 = np.float32(0.2)
    p1 = max(np.float32(0), p0 + step)
    assert a0["p"] == [float(p0), float(p1), float(p1), float(max(np.float32(0), p1 + step))]
    assert float(a0["acc"].abs().sum()) == 0.0 and float(a1["acc"].abs().sum()) == 0.0
