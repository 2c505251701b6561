"""CPU: host logic of gradient accumulation (opt.micro_batches) on the kernel emulation, in fp64.

* k = 1: a D + R1 and a G update make exactly the kernel calls they made before the option existed;
* k = 2: one update equals, bitwise, the trainer's own bodies run with step=False on micro-batch 0 then 1, their gradients
  summed in that order and one Adam step with grad_scale = 1 / 2; the returned losses are the means of the micro-batch losses;
* the D / G schedule, lazy R1 and the model's iteration buffer advance once per update;
* a batch that does not split raises ValueError before any kernel call;
* two ranks over gloo: one all-reduce per update, and the update equals Adam on the average of the four micro-batch
  gradients."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle.fixtures import TINY, rnd
from swapping_autoencoder_pytorch_b200 import backend, default_options
from tests.cpu_emulation import EmulatedKernels


class SpyKernels(EmulatedKernels):
    """the emulation, recording the optimizer's and the bucket's calls"""

    def __init__(self):
        self.log = []

    def adam_step(self, *args, **kw):
        self.log.append(("adam_step", len(args), tuple(sorted(kw))))
        return super().adam_step(*args, **kw)

    def bucket_pack(self, *args):
        self.log.append(("bucket_pack", len(args), ()))
        return super().bucket_pack(*args)

    def bucket_accumulate(self, *args):
        self.log.append(("bucket_accumulate", len(args), ()))
        raise NotImplementedError


@pytest.fixture
def spy():
    prev = backend.set_kernels(SpyKernels())
    yield backend.kernels()
    backend.set_kernels(prev)


def _trainer(**over):
    import swapping_autoencoder_pytorch_b200 as S
    opt = default_options(**dict(TINY, **over))
    torch.manual_seed(0)
    return S.create_optimizer(opt, S.create_model(opt))


def _state(tr):
    """every parameter and every Adam tensor of both groups, copied"""
    out = [p.detach().clone() for p in tr.model.singlegpu_model.parameters()]
    for o in (tr.optimizer_G, tr.optimizer_D):
        st = o._state()
        out += [st.exp_avg.clone(), st.exp_avg_sq.clone(), st.steps.clone()]
    return out


def _bitwise_equal(a, b):
    return len(a) == len(b) and all(x.dtype == y.dtype and torch.equal(x, y) for x, y in zip(a, b))


def test_one_micro_batch_makes_todays_calls(spy, fp64_default):
    tr = _trainer(R1_once_every=1)
    assert tr.opt.micro_batches == 1
    real = rnd(900, 2, 3, 64, 64).clamp(-1, 1)
    tr.train_one_step({"real_A": real}, 0)          # D + R1
    tr.train_one_step({"real_A": real}, 0)          # G
    assert spy.log == [("adam_step", 13, ())] * 3


def _compose(tr, kind, chunks, optimizer):
    """the reference composition of one accumulated update: the trainer's body with step=False on each micro-batch in order,
    the gradients summed in that order, one Adam step reading the sums with grad_scale = 1 / k"""
    body = {"D": tr._discriminator_body, "R1": tr._r1_body, "G": tr._generator_body}[kind]
    params = optimizer.params
    total, outs = None, []
    for chunk in chunks:
        outs.append(body(chunk, step=False))
        g = [None if p.grad is None else p.grad.clone() for p in params]
        total = g if total is None else [None if a is None else a + b for a, b in zip(total, g)]
    optimizer.step(grads=total, grad_scale=1.0 / len(chunks))
    means = {k: torch.stack([o[k].detach().mean() for o in outs]).mean() for k in outs[0] if not k.startswith("_")}
    return means, outs


def test_two_micro_batches_equal_the_composition(spy, fp64_default):
    real = rnd(901, 4, 3, 64, 64).clamp(-1, 1)
    tr = _trainer(R1_once_every=1, micro_batches=2)
    torch.manual_seed(7)
    d = tr.train_one_step({"real_A": real}, 0)      # D + R1
    sp = tr.previous_sp
    g = tr.train_one_step({"real_A": real}, 0)      # G

    ref = _trainer(R1_once_every=1)
    chunks = [real[:2], real[2:]]
    torch.manual_seed(7)
    d_ref, d_outs = _compose(ref, "D", chunks, ref.optimizer_D)
    r1_ref, _ = _compose(ref, "R1", chunks, ref.optimizer_D)
    g_ref, _ = _compose(ref, "G", chunks, ref.optimizer_G)

    assert _bitwise_equal(_state(tr), _state(ref))
    d_ref.update(r1_ref)
    d_ref["D_total"] = sum(v.mean() for v in d_ref.values())
    assert set(d) == set(d_ref) and "D_R1" in d
    for k, v in d_ref.items():
        assert float(d[k]) == float(v), k
    assert set(g) == set(g_ref) and "L1_dist" in g
    for k, v in g_ref.items():
        assert float(g[k]) == float(v), k
    assert sp.shape[0] == 4 and torch.equal(sp, torch.cat([o["_sp"] for o in d_outs]))
    assert tr.model.singlegpu_model.num_discriminator_iters.item() == 1
    # k = 2 makes no bucket call on a CPU device (the sums are formed in torch) and one Adam update per kind
    assert spy.log == [("adam_step", 13, ())] * 6


def test_schedule_counts_updates(spy, fp64_default):
    tr = _trainer(R1_once_every=2, micro_batches=2)
    real = rnd(902, 4, 3, 64, 64).clamp(-1, 1)
    r1 = []
    for _ in range(4):
        out = tr.train_discriminator_one_step(real)
        r1.append("D_R1" in out)
    assert r1 == [False, True, False, True]
    assert tr.discriminator_iter_counter == 4
    assert tr.model.singlegpu_model.num_discriminator_iters.item() == 4
    assert spy.log == [("adam_step", 13, ())] * 6              # 4 D updates, 2 R1 updates


@pytest.mark.parametrize("batch,k", [(6, 2), (4, 3), (4, 0)])
def test_batches_that_do_not_split_raise(spy, fp64_default, batch, k):
    tr = _trainer(micro_batches=k)
    real = rnd(903, batch, 3, 64, 64).clamp(-1, 1)
    with pytest.raises(ValueError):
        tr.train_one_step({"real_A": real}, 0)
    with pytest.raises(ValueError):
        tr.train_generator_one_step(real)
    assert spy.log == []
    assert tr.train_mode_counter == 0 and tr.discriminator_iter_counter == 0


# ---------------------------------------------------------------------------------------------------------------------
# two ranks over gloo: the trainer's bucket path (host branch), one all-reduce per update
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _tiny_trainer(seed, **over):
    import swapping_autoencoder_pytorch_b200 as S
    backend.set_kernels(EmulatedKernels())
    torch.set_default_dtype(torch.float64)
    opt = default_options(**dict(TINY, R1_once_every=1, **over))
    torch.manual_seed(seed)
    model = S.create_model(opt)
    return opt, model, S.create_optimizer(opt, model)


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    opt, model, trainer = _tiny_trainer(100 + rank, micro_batches=2)       # rank 0's parameters are broadcast
    assert trainer.world == 2
    calls = []
    all_reduce = dist.all_reduce

    def counting_all_reduce(t, *a, **kw):
        calls.append(t.numel())
        return all_reduce(t, *a, **kw)
    dist.all_reduce = counting_all_reduce
    try:
        x = model.shard(rnd(904, 8, 3, 64, 64).clamp(-1, 1))
        torch.manual_seed(7)
        trainer.train_one_step({"real_A": x}, 0)          # D + R1
        n_d = len(calls)
        trainer.train_one_step({"real_A": x}, 0)          # G
    finally:
        dist.all_reduce = all_reduce
    sd = {k: v.clone() for k, v in model.singlegpu_model.state_dict().items()}
    torch.save({"sd": sd, "calls": calls, "n_d": n_d}, os.path.join(out, "r%d.pt" % rank))
    dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_two_ranks_one_all_reduce_per_update(tmp_path):
    world = 2
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    r0 = torch.load(os.path.join(tmp_path, "r0.pt"))
    r1 = torch.load(os.path.join(tmp_path, "r1.pt"))
    for k in r0["sd"]:
        assert torch.equal(r0["sd"][k], r1["sd"][k]), "ranks diverged on %s" % k
    assert r0["n_d"] == 2 and len(r0["calls"]) == 3                 # D, R1, G: one all-reduce each
    prev = torch.get_default_dtype()
    try:
        opt, model, trainer = _tiny_trainer(100)                     # rank 0's initialisation
        inner = model.singlegpu_model
        full = rnd(904, 8, 3, 64, 64).clamp(-1, 1)
        ranks = [[full[0:2], full[2:4]], [full[4:6], full[6:8]]]
        c = opt.R1_once_every / (1 + opt.R1_once_every)
        adam_d = torch.optim.Adam(trainer.Dparams, lr=opt.lr * c, betas=(opt.beta1 ** c, opt.beta2 ** c))
        adam_g = torch.optim.Adam(trainer.Gparams, lr=opt.lr, betas=(opt.beta1, opt.beta2))

        def averaged_step(params, frozen, adam, loss_fn, state):
            """every rank starts its micro-batches from the same generator state: replay each rank's sequence from it"""
            trainer.set_requires_grad(frozen, False)
            trainer.set_requires_grad(params, True)
            grads, n = None, 0
            for chunks in ranks:
                torch.set_rng_state(state)
                for chunk in chunks:
                    adam.zero_grad()
                    loss_fn(chunk).backward()
                    g = [None if p.grad is None else p.grad.clone() for p in params]
                    grads = g if grads is None else [a if b is None else a + b for a, b in zip(grads, g)]
                    n += 1
            for p, g in zip(params, grads):
                p.grad = None if g is None else g / n
            adam.step()
            return torch.get_rng_state()

        torch.manual_seed(7)
        s = torch.get_rng_state()
        s = averaged_step(trainer.Dparams, trainer.Gparams, adam_d,
                          lambda x: sum(v.mean() for v in inner(x, command="compute_discriminator_losses")[0].values()), s)
        s = averaged_step(trainer.Dparams, trainer.Gparams, adam_d,
                          lambda x: sum(v.mean() for v in inner(x, command="compute_R1_loss").values()) * opt.R1_once_every, s)
        averaged_step(trainer.Gparams, trainer.Dparams, adam_g,
                      lambda x: sum(v.mean() for v in inner(x, None, None, command="compute_generator_losses")[0].values()), s)
        ref = inner.state_dict()
        worst = max(float((r0["sd"][k].double() - ref[k].double()).abs().max()) for k in ref
                    if ref[k].dtype.is_floating_point and k != "num_discriminator_iters")
        assert worst < 1e-9, worst
        assert int(r0["sd"]["num_discriminator_iters"]) == 1
    finally:
        torch.set_default_dtype(prev)
        backend.set_kernels(None)
