"""CPU: host logic of the training statistics (opt.training_stats; optimizer.TrainingStats) on the kernel emulation.

* statistics off: a D + R1 and a G half-step make exactly the kernel calls they made before the option existed, the
  trainer's and the model's state_dict keys are unchanged and the model has no sink;
* statistics on, fp64, 24 half-steps with one lazy R1 (micro_batches 1 and 2): the window equals a restatement from the
  gradients Adam read (.grad, or the accumulated bucket), the parameters and the moments after every update;
* the score statistics are the logits the model computes, and equal with batch_discriminator_passes on and off;
* a guard-dropped update adds nothing; reset semantics; an empty window is zeros; state_dict does not carry the window;
* two ranks over gloo return identical dictionaries whose score sums are the sums of the ranks' local windows."""
import math
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle.fixtures import TINY, rnd
from swapping_autoencoder_pytorch_b200 import backend, default_options
from swapping_autoencoder_pytorch_b200.optimizer import NONFINITE_KINDS, STATS_NORMS, STATS_SCORES
from tests.cpu_emulation import EmulatedKernels


class StatsKernels(EmulatedKernels):
    """the emulation with the guard's entry points and the three statistics entry points (include/sae_b200.h, ABI 19),
    recording the optimizer's calls"""

    def __init__(self):
        self.log = []

    def adam_step(self, *args, skip=None):
        self.log.append(("adam_step", len(args), () if skip is None else ("skip",)))
        if skip is not None and int(skip.reshape(-1)[0]) != 0:
            return
        return EmulatedKernels.adam_step(self, *args)

    def nonfinite_count(self, tensors, sizes, counts, cache):
        self.log.append(("nonfinite_count", len(tensors), ()))
        for i, t in enumerate(tensors):
            if t is not None:
                c = int((~torch.isfinite(t)).sum())
                counts[i] += c
                counts[-1] += c

    def sumsq(self, tensors, sizes, out, partials, cache, scale=1.0, skip=None):
        self.log.append(("sumsq", len(tensors), float(scale)))
        if skip is not None and int(skip.reshape(-1)[0]) != 0:
            return
        s2 = float(np.float32(scale)) ** 2
        for i, t in enumerate(tensors):
            if t is not None:
                out[i] += s2 * float((t.double() ** 2).sum())

    def adam_norms(self, params, grads, offsets, sizes, exp_avg, exp_avg_sq, steps, lr, beta1, beta2, eps, weight_out,
                   update_out, updates, partials, cache, skip=None):
        self.log.append(("adam_norms", len(params), ()))
        if skip is not None and int(skip.reshape(-1)[0]) != 0:
            return
        for i, p in enumerate(params):
            weight_out[i] += float((p.double() ** 2).sum())
            if grads[i] is None:
                continue
            o, n, t = int(offsets[i]), int(sizes[i]), float(steps[i])
            m, v = exp_avg[o:o + n].double(), exp_avg_sq[o:o + n].double()
            d = lr / (1 - beta1 ** t) * m / (v.sqrt() / (1 - beta2 ** t) ** 0.5 + eps)
            update_out[i] += float((d ** 2).sum())
        if updates is not None:
            updates += 1

    def score_stats(self, x, acc):
        self.log.append(("score_stats", tuple(x.shape), ()))
        fin = torch.isfinite(x)
        acc[0] += float(x[fin].double().sum())
        acc[1] += float(torch.sign(x[fin]).double().sum())
        acc[2] += int(fin.sum())
        acc[3] += int((~fin).sum())


@pytest.fixture
def kern():
    prev = backend.set_kernels(StatsKernels())
    yield backend.kernels()
    backend.set_kernels(prev)


def _trainer(**over):
    import swapping_autoencoder_pytorch_b200 as S
    opt = default_options(**dict(TINY, **over))
    torch.manual_seed(0)
    return S.create_optimizer(opt, S.create_model(opt))


def _names(tr, params):
    names = {id(p): n for n, p in tr.model.singlegpu_model.named_parameters()}
    return [names[id(p)] for p in params]


def _restate(tr):
    """wrap tr.exchange_and_step so that every update adds to a plain-Python window: the gradients Adam read (.grad, or the
    accumulated bucket views with scale 1 / k), the parameters and Adam's step restated from the moments after the update"""
    exp = {k: {"updates": 0, **{s: {} for s in STATS_NORMS}} for k in NONFINITE_KINDS}
    orig = tr.exchange_and_step

    def wrapped(optimizer, params, kind=None, micro_batches=1, images=None):
        if micro_batches > 1:
            box, real = {}, tr.model.reduce_accumulated

            def grab():
                box["g"] = real()
                return box["g"]
            tr.model.reduce_accumulated = grab
            try:
                orig(optimizer, params, kind=kind, micro_batches=micro_batches, images=images)
            finally:
                del tr.model.reduce_accumulated
            grads, scale = [None if g is None else g.detach().clone() for g in box["g"]], 1.0 / micro_batches
        else:
            orig(optimizer, params, kind=kind, micro_batches=micro_batches, images=images)
            grads, scale = [p.grad for p in params], 1.0
        e = exp[kind]
        e["updates"] += 1
        st, g = optimizer._state(), optimizer.param_groups[0]
        b1, b2 = g["betas"]
        for i, (name, p) in enumerate(zip(_names(tr, params), params)):
            add = {"weight_norm": float((p.detach().double() ** 2).sum()), "grad_norm": 0.0, "update_norm": 0.0}
            if grads[i] is not None:
                add["grad_norm"] = scale ** 2 * float((grads[i].double() ** 2).sum())
                o, n, t = optimizer._offsets[i], optimizer._sizes[i], float(st.steps[i])
                m, v = st.exp_avg[o:o + n].double(), st.exp_avg_sq[o:o + n].double()
                d = g["lr"] / (1 - b1 ** t) * m / (v.sqrt() / (1 - b2 ** t) ** 0.5 + g["eps"])
                add["update_norm"] = float((d ** 2).sum())
            for s, v in add.items():
                e[s][name] = e[s].get(name, 0.0) + v
    tr.exchange_and_step = wrapped
    return exp


def _close(a, b, rel=1e-12):
    return abs(a - b) <= rel * max(abs(a), abs(b), 1e-300)


def test_off_makes_todays_calls_and_keys(kern, fp64_default):
    tr = _trainer(R1_once_every=1)
    assert tr.opt.training_stats is False and tr.stats is None and tr.stats_key() == ()
    assert tr.model.singlegpu_model.score_sink is None
    real = rnd(920, 2, 3, 64, 64).clamp(-1, 1)
    tr.train_one_step({"real_A": real}, 0)          # D + R1
    tr.train_one_step({"real_A": real}, 0)          # G
    assert kern.log == [("adam_step", 13, ())] * 3
    assert sorted(tr.state_dict()) == ["discriminator_iter_counter", "optimizer_D", "optimizer_G", "train_mode_counter"]
    with pytest.raises(RuntimeError):
        tr.training_stats()
    on = _trainer(training_stats=True)
    assert sorted(on.state_dict()) == sorted(tr.state_dict())                     # the window is not saved
    assert list(tr.model.singlegpu_model.state_dict()) == list(on.model.singlegpu_model.state_dict())
    assert on.stats_key() == (("stats",),)


@pytest.mark.parametrize("micro_batches", [1, 2])
def test_window_matches_a_restatement(kern, fp64_default, micro_batches):
    tr = _trainer(training_stats=True, R1_once_every=8, micro_batches=micro_batches)
    exp = _restate(tr)
    real = rnd(921, 4, 3, 64, 64).clamp(-1, 1)
    for _ in range(24):                                   # 12 D, 12 G, one R1 (the 8th D update)
        tr.train_one_step({"real_A": real}, 0)
    got = tr.training_stats(reset=False, per_tensor=True)
    assert [got[k + "/updates"] for k in NONFINITE_KINDS] == [12, 1, 12]
    assert [exp[k]["updates"] for k in NONFINITE_KINDS] == [12, 1, 12]
    calls = [e for e in kern.log if e[0] == "sumsq"]
    assert sorted(calls) == sorted([("sumsq", len(tr.Dparams), 1.0 / micro_batches)] * 13
                                   + [("sumsq", len(tr.Gparams), 1.0 / micro_batches)] * 12)
    for kind in NONFINITE_KINDS:
        u = exp[kind]["updates"]
        for stat in STATS_NORMS:
            per = exp[kind][stat]
            assert _close(got["%s/%s" % (kind, stat)], math.sqrt(sum(per.values()) / u)), (kind, stat)
            for name, v in per.items():
                assert _close(got["per_tensor"][name]["%s/%s" % (kind, stat)], math.sqrt(v / u)), (kind, stat, name)
            assert got["%s/%s" % (kind, stat)] > 0.0
    # R1 leaves the last bias of D without a gradient: no gradient and no step there, but a weight norm
    last = _names(tr, tr.Dparams)
    zero = [n for n in last if got["per_tensor"][n]["R1/grad_norm"] == 0.0]
    assert zero and all(got["per_tensor"][n]["R1/update_norm"] == 0.0 and got["per_tensor"][n]["R1/weight_norm"] > 0.0
                        for n in zero)
    # the score statistics: one call per logit tensor and micro-batch
    assert sum(1 for e in kern.log if e[0] == "score_stats") == (12 * 5 + 12 * 3) * micro_batches
    for kind, name in STATS_SCORES:
        assert got["%s/scores/%s/nonfinite" % (kind, name)] == 0
        assert -1.0 <= got["%s/signs/%s" % (kind, name)] <= 1.0 and got["%s/scores/%s" % (kind, name)] != 0.0


def test_scores_are_the_model_logits(kern, fp64_default):
    tr = _trainer(training_stats=True)
    inner = tr.model.singlegpu_model
    seen = []
    sink = inner.score_sink
    inner.score_sink = lambda kind, name, x: (seen.append((kind, name, x.detach().clone())), sink(kind, name, x))
    real = rnd(922, 2, 3, 64, 64).clamp(-1, 1)
    with torch.no_grad():
        pred_real = inner.D(real)                         # D draws nothing: the D step sees the same logits
    for _ in range(4):
        tr.train_one_step({"real_A": real}, 0)            # D, G, D, G
    got = tr.training_stats()
    assert [(k, n) for k, n, _ in seen[:8]] == list(STATS_SCORES)
    assert torch.equal(seen[0][2], pred_real)
    for kind, name in STATS_SCORES:
        xs = torch.cat([x.reshape(-1) for k, n, x in seen if (k, n) == (kind, name)])
        assert _close(got["%s/scores/%s" % (kind, name)], float(xs.mean()), 1e-12)
        assert _close(got["%s/signs/%s" % (kind, name)], float(torch.sign(xs).mean()), 1e-12)
    assert tr.training_stats() == {k: (0 if isinstance(v, int) else 0.0) for k, v in got.items()}


def test_batched_discriminator_passes_give_the_same_scores(kern, fp64_default):
    real = rnd(923, 4, 3, 64, 64).clamp(-1, 1)
    out = []
    for batched in (True, False):
        tr = _trainer(training_stats=True, batch_discriminator_passes=batched)
        torch.manual_seed(5)
        for _ in range(4):
            tr.train_one_step({"real_A": real}, 0)
        out.append(tr.training_stats())
    a, b = out
    assert sorted(a) == sorted(b)
    for k in a:
        assert abs(a[k] - b[k]) <= 1e-9 * max(1.0, abs(a[k])), (k, a[k], b[k])


def test_dropped_update_adds_nothing(kern, fp64_default):
    tr = _trainer(training_stats=True, skip_nonfinite_steps=True)
    real = rnd(924, 2, 3, 64, 64).clamp(-1, 1)
    for _ in range(2):
        tr.train_generator_one_step(real)
    norms_at = tr.stats._scores_at
    before = tr.stats.window[:norms_at].clone()
    p = next(p for n, p in tr.model.singlegpu_model.named_parameters() if n.startswith("G."))
    handle = p.register_post_accumulate_grad_hook(lambda q: q.grad.view(-1).__setitem__(0, float("nan")))
    tr.train_generator_one_step(real)
    handle.remove()
    assert tr.nonfinite_steps()["G"] == 1
    assert torch.equal(tr.stats.window[:norms_at], before)                      # norms and the update count untouched
    assert [e[0] for e in kern.log[-3:]] == ["adam_step", "sumsq", "adam_norms"]      # issued, dropped on the device
    got = tr.training_stats()
    assert got["G/updates"] == 2


def test_reset_and_empty_window(kern, fp64_default):
    tr = _trainer(training_stats=True)
    empty = tr.training_stats(per_tensor=True)
    assert all(v == 0 for k, v in empty.items() if k != "per_tensor")
    assert all(v == 0.0 for d in empty["per_tensor"].values() for v in d.values())
    assert set(empty["per_tensor"]) == set(_names(tr, tr.Dparams)) | set(_names(tr, tr.Gparams))
    assert all(not (isinstance(v, float) and math.isnan(v)) for v in empty.values() if not isinstance(v, dict))
    real = rnd(925, 2, 3, 64, 64).clamp(-1, 1)
    tr.train_one_step({"real_A": real}, 0)
    a = tr.training_stats(reset=False)
    b = tr.training_stats(reset=False)
    assert a == b and a["D/updates"] == 1
    c = tr.training_stats()                                                      # reads, then clears
    assert c == a
    assert tr.training_stats() == {k: (0 if isinstance(v, int) else 0.0) for k, v in a.items()}
    tr.train_one_step({"real_A": real}, 0)
    d = tr.training_stats()
    assert d["G/updates"] == 1 and d["D/updates"] == 0
    # a loaded optimizer starts an empty window
    fresh = _trainer(training_stats=True)
    fresh.load_state_dict(tr.state_dict())
    assert float(fresh.stats.window.abs().sum()) == 0.0


# ---------------------------------------------------------------------------------------------------------------------
# two ranks over gloo
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
    backend.set_kernels(StatsKernels())
    torch.set_default_dtype(torch.float64)
    opt = default_options(**dict(TINY, R1_once_every=1, training_stats=True))
    torch.manual_seed(100 + rank)                                # rank 0's parameters are broadcast
    model = S.create_model(opt)
    trainer = S.create_optimizer(opt, model)
    x = model.shard(rnd(926, 4, 3, 64, 64).clamp(-1, 1))
    torch.manual_seed(7 + rank)                                  # each rank draws its own noise
    for _ in range(4):
        trainer.train_one_step({"real_A": x}, 0)                 # D + R1, G, D + R1, G
    local = trainer.stats.window.clone()
    got = trainer.training_stats(per_tensor=True)
    torch.save({"local": local, "scores_at": trainer.stats._scores_at, "got": got,
                "after": trainer.stats.window.clone()}, os.path.join(out, "s%d.pt" % rank))
    dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_two_ranks_return_identical_dictionaries(tmp_path):
    world = 2
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    s0 = torch.load(os.path.join(tmp_path, "s0.pt"))
    s1 = torch.load(os.path.join(tmp_path, "s1.pt"))
    assert s0["got"] == s1["got"]
    at = s0["scores_at"]
    assert torch.equal(s0["local"][:at], s1["local"][:at])              # the norms: the same on every rank already
    assert not torch.equal(s0["local"][at:], s1["local"][at:])          # the scores: local
    both = (s0["local"][at:] + s1["local"][at:]).view(-1, 4).tolist()
    for (kind, name), (s, sign, finite, bad) in zip(STATS_SCORES, both):
        assert _close(s0["got"]["%s/scores/%s" % (kind, name)], s / finite)
        assert _close(s0["got"]["%s/signs/%s" % (kind, name)], sign / finite, 1e-15) or sign == 0
        assert s0["got"]["%s/scores/%s/nonfinite" % (kind, name)] == bad == 0
    assert s0["got"]["D/updates"] == 2 and s0["got"]["R1/updates"] == 2 and s0["got"]["G/updates"] == 2
    assert float(s0["after"].abs().sum()) == 0.0 and float(s1["after"].abs().sum()) == 0.0
