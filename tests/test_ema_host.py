"""CPU: host logic of the weight average (opt.ema_kimg; optimizer.ParameterEMA) on the kernel emulation.

* average off: a D + R1 and a G half-step make exactly the kernel calls they made before the option existed, and the
  trainer's and the model's state_dict keys are unchanged;
* average on, fp64, 40 G updates through the ramp into the plateau: beta and the shadow follow a plain-Python restatement of
  the schedule applied to the parameters after each G update, and t counts G updates only;
* a G update the guard drops leaves shadow and t bitwise unchanged; micro_batches = 2 makes one averaging update per update;
* state_dict round trip: a resumed run matches the uninterrupted one bitwise; a state without "ema" keeps the shadow;
* trainer.save writes <N>k_ema_checkpoint.pth with the reference's key / shape / dtype set; model.load takes it;
* two ranks over gloo keep identical shadows and only rank 0 writes files."""
import json
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle.fixtures import GOLDEN_DIR, TINY, rnd
from swapping_autoencoder_pytorch_b200 import backend, default_options
from tests.cpu_emulation import EmulatedKernels


def _f32(x):
    """the value a C float argument carries"""
    return float(np.float32(x))


def restated_beta(t, batch_images, half_life_images, rampup):
    """INTEGRATION §2f: h = half-life (with a ramp: min(h, t * B * rampup)), beta = 0.5^(B / max(h, 1e-8)) in fp64,
    rounded to fp32 once"""
    b, h, r = _f32(batch_images), _f32(half_life_images), _f32(rampup)
    if r > 0:
        h = min(h, t * b * r)
    return _f32(0.5 ** (b / max(h, 1e-8)))


class EmaKernels(EmulatedKernels):
    """the emulation with the guard's entry points and sae_ema_update (include/sae_b200.h), recording the optimizer's calls"""

    def __init__(self):
        self.log = []
        self.betas = []

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

    def ema_update(self, params, offsets, sizes, shadow, updates, batch_images, half_life_images, rampup, cache, skip=None):
        self.log.append(("ema_update", len(params), batch_images))
        if skip is not None and int(skip.reshape(-1)[0]) != 0:
            return
        t = int(updates[0])
        # the kernel's own arithmetic: fp64 from the counter, one rounding to fp32
        h = float(np.float32(half_life_images))
        if np.float32(rampup) > 0:
            h = min(h, float(t) * float(np.float32(batch_images)) * float(np.float32(rampup)))
        beta = float(np.float32(np.exp2(-float(np.float32(batch_images)) / max(h, 1e-8))))
        self.betas.append(beta)
        with torch.no_grad():
            for i, p in enumerate(params):
                if p is None:
                    continue
                o, n = int(offsets[i]), int(sizes[i])
                s = shadow[o:o + n].view_as(p)
                s.copy_(torch.addcmul(p, s - p, torch.tensor(beta, dtype=p.dtype)))
            updates += 1


@pytest.fixture
def kern():
    prev = backend.set_kernels(EmaKernels())
    yield backend.kernels()
    backend.set_kernels(prev)


def _trainer(**over):
    import swapping_autoencoder_pytorch_b200 as S
    opt = default_options(**dict(TINY, **over))
    torch.manual_seed(0)
    return S.create_optimizer(opt, S.create_model(opt))


def _bitwise_equal(a, b):
    return len(a) == len(b) and all(x.dtype == y.dtype and torch.equal(x, y) for x, y in zip(a, b))


def _shadow(tr):
    return [v.detach().clone() for v in tr.ema.averaged()] + [tr.ema.updates.clone()]


def test_off_makes_todays_calls_and_keys(kern, fp64_default):
    tr = _trainer(R1_once_every=1)
    assert tr.opt.ema_kimg == 0.0 and tr.ema is None and tr.ema_key() == ()
    real = rnd(900, 2, 3, 64, 64).clamp(-1, 1)
    tr.train_one_step({"real_A": real}, 0)          # D + R1
    tr.train_one_step({"real_A": real}, 0)          # G
    assert kern.log == [("adam_step", 13, ())] * 3
    assert sorted(tr.state_dict()) == ["discriminator_iter_counter", "optimizer_D", "optimizer_G", "train_mode_counter"]
    on = _trainer(ema_kimg=1.0)
    assert list(tr.model.singlegpu_model.state_dict()) == list(on.model.singlegpu_model.state_dict())
    with pytest.raises(RuntimeError):
        tr.ema_state_dict()


def test_schedule_and_shadow_follow_the_recurrence(kern, fp64_default):
    # B = 2 images; half-life 2 images; the ramp (0.1 t images) reaches it at t = 20: 40 updates cover ramp and plateau
    tr = _trainer(ema_kimg=0.002, ema_rampup=0.05)
    real = rnd(905, 2, 3, 64, 64).clamp(-1, 1)
    shadow = [p.detach().clone() for p in tr.Gparams]
    assert _bitwise_equal(_shadow(tr)[:-1], shadow)              # the construction-time copy
    betas, n_g = [], 0
    for i in range(48):
        if i % 6 == 5:
            tr.train_discriminator_one_step(real)                 # D (and R1) updates do not move the average
            continue
        tr.train_generator_one_step(real)
        beta = restated_beta(n_g, 2, 2.0, 0.05)
        betas.append(beta)
        shadow = [p.detach() + beta * (s - p.detach()) for s, p in zip(shadow, tr.Gparams)]
        n_g += 1
    assert n_g == 40 and int(tr.ema.updates) == 40
    assert betas[0] == 0.0 and betas[-1] == 0.5 and 0.0 < betas[10] < 0.5
    assert kern.betas == betas
    worst = max(float((a - b).abs().max()) for a, b in zip(_shadow(tr)[:-1], shadow))
    assert worst < 1e-12, worst
    assert not _bitwise_equal(_shadow(tr)[:-1], [p.detach() for p in tr.Gparams])
    assert [e[2] for e in kern.log if e[0] == "ema_update"] == [2.0] * 40


def test_dropped_g_update_drops_the_average(kern, fp64_default):
    tr = _trainer(ema_kimg=0.01, skip_nonfinite_steps=True)
    real = rnd(906, 2, 3, 64, 64).clamp(-1, 1)
    for _ in range(3):
        tr.train_generator_one_step(real)
    before = _shadow(tr)
    p = next(p for n, p in tr.model.singlegpu_model.named_parameters() if n.startswith("E."))
    handle = p.register_post_accumulate_grad_hook(lambda q: q.grad.view(-1).__setitem__(0, float("nan")))
    tr.train_generator_one_step(real)
    handle.remove()
    assert tr.nonfinite_steps()["G"] == 1
    assert _bitwise_equal(_shadow(tr), before) and int(tr.ema.updates) == 3
    assert kern.log[-1] == ("ema_update", len(tr.Gparams), 2.0)           # issued, and dropped on the device
    tr.train_generator_one_step(real)
    assert int(tr.ema.updates) == 4 and not _bitwise_equal(_shadow(tr)[:-1], before[:-1])


def test_micro_batches_make_one_averaging_update(kern, fp64_default):
    tr = _trainer(ema_kimg=0.01, micro_batches=2)
    real = rnd(907, 4, 3, 64, 64).clamp(-1, 1)
    for _ in range(4):
        tr.train_one_step({"real_A": real}, 0)                   # D, G, D, G
    assert int(tr.ema.updates) == 2
    assert [e for e in kern.log if e[0] == "ema_update"] == [("ema_update", len(tr.Gparams), 4.0)] * 2


def _run(tr, real, n):
    for _ in range(n):
        tr.train_one_step({"real_A": real}, 0)


def test_state_dict_round_trip_continues_bitwise(kern):
    # fp32, the dtype of the Adam moments a fresh trainer restores into
    real = rnd(908, 2, 3, 64, 64).clamp(-1, 1).float()
    a = _trainer(ema_kimg=0.005, R1_once_every=2)
    torch.manual_seed(3)
    _run(a, real, 5)
    sd, model_sd, rng = a.state_dict(), {k: v.clone() for k, v in a.model.singlegpu_model.state_dict().items()}, \
        torch.get_rng_state()
    assert set(sd["ema"]) == {"shadow", "t"} and sd["ema"]["t"] == 2
    assert list(sd["ema"]["shadow"]) == a.ema.names and a.ema.names[0].startswith("G.") and a.ema.names[-1].startswith("E.")
    _run(a, real, 5)

    import swapping_autoencoder_pytorch_b200 as S
    opt = default_options(**dict(TINY, ema_kimg=0.005, R1_once_every=2))
    torch.manual_seed(99)                                        # other initial weights: the shadow must come from sd
    b = S.create_optimizer(opt, S.create_model(opt))
    kept = _shadow(b)
    b.load_state_dict({k: v for k, v in sd.items() if k != "ema"})
    assert _bitwise_equal(_shadow(b), kept)                      # no "ema": the construction-time copy stays
    b.model.singlegpu_model.load_state_dict(model_sd)
    b.load_state_dict(sd)
    torch.set_rng_state(rng)
    _run(b, real, 5)
    assert _bitwise_equal(_shadow(a), _shadow(b)) and int(b.ema.updates) == 5
    assert _bitwise_equal(list(a.model.singlegpu_model.state_dict().values()),
                          list(b.model.singlegpu_model.state_dict().values()))


def test_saved_ema_checkpoint_is_a_reference_checkpoint(kern, tmp_path):
    contract = json.load(open(os.path.join(GOLDEN_DIR, "state_dict_contract.json")))["tiny"]
    tr = _trainer(ema_kimg=0.005, checkpoints_dir=str(tmp_path), name="ema")
    real = rnd(909, 2, 3, 64, 64).clamp(-1, 1).float()
    _run(tr, real, 4)
    tr.save(5000)
    d = os.path.join(str(tmp_path), "ema")
    assert sorted(os.listdir(d)) == ["5k_checkpoint.pth", "5k_ema_checkpoint.pth", "5k_optimizer.pth",
                                     "latest_checkpoint.pth", "latest_ema_checkpoint.pth", "latest_optimizer.pth"]
    assert os.readlink(os.path.join(d, "latest_ema_checkpoint.pth")) == "5k_ema_checkpoint.pth"
    ckpt = torch.load(os.path.join(d, "latest_ema_checkpoint.pth"))
    assert {k: [list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in ckpt.items()} == contract
    assert "ema" in torch.load(os.path.join(d, "5k_optimizer.pth"))

    import swapping_autoencoder_pytorch_b200 as S
    torch.manual_seed(42)
    fresh = S.create_model(default_options(**dict(TINY, checkpoints_dir=str(tmp_path), name="ema",
                                                   resume_iter="5k_ema"))).singlegpu_model
    assert fresh.load()
    own = fresh.state_dict()
    live = tr.model.singlegpu_model.state_dict()
    averaged = dict(zip(tr.ema.names, tr.ema.averaged()))
    assert set(averaged) == {k for k in own if k.startswith(("E.", "G."))} - {k for k, _ in fresh.named_buffers()}
    for k, v in own.items():
        want = averaged[k] if k in averaged else live[k]
        assert torch.equal(v, want), k
    assert any(not torch.equal(averaged[k], live[k]) for k in averaged)


def test_no_ema_file_when_off(kern, tmp_path):
    tr = _trainer(checkpoints_dir=str(tmp_path), name="plain")
    tr.save(1000)
    assert sorted(os.listdir(os.path.join(str(tmp_path), "plain"))) == [
        "1k_checkpoint.pth", "1k_optimizer.pth", "latest_checkpoint.pth", "latest_optimizer.pth"]


@pytest.mark.parametrize("over", [dict(ema_kimg=-1.0), dict(ema_kimg=1.0, ema_rampup=-0.1), dict(ema_kimg=float("nan"))])
def test_bad_settings_raise(kern, over):
    with pytest.raises(ValueError):
        _trainer(**over)


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
    backend.set_kernels(EmaKernels())
    torch.set_default_dtype(torch.float64)
    opt = default_options(**dict(TINY, R1_once_every=1, ema_kimg=0.004, checkpoints_dir=os.path.join(out, "r%d" % rank),
                                 name="ema"))
    torch.manual_seed(100 + rank)                                # rank 0's parameters are broadcast
    model = S.create_model(opt)
    trainer = S.create_optimizer(opt, model)
    x = model.shard(rnd(910, 4, 3, 64, 64).clamp(-1, 1))
    torch.manual_seed(7 + rank)                                  # each rank draws its own noise
    for _ in range(4):
        trainer.train_one_step({"real_A": x}, 0)                 # D + R1, G, D + R1, G
    trainer.save(2000)
    calls = [e for e in backend.kernels().log if e[0] == "ema_update"]
    torch.save({"shadow": _shadow(trainer), "calls": calls}, os.path.join(out, "s%d.pt" % rank))
    dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_two_ranks_keep_identical_shadows(tmp_path):
    world = 2
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    s0 = torch.load(os.path.join(tmp_path, "s0.pt"))
    s1 = torch.load(os.path.join(tmp_path, "s1.pt"))
    assert _bitwise_equal(s0["shadow"], s1["shadow"]) and int(s0["shadow"][-1]) == 2
    assert [c[2] for c in s0["calls"]] == [4.0, 4.0]                 # 2 images per rank, 2 ranks
    assert "latest_ema_checkpoint.pth" in os.listdir(os.path.join(tmp_path, "r0", "ema"))
    assert not os.path.exists(os.path.join(tmp_path, "r1"))
