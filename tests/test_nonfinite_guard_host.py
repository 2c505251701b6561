"""CPU: host logic of the skip-on-non-finite guard (opt.skip_nonfinite_steps) on the kernel emulation.

* guard off: ``MultiTensorAdam.step`` and a training half-step make exactly the kernel calls they made before the guard
  existed (one ``adam_step`` with its thirteen positional arguments, no ``nonfinite_count``);
* guard on: a half-step whose gradients hold an Inf or a NaN leaves parameters and Adam state bitwise unchanged while the
  schedule counters advance, ``nonfinite_steps`` / ``nonfinite_report`` say which kind and which tensor, the next clean
  half-step updates, and the skip counters round-trip through ``state_dict`` (saved only with the guard on)."""
import pytest
import torch

from oracle.fixtures import TINY, rnd
from swapping_autoencoder_pytorch_b200 import backend, default_options
from swapping_autoencoder_pytorch_b200.optimizer import MultiTensorAdam
from tests.cpu_emulation import EmulatedKernels


class SpyKernels(EmulatedKernels):
    """the emulation, recording (method, number of positional arguments, keyword names) of the optimizer's calls"""

    def __init__(self):
        self.log = []

    def adam_step(self, *args, **kw):
        self.log.append(("adam_step", len(args), tuple(sorted(kw))))
        return super().adam_step(*args, **kw)


class GuardedKernels(SpyKernels):
    """the emulation with the guard's two entry points (include/sae_b200.h: sae_nonfinite_count, sae_adam_step_guarded)"""

    def nonfinite_count(self, tensors, sizes, counts, cache):
        self.log.append(("nonfinite_count", len(tensors), ()))
        for i, t in enumerate(tensors):
            if t is not None:
                assert t.numel() == int(sizes[i])
                c = int((~torch.isfinite(t)).sum())
                counts[i] += c
                counts[-1] += c

    def adam_step(self, *args, skip=None):
        self.log.append(("adam_step", len(args), () if skip is None else ("skip",)))
        if skip is not None and int(skip.reshape(-1)[0]) != 0:
            return
        return EmulatedKernels.adam_step(self, *args)


@pytest.fixture
def spy():
    prev = backend.set_kernels(SpyKernels())
    yield backend.kernels()
    backend.set_kernels(prev)


@pytest.fixture
def guarded():
    prev = backend.set_kernels(GuardedKernels())
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
    return all(x.dtype == y.dtype and torch.equal(x, y) for x, y in zip(a, b))


def test_guard_off_adam_makes_todays_calls(spy, fp64_default):
    params = [rnd(1, 5, 3).requires_grad_(), rnd(2, 8).requires_grad_()]
    opt = MultiTensorAdam(params, lr=0.01, betas=(0.0, 0.99))
    for p, s in zip(params, (3, 4)):
        p.grad = rnd(s, *p.shape)
    opt.step()
    opt.step(grads=[rnd(5, 5, 3), None], grad_scale=0.5)
    assert spy.log == [("adam_step", 13, ())] * 2


def test_guard_off_half_steps_make_todays_calls(spy, fp64_default):
    tr = _trainer(R1_once_every=1)
    real = rnd(900, 2, 3, 64, 64).clamp(-1, 1)
    tr.train_one_step({"real_A": real}, 0)          # D + R1
    tr.train_one_step({"real_A": real}, 0)          # G
    assert spy.log == [("adam_step", 13, ())] * 3
    assert "nonfinite_steps" not in tr.state_dict()
    assert tr.nonfinite_steps() == {"D": 0, "R1": 0, "G": 0} and tr.nonfinite_report("G") == {}


@pytest.mark.parametrize("kind,net,value", [("D", "Dpatch", float("inf")), ("R1", "D", float("nan")),
                                            ("G", "E", float("-inf"))])
def test_skip_report_and_state_dict(guarded, fp64_default, kind, net, value):
    every = 2 if kind == "R1" else 4             # D, G, D (+ R1 at every = 2), G: no R1 except where it is poisoned
    tr = _trainer(R1_once_every=every, skip_nonfinite_steps=True)
    real = rnd(900, 2, 3, 64, 64).clamp(-1, 1)
    for _ in range(3 if kind == "G" else 2):
        tr.train_one_step({"real_A": real}, 0)
    before = _state(tr)
    counters = (tr.train_mode_counter, tr.discriminator_iter_counter)
    # a post-accumulate-grad hook writes `value` into element 0 of the gradient of the first tensor of network `net`; for R1
    # only in the R1 backward, so that the D update of the same half-step is clean and applied
    name, p = next((n, p) for n, p in tr.model.singlegpu_model.named_parameters() if n.startswith(net + "."))
    armed, after_d = [kind != "R1"], []

    def hook(param):
        if armed[0]:
            with torch.no_grad():
                param.grad.view(-1)[0] = value
    frozen = not p.requires_grad            # the trainer toggles requires_grad per half-step; a hook needs it on
    handle = p.requires_grad_(True).register_post_accumulate_grad_hook(hook)
    p.requires_grad_(not frozen)
    if kind == "R1":
        def r1_body(images, step=True):
            after_d.append(_state(tr))
            armed[0] = True
            return type(tr)._r1_body(tr, images, step)
        tr._r1_body = r1_body
    out = tr.train_one_step({"real_A": real}, 0)
    handle.remove()
    tr.__dict__.pop("_r1_body", None)
    assert (tr.train_mode_counter, tr.discriminator_iter_counter) != counters      # the schedule advanced
    if kind == "R1":
        assert "D_R1" in out and after_d
        assert _bitwise_equal(_state(tr), after_d[0])
        assert not _bitwise_equal(after_d[0], before)          # the clean D update of the same half-step ran
    else:
        assert ("D_R1" in out) is False
        assert _bitwise_equal(_state(tr), before)
    assert tr.nonfinite_steps() == {k: int(k == kind) for k in ("D", "R1", "G")}
    assert tr.nonfinite_report(kind) == {name: 1}
    assert all(tr.nonfinite_report(k) == {} for k in ("D", "R1", "G") if k != kind)

    sd = tr.state_dict()
    assert sd["nonfinite_steps"] == tr.nonfinite_steps()
    tr2 = _trainer(R1_once_every=every, skip_nonfinite_steps=True)
    tr2.load_state_dict(sd)
    assert tr2.nonfinite_steps() == tr.nonfinite_steps()
    tr.opt.skip_nonfinite_steps = False
    assert "nonfinite_steps" not in tr.state_dict()
    tr.opt.skip_nonfinite_steps = True

    # the next clean half-steps update normally and leave the counters alone
    for _ in range(2):
        before = _state(tr)
        tr.train_one_step({"real_A": real}, 0)
        assert not _bitwise_equal(_state(tr), before)
    assert tr.nonfinite_steps() == {k: int(k == kind) for k in ("D", "R1", "G")}
    assert ("nonfinite_count", len(tr.Gparams), ()) in guarded.log
    assert all(entry[2] == ("skip",) for entry in guarded.log if entry[0] == "adam_step")
