"""GPU (H100): the skip-on-non-finite guard (opt.skip_nonfinite_steps; sae_nonfinite_count, sae_adam_step_guarded).

* the scan against torch.isfinite, exact counts: float4 body and scalar tail, a misaligned view, null entries and empty
  tensors, NaN / +Inf / -Inf at the edges, +-FLT_MAX / denormals / -0.0 (finite), one tensor of more than 2^31 elements;
* the guarded Adam: with *skip == 0 bitwise equal to sae_adam_step on every path, with *skip != 0 nothing written;
* D, D + R1 and G half-steps, eager and replayed, TF32 and fp32, deterministic mode: a post-accumulate-grad hook poisons one
  element of one gradient; the update of exactly that half-step is dropped (bitwise), counted and reported, and the next clean
  half-step updates.  A batch with one NaN pixel is skipped too;
* finite training is untouched: in deterministic mode a D, G, D + R1, G, ... run with the guard on is bitwise the run with it
  off (losses, gradients, parameters, moments, step counts), eager and replayed; toggling the guard captures new graphs and
  toggling it back replays the old ones."""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle.fixtures import TINY
from swapping_autoencoder_pytorch_b200 import _lib, backend, default_options

pytestmark = pytest.mark.gpu
DEV = "cuda"
FLT_MAX = float(np.finfo(np.float32).max)


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _table(ts):
    return torch.tensor([0 if t is None else t.data_ptr() for t in ts], dtype=torch.int64, device=DEV)


def _scan(ts):
    """sae_nonfinite_count over the tensors ts (None: a null entry) -> counts [n + 1] on the host"""
    counts = torch.zeros(len(ts) + 1, dtype=torch.int64, device=DEV)
    sizes = torch.tensor([0 if t is None else t.numel() for t in ts], dtype=torch.int64, device=DEV)
    tab = _table(ts)
    _lib.check(_lib.load().sae_nonfinite_count(_p(tab), _p(sizes), len(ts), _p(counts), _stream()), "sae_nonfinite_count")
    return counts.tolist()


def _expected(ts):
    c = [0 if t is None else int((~torch.isfinite(t)).sum()) for t in ts]
    return c + [sum(c)]


# ------------------------------------------------------------------------------------------------ scan kernel
def test_scan_matches_isfinite_exactly():
    g = torch.Generator(DEV).manual_seed(3)
    ts = []
    for size in (4096, 4097, 4098, 4099, 1 << 20, (1 << 20) + 3, 1, 2, 3, 4, 0):      # float4 body, scalar tail, tiny, empty
        ts.append(torch.randn(size, device=DEV, generator=g))
    base = torch.randn(5001, device=DEV, generator=g)
    ts.append(base[1:])                                   # storage offset 1: the unaligned, element-by-element loop
    ts.append(base[1:4097])                               # unaligned with a multiple-of-4 size
    ts.insert(3, None)
    ts.append(None)
    specials = (float("nan"), float("inf"), float("-inf"))
    for i, t in enumerate(ts):
        if t is None or t.numel() == 0:
            continue
        n = t.numel()
        t[0] = specials[i % 3]                            # first element
        t[n - 1] = specials[(i + 1) % 3]                  # last element (inside the scalar tail when n % 4 != 0)
        if n >= 8:
            t[n - 2] = specials[(i + 2) % 3]
            t[n // 2] = FLT_MAX
            t[n // 2 + 1] = -FLT_MAX
            t[n // 2 + 2] = 1e-40                        # denormal
            t[n // 2 + 3] = -0.0
            t[n // 3] = -1e-45
        if n > 64:
            idx = torch.randint(0, n, (n // 97 + 1,), device=DEV, generator=g)
            t[idx] = torch.tensor(specials, device=DEV)[idx % 3]
    got, want = _scan(ts), _expected(ts)
    assert got == want
    assert got[-1] > 0 and got[3] == 0
    # finite-only values count nothing
    fin = torch.tensor([FLT_MAX, -FLT_MAX, 1e-40, -1e-40, -0.0, 0.0, 1.0, -1e-45], device=DEV)
    assert _scan([fin, fin[1:], fin[:7]]) == [0, 0, 0, 0]


def test_scan_of_a_tensor_beyond_2_31_elements():
    n = (1 << 31) + 7
    big = torch.zeros(n, device=DEV)
    where = [0, (1 << 31) - 1, 1 << 31, (1 << 31) + 2, n - 1]
    big[where] = torch.tensor([float("nan"), float("inf"), float("-inf"), float("nan"), float("inf")], device=DEV)
    small = torch.full((9,), float("nan"), device=DEV)
    assert _scan([small, big]) == [9, 5, 14]
    assert _scan([big[1:]]) == [4, 4]                     # the unaligned loop over 2^31 + 6 elements
    del big
    torch.cuda.empty_cache()


def test_scan_rejects_bad_arguments():
    lib = _lib.load()
    assert lib.sae_nonfinite_count(None, None, 0, None, None) == 0
    assert lib.sae_nonfinite_count(None, None, 2, None, None) == -1


# ------------------------------------------------------------------------------------------------ guarded Adam
def _adam_case(sizes, offsets, null, gscale, seed):
    g = torch.Generator(DEV).manual_seed(seed)
    params, grads, layout = [], [], [0]
    for i, (sz, o) in enumerate(zip(sizes, offsets)):
        params.append(torch.randn(sz + o, device=DEV, generator=g)[o:])
        grads.append(None if i in null else torch.randn(sz, device=DEV, generator=g) * 0.1)
        layout.append(layout[-1] + (sz + 3) // 4 * 4)
    m = torch.randn(layout[-1], device=DEV, generator=g) * 0.01
    v = torch.rand(layout[-1], device=DEV, generator=g) * 0.01
    steps = torch.tensor([float(i + 1) for i in range(len(sizes))], device=DEV)
    return params, grads, layout[:-1], m, v, steps


def _adam(name, state, gscale, skip=None):
    params, grads, offsets, m, v, steps = state
    # the device tables stay referenced until the kernels have run (the synchronize below)
    tables = (_table(params), _table(grads), torch.tensor(offsets, dtype=torch.int64, device=DEV),
              torch.tensor([p.numel() for p in params], dtype=torch.int64, device=DEV))
    args = tuple(_p(t) for t in tables) + (len(params), _p(m), _p(v), _p(steps), 2e-3, 0.5, 0.99, 1e-8, gscale)
    fn = getattr(_lib.load(), name)
    _lib.check(fn(*args, _p(skip), _stream()) if skip is not None else fn(*args, _stream()), name)
    torch.cuda.synchronize()


def _clone(state):
    params, grads, offsets, m, v, steps = state
    return [p.clone() for p in params], grads, offsets, m.clone(), v.clone(), steps.clone()


def _bits(a, b):
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize("sizes,offsets,null,gscale", [((4096, 1024), (0, 0), (), 1.0),          # float4
                                                       ((1001, 7), (0, 0), (), 1.0),             # scalar (size)
                                                       ((4096, 515), (1, 0), (), 0.5),           # scalar (offset), scale
                                                       ((4096, 333, 64), (0, 0, 0), (1,), 0.25)],  # null gradient
                         ids=["f4", "scalar_odd", "scalar_offset1_gscale", "null_grad_gscale"])
def test_guarded_adam(sizes, offsets, null, gscale):
    state = _adam_case(sizes, offsets, null, gscale, seed=len(sizes) + int(gscale * 8))
    plain, guarded, skipped = _clone(state), _clone(state), _clone(state)
    _adam("sae_adam_step", plain, gscale)
    _adam("sae_adam_step_guarded", guarded, gscale, skip=torch.zeros(1, dtype=torch.int64, device=DEV))
    for a, b in zip(plain[0] + [plain[3], plain[4], plain[5]], guarded[0] + [guarded[3], guarded[4], guarded[5]]):
        assert _bits(a, b)
    assert not _bits(plain[0][0], state[0][0])
    _adam("sae_adam_step_guarded", skipped, gscale, skip=torch.full((1,), 3, dtype=torch.int64, device=DEV))
    for a, b in zip(skipped[0] + [skipped[3], skipped[4], skipped[5]], state[0] + [state[3], state[4], state[5]]):
        assert _bits(a, b)
    lib = _lib.load()
    assert lib.sae_adam_step_guarded(*([None] * 4), 1, None, None, None, 2e-3, 0.5, 0.99, 1e-8, 1.0, None, None) == -1


# ------------------------------------------------------------------------------------------------ half-steps
@pytest.fixture
def kern():
    k = backend.kernels()
    prev = (k.precision, k.deterministic)
    yield k
    k.precision, k.deterministic = prev


def _trainer(**over):
    import swapping_autoencoder_pytorch_b200 as S
    opt = default_options(**dict(TINY, num_gpus=1, **over))
    torch.manual_seed(0)
    return S.create_optimizer(opt, S.create_model(opt))


def _real(seed=5):
    return torch.randn(2, 3, 64, 64, device=DEV, generator=torch.Generator(DEV).manual_seed(seed)).clamp(-1, 1)


def _state(tr):
    out = [p.detach().clone() for p in tr.model.singlegpu_model.parameters()]
    for o in (tr.optimizer_G, tr.optimizer_D):
        st = o._state()
        out += [st.exp_avg.clone(), st.exp_avg_sq.clone(), st.steps.clone()]
    return out


def _same(a, b):
    return len(a) == len(b) and all(_bits(x, y) for x, y in zip(a, b))


class Poison:
    """Post-accumulate-grad hooks that overwrite element 0 of the gradient of one chosen tensor per kind of half-step — with
    a device-side select, so the same hook works eagerly and inside a captured graph.  Before each half-step body the
    trainer's ``_run`` sets the device flags (only the body of kind ``target`` is poisoned) and snapshots the state."""

    def __init__(self, tr, targets):
        self.tr = tr
        self.flags, self.names, self.handles = {}, {}, []
        named = dict(tr.model.singlegpu_model.named_parameters())
        for kind, (net, value) in targets.items():
            name = next(n for n in named if n.startswith(net + "."))
            p = named[name]
            flag = torch.zeros(1, dtype=torch.bool, device=DEV)
            val = torch.full((1,), value, device=DEV)
            self.flags[kind], self.names[kind] = flag, name

            def hook(param, flag=flag, val=val):
                with torch.no_grad():
                    g0 = param.grad.view(-1)[:1]
                    g0.copy_(torch.where(flag, val, g0))
            frozen = not p.requires_grad
            self.handles.append(p.requires_grad_(True).register_post_accumulate_grad_hook(hook))
            p.requires_grad_(not frozen)
        self.target, self.snapshots = None, {}
        orig = tr._run

        def run(kind, images):
            for k, f in self.flags.items():
                f.fill_(k == kind and kind == self.target)
            self.snapshots[kind] = _state(tr)
            return orig(kind, images)
        tr._run = run


@pytest.mark.parametrize("graphs,precision,det", [(False, "tf32", False), (True, "tf32", False), (False, "fp32", False),
                                                 (True, "fp32", False), (False, "tf32", True), (True, "tf32", True)],
                         ids=["eager-tf32", "graphs-tf32", "eager-fp32", "graphs-fp32", "eager-det", "graphs-det"])
def test_poisoned_half_steps_are_skipped(kern, graphs, precision, det):
    kern.precision, kern.deterministic = precision, det
    tr = _trainer(cuda_graphs=graphs, R1_once_every=2, skip_nonfinite_steps=True)
    poison = Poison(tr, {"D": ("Dpatch", float("inf")), "R1": ("D", float("nan")), "G": ("E", float("-inf"))})
    real = _real()
    torch.manual_seed(1)
    for _ in range(12):              # D, G, D + R1, G, ...: with graphs, every body is captured and then replayed
        tr.train_one_step({"real_A": real}, 0)
    if graphs:
        assert tr.graphs.disabled is None, (tr.graphs.disabled, tr.graphs.last_traceback)
        assert {k[0] for k in tr.graphs.captured} == {"D", "R1", "G"}
        assert all(k[4] for k in tr.graphs.captured)
    assert tr.nonfinite_steps() == {"D": 0, "R1": 0, "G": 0}
    expected = {"D": 0, "R1": 0, "G": 0}
    # half-step 13: D without R1 (iteration 7), poisoned; 14: G, clean; 15: D + R1 with R1 poisoned; 16: G, poisoned
    for kind in ("D", None, "R1", "G"):
        poison.target = kind
        before = _state(tr)
        counters = (tr.train_mode_counter, tr.discriminator_iter_counter)
        out = tr.train_one_step({"real_A": real}, 0)
        assert (tr.train_mode_counter, tr.discriminator_iter_counter) != counters
        if kind is None:
            assert not _same(_state(tr), before)
            continue
        expected[kind] += 1
        if kind == "R1":
            assert "D_R1" in out
            assert not _same(poison.snapshots["R1"], before)            # the D update of the same half-step was applied
            assert _same(_state(tr), poison.snapshots["R1"])
        else:
            assert "D_R1" not in out
            assert _same(_state(tr), before)
        assert tr.nonfinite_steps() == expected
        assert tr.nonfinite_report(kind) == {poison.names[kind]: 1}
    poison.target = None
    for _ in range(2):               # D, G: clean again, both update
        before = _state(tr)
        tr.train_one_step({"real_A": real}, 0)
        assert not _same(_state(tr), before)
    assert tr.nonfinite_steps() == expected
    if graphs:
        assert len(tr.graphs.captured) == 3


@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
def test_batch_with_a_nan_pixel_is_skipped(graphs):
    # no R1 in this window: its penalty's weight gradients depend on the image only through the activations' signs, so a NaN
    # pixel can leave them finite — the guard looks at gradients, and such an R1 update would go ahead
    tr = _trainer(cuda_graphs=graphs, R1_once_every=8, skip_nonfinite_steps=True)
    real = _real()
    for _ in range(6):
        tr.train_one_step({"real_A": real}, 0)
    bad = real.clone()
    bad[1, 2, 17, 33] = float("nan")
    for kind in ("D", "G"):
        before = _state(tr)
        out = tr.train_one_step({"real_A": bad}, 0)
        assert "D_R1" not in out
        assert _same(_state(tr), before), kind
        assert tr.nonfinite_steps()[kind] == 1 and tr.nonfinite_report(kind)
    assert tr.nonfinite_steps()["R1"] == 0
    before = _state(tr)
    tr.train_one_step({"real_A": real}, 0)
    assert not _same(_state(tr), before)


def _record(tr, real, steps):
    """per half-step: (loss values, gradients of the active group, parameters + Adam state), all copied"""
    rows = []
    for i in range(steps):
        out = tr.train_one_step({"real_A": real}, 0)
        group = tr.Dparams if i % 2 == 0 else tr.Gparams
        grads = [p.grad.clone() for p in group if p.grad is not None]
        rows.append(({k: float(v) for k, v in out.items()}, grads, _state(tr)))
    return rows


@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
def test_finite_steps_bitwise_unchanged_by_the_guard(kern, graphs):
    kern.deterministic = True
    steps = 16 if graphs else 4     # with graphs: warm-up, capture and then replays of all three bodies
    real = _real()
    runs = []
    for guard in (False, True):
        tr = _trainer(cuda_graphs=graphs, R1_once_every=2, skip_nonfinite_steps=guard)
        torch.manual_seed(123)
        runs.append((tr, _record(tr, real, steps)))
    (_, a), (tg, b) = runs
    for i, (ra, rb) in enumerate(zip(a, b)):
        assert ra[0] == rb[0] and all(math.isfinite(v) for v in ra[0].values()), i
        assert _same(ra[1], rb[1]) and _same(ra[2], rb[2]), i
    assert tg.nonfinite_steps() == {"D": 0, "R1": 0, "G": 0}
    if graphs:
        assert tg.graphs.disabled is None, (tg.graphs.disabled, tg.graphs.last_traceback)
        first = dict(tg.graphs.captured)
        assert {k[4] for k in first} == {True} and len(first) == 3
        tg.opt.skip_nonfinite_steps = False          # new graphs, after warm-up calls of their own (three R1 calls need 12)
        for _ in range(12):
            tg.train_one_step({"real_A": real}, 0)
        assert {(k[0], k[4]) for k in tg.graphs.captured} == {(k, g) for k in ("D", "G", "R1") for g in (False, True)}
        tg.opt.skip_nonfinite_steps = True           # back: the first graphs replay, nothing is captured
        n = len(tg.graphs.captured)
        replayed = tg.graphs.replayed_launches
        for _ in range(2):
            tg.train_one_step({"real_A": real}, 0)
        assert len(tg.graphs.captured) == n and tg.graphs.replayed_launches > replayed
        assert all(tg.graphs.captured[k] is v for k, v in first.items())
