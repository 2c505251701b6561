"""GPU (H100): the training statistics (opt.training_stats; sae_sumsq, sae_adam_norms, sae_score_stats).

* sae_sumsq through the C ABI against fp64 to 1e-12 relative: odd sizes, a view at storage offset 1, a NULL entry, added
  into what the output held; the same values at an aligned and an unaligned address give bitwise the same sums; two launches
  are bitwise equal; exact over a tensor of 2^31 + 5 elements;
* sae_adam_norms after a real sae_adam_step: against fp64 of Adam's step formula and against |p_before - p_after|; a NULL
  gradient adds no step; a non-zero skip word adds nothing, the update count included;
* sae_score_stats on a strided view with planted NaN / +-Inf against fp64; bitwise repeatable;
* bad arguments fail before any launch;
* training at the 256^2 default nets, TF32 and fp32, eager and replayed: after every half-step the window equals the norms
  of the trainer's own gradients, parameters and moments;
* deterministic mode: eager and replayed runs, and two replayed runs, give bitwise equal windows, losses and parameters;
* a replayed half-step launches exactly the new kernels more than with the statistics off."""
import ctypes

import pytest
import torch

from oracle.fixtures import TINY
from swapping_autoencoder_pytorch_b200 import _lib, backend, default_options
from swapping_autoencoder_pytorch_b200.optimizer import NONFINITE_KINDS

pytestmark = pytest.mark.gpu
DEV = "cuda"
B = _lib.SAE_STATS_BLOCKS


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _i64(xs):
    return torch.tensor(list(xs), dtype=torch.int64, device=DEV)


def _sumsq(tensors, out, scale=1.0, skip=None):
    lib = _lib.load()
    tab = _i64([0 if t is None else t.data_ptr() for t in tensors])
    sizes = _i64([0 if t is None else t.numel() for t in tensors])
    partials = torch.full((len(tensors) * B,), float("nan"), dtype=torch.float64, device=DEV)
    rc = lib.sae_sumsq(_p(tab), _p(sizes), len(tensors), scale, _p(out), _p(partials), _p(skip), _stream())
    _lib.check(rc, "sae_sumsq")
    torch.cuda.synchronize()


def _rel(a, b):
    return abs(a - b) / max(abs(b), 1e-300)


def _rand(n, seed):
    return torch.randn(n, device=DEV, generator=torch.Generator(DEV).manual_seed(seed))


def test_sumsq_against_fp64():
    sizes = [1, 3, 4, 5, 7, 1023, 4097, 100003, 1 << 20]
    xs = [_rand(n, i) * (i + 1) for i, n in enumerate(sizes)]
    store = _rand(5001, 99)
    xs.append(store[1:])                                  # storage offset 1: four scalar loads per group
    xs.insert(3, None)
    scale = 0.37
    out = torch.arange(len(xs), dtype=torch.float64, device=DEV)     # the sums are added to what is there
    _sumsq(xs, out, scale)
    for i, x in enumerate(xs):
        want = float(i) + (0.0 if x is None else float((x.double() ** 2).sum()) * float(torch.tensor(scale).double()) ** 2)
        assert _rel(float(out[i]), want) < 1e-12, (i, float(out[i]), want)
    again = torch.arange(len(xs), dtype=torch.float64, device=DEV)
    _sumsq(xs, again, scale)
    assert torch.equal(out, again)                        # two launches: bitwise equal
    # the partition does not depend on the alignment: the same values at an aligned address give the same bits
    aligned = store[1:].clone()
    a, b = torch.zeros(1, dtype=torch.float64, device=DEV), torch.zeros(1, dtype=torch.float64, device=DEV)
    _sumsq([aligned], a)
    _sumsq([store[1:]], b)
    assert torch.equal(a, b)


def test_sumsq_beyond_2_31_elements():
    n = (1 << 31) + 5
    x = torch.full((n,), 0.5, device=DEV)
    x[-1] = 3.0                                            # beyond 2^31: in the scalar tail of the last group
    x[(1 << 31) + 1] = -2.0
    out = torch.zeros(1, dtype=torch.float64, device=DEV)
    _sumsq([x], out)
    assert float(out[0]) == 0.25 * (n - 2) + 9.0 + 4.0     # every partial sum is exact in fp64
    del x
    torch.cuda.empty_cache()


def _adam_setup(sizes, seed=1):
    params = [_rand(n, seed + i) for i, n in enumerate(sizes)]
    grads = [_rand(n, seed + 100 + i) * 0.1 for i, n in enumerate(sizes)]
    offsets, o = [], 0
    for n in sizes:
        offsets.append(o)
        o += (n + 3) // 4 * 4
    m = torch.zeros(o, device=DEV)
    v = torch.zeros(o, device=DEV)
    steps = torch.zeros(len(sizes), device=DEV)
    return params, grads, _i64(offsets), _i64(sizes), m, v, steps


def _norms(params, grads, offsets, sizes, m, v, steps, hp, skip=None):
    cache = backend.PointerTables(len(params), torch.device(DEV))
    w = torch.zeros(len(params), dtype=torch.float64, device=DEV)
    u = torch.zeros(len(params), dtype=torch.float64, device=DEV)
    cnt = torch.zeros(1, dtype=torch.float64, device=DEV)
    partials = torch.zeros(2 * len(params) * B, dtype=torch.float64, device=DEV)
    backend.kernels().adam_norms(params, grads, offsets, sizes, m, v, steps, *hp, w, u, cnt, partials, cache, skip=skip)
    torch.cuda.synchronize()
    return w, u, cnt


def test_adam_norms_against_fp64_and_the_parameter_change():
    sizes = [3, 4, 17, 1000, 65537, 300001]
    params, grads, offsets, sizes_t, m, v, steps = _adam_setup(sizes)
    grads[2] = None                                        # Adam skips it: no step, but a weight norm
    hp = (0.01, 0.9, 0.99, 1e-8)
    cache = backend.PointerTables(len(params), torch.device(DEV))
    k = backend.kernels()
    for it in range(3):
        before = [p.clone() for p in params]
        k.adam_step(params, grads, offsets, sizes_t, m, v, steps, *hp, 0.5, cache)
        w, u, cnt = _norms(params, grads, offsets, sizes_t, m, v, steps, hp)
        assert float(cnt) == 1.0
        lr, b1, b2, eps = hp
        for i, p in enumerate(params):
            assert _rel(float(w[i]), float((p.double() ** 2).sum())) < 1e-12
            if grads[i] is None:
                assert float(u[i]) == 0.0 and float(steps[i]) == 0.0
                continue
            o, n, t = int(offsets[i]), sizes[i], float(steps[i])
            mm, vv = m[o:o + n].double(), v[o:o + n].double()
            d = lr / (1 - b1 ** t) * mm / (vv.sqrt() / (1 - b2 ** t) ** 0.5 + eps)
            assert _rel(float(u[i]), float((d ** 2).sum())) < 1e-5, (it, i)             # fp32 rounding of the step
            dp = float(((before[i].double() - p.double()) ** 2).sum())
            assert _rel(float(u[i]) ** 0.5, dp ** 0.5) < 1e-4, (it, i)                 # within the rounding of p
    # a dropped update adds nothing, to the count included
    skip = torch.ones(1, dtype=torch.int64, device=DEV)
    w, u, cnt = _norms(params, grads, offsets, sizes_t, m, v, steps, hp, skip=skip)
    assert float(cnt) == 0.0 and float(w.abs().sum()) == 0.0 and float(u.abs().sum()) == 0.0
    out = torch.zeros(len(params), dtype=torch.float64, device=DEV)
    _sumsq(params, out, skip=skip)
    assert float(out.abs().sum()) == 0.0
    # bitwise repeatable
    a, b = _norms(params, grads, offsets, sizes_t, m, v, steps, hp), _norms(params, grads, offsets, sizes_t, m, v, steps, hp)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_score_stats_with_planted_nonfinite():
    base = _rand(3 * 777, 7).view(777, 3) * 3
    base[5, 1] = float("nan")
    base[100, 1] = float("inf")
    base[200, 1] = -float("inf")
    base[300, 1] = 0.0
    base[301, 1] = -0.0
    x = base[:, 1]                                         # stride 3
    acc = torch.tensor([1.0, 2.0, 3.0, 4.0], dtype=torch.float64, device=DEV)
    k = backend.kernels()
    k.score_stats(x, acc)
    torch.cuda.synchronize()
    fin = torch.isfinite(x)
    want = [1.0 + float(x[fin].double().sum()), 2.0 + float(torch.sign(x[fin]).double().sum()), 3.0 + int(fin.sum()), 4.0 + 3]
    assert _rel(float(acc[0]), want[0]) < 1e-12
    assert acc[1:].tolist() == want[1:]
    # 2-D, transposed, and bitwise repeatable
    y = base[:64].t()
    a = torch.zeros(4, dtype=torch.float64, device=DEV)
    b = torch.zeros(4, dtype=torch.float64, device=DEV)
    k.score_stats(y, a)
    k.score_stats(y, b)
    torch.cuda.synchronize()
    assert torch.equal(a, b) and float(a[3]) == 1.0 and float(a[2]) == 64 * 3 - 1


def test_bad_arguments_fail_before_any_launch():
    lib = _lib.load()
    out = torch.zeros(4, dtype=torch.float64, device=DEV)
    x = torch.zeros(8, device=DEV)
    tab, sizes = _i64([x.data_ptr()]), _i64([8])
    sz, st = (ctypes.c_int64 * 1)(8), (ctypes.c_int64 * 1)(1)
    n0 = _lib.launch_count()
    assert lib.sae_sumsq(_p(tab), _p(sizes), 1, 1.0, _p(out), None, None, None) == -1
    assert lib.sae_sumsq(_p(tab), _p(sizes), 70000, 1.0, _p(out), _p(out), None, None) == -1
    assert lib.sae_sumsq(_p(tab), _p(sizes), 1, float("inf"), _p(out), _p(out), None, None) == -1
    assert lib.sae_adam_norms(_p(tab), _p(tab), _p(sizes), _p(sizes), 1, _p(x), _p(x), _p(x), 0.1, 1.0, 0.9, 1e-8,
                              _p(out), _p(out), None, _p(out), None, None) == -1                # beta1 = 1
    assert lib.sae_adam_norms(_p(tab), None, _p(sizes), _p(sizes), 1, _p(x), _p(x), _p(x), 0.1, 0.0, 0.9, 1e-8,
                              _p(out), _p(out), None, _p(out), None, None) == -1
    assert lib.sae_score_stats(_p(x), 5, sz, st, _p(out), None) == -1
    assert lib.sae_score_stats(_p(x), 1, sz, st, None, None) == -1
    assert lib.sae_score_stats(None, 1, sz, st, _p(out), None) == -1
    assert _lib.launch_count() == n0


# ------------------------------------------------------------------------------------------------ training
@pytest.fixture
def kern():
    k = backend.kernels()
    prev = (k.precision, k.deterministic)
    yield k
    k.precision, k.deterministic = prev


def _trainer(base, seed=0, **over):
    import swapping_autoencoder_pytorch_b200 as S
    opt = default_options(**dict(base, num_gpus=1, **over))
    torch.manual_seed(seed)
    return S.create_optimizer(opt, S.create_model(opt))


def _real(n, size, seed=5):
    return torch.randn(n, 3, size, size, device=DEV, generator=torch.Generator(DEV).manual_seed(seed)).clamp(-1, 1)


def _expected(tr, kind):
    """per-tensor (grad^2, weight^2, step^2) of the update just made, from the trainer's own .grad, parameters and moments"""
    adam = tr.optimizer_G if kind == "G" else tr.optimizer_D
    g = adam.param_groups[0]
    lr, (b1, b2), eps = g["lr"], g["betas"], g["eps"]
    out = []
    for i, p in enumerate(adam.params):
        gr = p.grad
        w = float((p.detach().double() ** 2).sum())
        if gr is None:
            out.append((0.0, w, 0.0))
            continue
        o, n, t = adam._offsets[i], adam._sizes[i], float(adam.steps[i])
        m, v = adam.exp_avg[o:o + n].double(), adam.exp_avg_sq[o:o + n].double()
        d = lr / (1 - b1 ** t) * m / (v.sqrt() / (1 - b2 ** t) ** 0.5 + eps)
        out.append((float((gr.double() ** 2).sum()), w, float((d ** 2).sum())))
    return out


@pytest.mark.parametrize("precision", ["tf32", "fp32"])
@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
def test_default_nets_window_is_the_trainer_norms(kern, precision, graphs):
    kern.precision, kern.deterministic = precision, False
    tr = _trainer({}, batch_size=4, cuda_graphs=graphs, R1_once_every=2, training_stats=True)
    real = _real(4, 256)
    for step in range(12):                                 # 6 D, 6 G, 3 R1: every body replayed from its 3rd call on
        if tr.train_mode_counter == 1:
            kinds = ["G"]
        else:
            kinds = ["D", "R1"] if (tr.discriminator_iter_counter + 1) % 2 == 0 else ["D"]
        tr.train_one_step({"real_A": real}, 0)
        torch.cuda.synchronize()
        kind = kinds[-1]                                   # D's gradients are gone once R1 has run: check the last update
        u, gsq, wsq, usq = tr.stats._views(kind)
        assert float(u) == 1.0, (step, kind)
        for i, (eg, ew, eu) in enumerate(_expected(tr, kind)):
            assert _rel(float(gsq[i]), eg) < 1e-9 or eg == float(gsq[i]) == 0.0, (step, kind, i)
            assert _rel(float(wsq[i]), ew) < 1e-9, (step, kind, i)
            assert _rel(float(usq[i]), eu) < 1e-4 or eu == float(usq[i]) == 0.0, (step, kind, i)
        got = tr.training_stats()
        for kind in NONFINITE_KINDS:
            assert got[kind + "/updates"] == (1 if kind in kinds else 0)
        assert all(v == v for v in got.values())
        if kinds == ["G"]:
            assert got["G/scores/rec/nonfinite"] == 0 and got["G/signs/mix"] != 0.0
        else:
            assert got["D/grad_norm"] > 0.0 and got["D/update_norm"] > 0.0
    if graphs:
        assert tr.graphs.disabled is None, (tr.graphs.disabled, tr.graphs.last_traceback)
        assert sorted(k[0] for k in tr.graphs.captured) == ["D", "G", "R1"]
        assert all(k[-1] == ("stats",) and len(k) == 6 for k in tr.graphs.captured)


def _deterministic_run(monkeypatch, graphs, steps=12):
    from swapping_autoencoder_pytorch_b200.stylegan2_layers import NoiseInjection

    def zero_noise(self, image, noise=None):
        if self.image_size is None:
            self.image_size = image.shape
        b, _, h, w = image.shape
        return image.new_empty(b, 1, h, w).zero_()
    # graph replay and eager execution draw different random numbers: without noise maps and crops a step draws none
    monkeypatch.setattr(NoiseInjection, "resolve_noise", zero_noise)
    tr = _trainer(TINY, batch_size=4, cuda_graphs=graphs, R1_once_every=2, lambda_PatchGAN=0.0, lambda_patch_R1=0.0,
                  training_stats=True)
    real = _real(4, 64)
    torch.manual_seed(123)
    losses = [tr.train_one_step({"real_A": real}, 0) for _ in range(steps)]
    torch.cuda.synchronize()
    if graphs:
        assert tr.graphs.disabled is None, (tr.graphs.disabled, tr.graphs.last_traceback)
    state = [p.detach().clone() for p in tr.model.singlegpu_model.parameters()] + [tr.stats.window.clone()]
    losses = [{k: float(v) for k, v in d.items()} for d in losses]
    return state, losses, tr.training_stats(per_tensor=True)


def test_deterministic_eager_replay_and_reruns_bitwise(kern, monkeypatch):
    kern.deterministic = True
    runs = [_deterministic_run(monkeypatch, g) for g in (False, True, True)]
    for state, losses, stats in runs[1:]:
        assert all(a.dtype == b.dtype and torch.equal(a, b) for a, b in zip(runs[0][0], state))
        assert losses == runs[0][1]
        assert stats == runs[0][2]
    assert runs[0][2]["G/updates"] == 6 and runs[0][2]["R1/updates"] == 3


def test_replay_launches_only_the_new_kernels(kern):
    kern.deterministic = False
    counts = []
    for on in (False, True):
        tr = _trainer(TINY, batch_size=4, cuda_graphs=True, R1_once_every=1, training_stats=on)
        real = _real(4, 64)
        for _ in range(8):
            tr.train_one_step({"real_A": real}, 0)
        torch.cuda.synchronize()
        assert tr.graphs.disabled is None, (tr.graphs.disabled, tr.graphs.last_traceback)
        counts.append({k[0]: v[3] for k, v in tr.graphs.captured.items()})
    off, on = counts
    # sumsq and adam_norms: two launches each; one score launch per logit tensor (D: 3 image + 2 patch, G: 2 + 1)
    assert {k: on[k] - off[k] for k in off} == {"D": 4 + 5, "R1": 4, "G": 4 + 3}
