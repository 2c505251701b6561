"""GPU (H100): the weight average (opt.ema_kimg; sae_ema_update).

* the kernel through the C ABI against an fp64 evaluation of  fmaf(beta, shadow - p, p)  within 1 ulp, beta from the device
  counter: odd sizes, a view at storage offset 1 (the element-by-element loop), a null entry, 50 updates through the ramp into
  the plateau; bitwise at beta = 1/2 over a tensor of 2^31 + 7 elements;
* a non-zero skip word leaves shadow and counter bitwise unchanged; bad arguments fail before any launch;
* training at the 256^2 default nets, eager and replayed, TF32 and fp32: the shadow is the recurrence applied to the
  parameters after each G update;
* deterministic mode: eager and replayed training bitwise equal, two runs bitwise equal, a resumed run bitwise equal;
* the guard drops the average with the G update it drops; micro_batches = 2 averages once per update;
* the averaged checkpoint loaded into a fresh isTrain=False model holds the shadow bit for bit and runs encode / decode."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from oracle.fixtures import TINY
from swapping_autoencoder_pytorch_b200 import _lib, backend, default_options

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _i64(xs):
    return torch.tensor(list(xs), dtype=torch.int64, device=DEV)


def _layout(sizes):
    offsets, o = [], 0
    for s in sizes:
        offsets.append(o)
        o += (s + 3) // 4 * 4
    return offsets, o


def _ema(params, sizes, shadow, updates, batch, half_life, rampup, skip=None):
    offsets, total = _layout(sizes)
    assert shadow.numel() >= total
    tab = _i64(0 if p is None else p.data_ptr() for p in params)
    offs, szs = _i64(offsets), _i64(sizes)
    _lib.check(_lib.load().sae_ema_update(_p(tab), _p(offs), _p(szs), len(params), _p(shadow), shadow.numel(), _p(updates),
                                          batch, half_life, rampup, _p(skip), _stream()), "sae_ema_update")
    torch.cuda.synchronize()
    return offsets


def _beta(t, batch, half_life, rampup):
    f = lambda x: float(np.float32(x))          # noqa: E731 — the value a C float argument carries
    b, h, r = f(batch), f(half_life), f(rampup)
    if r > 0:
        h = min(h, t * b * r)
    return f(0.5 ** (b / max(h, 1e-8)))


def _fma64(beta, s, p):
    """fp64 evaluation of fmaf(beta, s - p, p): the fp32 difference, then beta * d + p in fp64, rounded to fp32"""
    d = (s - p).double()
    return (beta * d + p.double()).float()


def _ulps(a, b):
    """largest distance between a and b in units of the fp32 spacing at the larger magnitude"""
    m = torch.maximum(a.abs(), b.abs())
    ulp = torch.nextafter(m, torch.full_like(m, math.inf)) - m
    return float(((a - b).abs() / ulp).max()) if a.numel() else 0.0


def _bits(a, b):
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


def _same(a, b):
    return len(a) == len(b) and all(_bits(x, y) if x.dtype == torch.float32 else torch.equal(x, y) for x, y in zip(a, b))


# ------------------------------------------------------------------------------------------------ kernel
def test_schedule_through_ramp_and_plateau_within_one_ulp():
    g = torch.Generator(DEV).manual_seed(21)
    sizes = [1, 3, 4, 5, 17, 4097, 1000003]
    params = [torch.randn(s, device=DEV, generator=g) for s in sizes]
    base = torch.randn(5002, device=DEV, generator=g)
    params += [base[1:], base[1:4097]]                   # storage offset 1: the unaligned, element-by-element loop
    sizes += [5001, 4096]
    params.insert(3, None)                               # a null entry: its segment is left alone
    sizes.insert(3, 9)
    offsets, total = _layout(sizes)
    shadow = torch.randn(total, device=DEV, generator=g)
    updates = torch.zeros(1, dtype=torch.int64, device=DEV)
    batch, half_life, rampup = 16.0, 20.0, 0.05          # ramp 0.8 t images: the plateau from t = 25
    worst, betas = 0.0, []
    for t in range(50):
        for p in params:
            if p is not None:
                p.add_(torch.randn(p.shape, device=DEV, generator=g) * 1e-2)
        before = shadow.clone()
        _ema(params, sizes, shadow, updates, batch, half_life, rampup)
        beta = _beta(t, batch, half_life, rampup)
        betas.append(beta)
        assert int(updates) == t + 1
        for p, o, s in zip(params, offsets, sizes):
            seg = shadow[o:o + s]
            if p is None:
                assert _bits(seg, before[o:o + s])
            else:
                worst = max(worst, _ulps(seg, _fma64(beta, before[o:o + s], p)))
    assert worst <= 1.0, worst
    assert betas[0] == 0.0 and 0.0 < betas[10] < betas[30] == betas[49] == _beta(10 ** 6, batch, half_life, 0.0)


def test_skip_leaves_shadow_and_counter():
    g = torch.Generator(DEV).manual_seed(22)
    p = torch.randn(1003, device=DEV, generator=g)
    shadow = torch.randn(1004, device=DEV, generator=g)
    updates = torch.full((1,), 7, dtype=torch.int64, device=DEV)
    skip = torch.full((1,), 3, dtype=torch.int64, device=DEV)
    before = shadow.clone()
    _ema([p], [1003], shadow, updates, 4.0, 10.0, 0.05, skip=skip)
    assert _bits(shadow, before) and int(updates) == 7
    skip.zero_()
    _ema([p], [1003], shadow, updates, 4.0, 10.0, 0.05, skip=skip)
    assert int(updates) == 8 and not _bits(shadow, before)
    assert _ulps(shadow[:1003], _fma64(_beta(7, 4.0, 10.0, 0.05), before[:1003], p)) <= 1.0


def test_bad_arguments_fail_before_any_launch():
    lib = _lib.load()
    p, shadow = torch.zeros(8, device=DEV), torch.zeros(8, device=DEV)
    updates = torch.zeros(1, dtype=torch.int64, device=DEV)
    tab, offs, szs = _i64([p.data_ptr()]), _i64([0]), _i64([8])
    good = [_p(tab), _p(offs), _p(szs), 1, _p(shadow), 8, _p(updates), 4.0, 10.0, 0.05, None, None]
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    for i, bad in [(0, None), (1, None), (2, None), (4, None), (6, None), (5, -1), (3, -1), (3, 65536), (7, 0.0), (7, -1.0),
                   (8, 0.0), (8, -2.0), (8, float("nan")), (9, -0.5), (9, float("nan"))]:
        args = list(good)
        args[i] = bad
        assert lib.sae_ema_update(*args) == -1, (i, bad)
    assert _lib.launch_count() == n0
    torch.cuda.synchronize()
    assert int(updates) == 0
    with pytest.raises(_lib.SaeError):
        backend.kernels().ema_update([p], offs, szs, shadow, updates, 4.0, 0.0, 0.05, backend.PointerTables(1, p.device))
    assert int(updates) == 0


def test_beyond_2_31_elements_bitwise_at_one_half():
    n = (1 << 31) + 7
    g = torch.Generator(DEV).manual_seed(23)
    p = torch.randn(n + 1, device=DEV, generator=g)
    shadow = torch.randn(n + 1, device=DEV, generator=g)
    updates = torch.zeros(1, dtype=torch.int64, device=DEV)
    chunk = 1 << 28
    for view, size in ((p[:n], n), (p[1:n], n - 1)):     # float4 body + tail; then the unaligned loop
        want = torch.empty(size, device=DEV)
        for i in range(0, size, chunk):                  # beta = 1/2 (no ramp, B = h): 0.5 * d is exact, one rounding
            j = min(i + chunk, size)
            want[i:j] = view[i:j] + 0.5 * (shadow[i:j] - view[i:j])
        _ema([view], [size], shadow, updates, 8.0, 8.0, 0.0)
        assert all(_bits(shadow[i:min(i + chunk, size)], want[i:min(i + chunk, size)]) for i in range(0, size, chunk))
        del want
    assert int(updates) == 2
    del p, shadow
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ training
@pytest.fixture
def kern():
    k = backend.kernels()
    prev = (k.precision, k.deterministic)
    yield k
    k.precision, k.deterministic = prev


def _zero_noise(monkeypatch):
    """graph replay and eager execution draw different random numbers: without noise maps and crops a step draws none"""
    from swapping_autoencoder_pytorch_b200.stylegan2_layers import NoiseInjection

    def zero_noise(self, image, noise=None):
        if self.image_size is None:
            self.image_size = image.shape
        b, _, h, w = image.shape
        return image.new_empty(b, 1, h, w).zero_()
    monkeypatch.setattr(NoiseInjection, "resolve_noise", zero_noise)


def _trainer(base, seed=0, **over):
    import swapping_autoencoder_pytorch_b200 as S
    opt = default_options(**dict(base, num_gpus=1, **over))
    torch.manual_seed(seed)
    return S.create_optimizer(opt, S.create_model(opt))


def _real(n, size, seed=5):
    return torch.randn(n, 3, size, size, device=DEV, generator=torch.Generator(DEV).manual_seed(seed)).clamp(-1, 1)


def _state(tr):
    out = [p.detach().clone() for p in tr.model.singlegpu_model.parameters()]
    out += [v.detach().clone() for v in tr.ema.averaged()] + [tr.ema.updates.clone()]
    return out


@pytest.mark.parametrize("precision", ["tf32", "fp32"])
@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
def test_default_nets_shadow_is_the_recurrence(kern, precision, graphs):
    kern.precision, kern.deterministic = precision, False
    batch, half_life, rampup = 4, 10.0, 1.0                # beta 0, 1/2, 0.71, then 0.76 from t = 3
    tr = _trainer({}, batch_size=batch, cuda_graphs=graphs, ema_kimg=half_life / 1000, ema_rampup=rampup)
    real = _real(batch, 256)
    ref = [p.detach().clone() for p in tr.Gparams]
    assert _same([v for v in tr.ema.averaged()], ref)
    n_g, worst = 0, 0.0
    for _ in range(12):                                    # D, G, ...: 6 G updates, with graphs 3 of them replayed
        if tr.train_mode_counter == 1:                     # the next half-step is a G update
            tr.train_one_step({"real_A": real}, 0)
            beta = _beta(n_g, batch, half_life, rampup)
            ref = [_fma64(beta, s, p.detach()) for s, p in zip(ref, tr.Gparams)]
            n_g += 1
            torch.cuda.synchronize()
            worst = max(worst, max(_ulps(a, b) for a, b in zip(tr.ema.averaged(), ref)))
        else:
            tr.train_one_step({"real_A": real}, 0)
    assert n_g == 6 and int(tr.ema.updates) == 6
    # each step is within 1 ulp of its fp64 evaluation; a difference in the shadow decays by beta per step
    assert worst <= 1.0 / (1.0 - 0.76) + 1.0, worst
    if graphs:
        assert tr.graphs.disabled is None, (tr.graphs.disabled, tr.graphs.last_traceback)
        g_keys = [k for k in tr.graphs.captured if k[0] == "G"]
        assert g_keys and all(k[-1] == ("ema", half_life, rampup) for k in g_keys)
        assert all(len(k) == 5 for k in tr.graphs.captured if k[0] != "G")


def _deterministic_run(monkeypatch, graphs, steps=12, seed=0):
    _zero_noise(monkeypatch)
    tr = _trainer(TINY, seed=seed, batch_size=4, cuda_graphs=graphs, R1_once_every=2, lambda_PatchGAN=0.0,
                  lambda_patch_R1=0.0, ema_kimg=0.002, ema_rampup=0.5)
    real = _real(4, 64)
    torch.manual_seed(123)
    for _ in range(steps):
        tr.train_one_step({"real_A": real}, 0)
    torch.cuda.synchronize()
    if graphs:
        assert tr.graphs.disabled is None, (tr.graphs.disabled, tr.graphs.last_traceback)
        assert sorted(k[0] for k in tr.graphs.captured) == ["D", "G", "R1"]
    return tr


def test_deterministic_eager_replay_and_reruns_bitwise(kern, monkeypatch):
    kern.deterministic = True
    eager = _state(_deterministic_run(monkeypatch, False))
    replay = _state(_deterministic_run(monkeypatch, True))
    again = _state(_deterministic_run(monkeypatch, True))
    assert int(eager[-1]) == 6
    assert _same(eager, replay)
    assert _same(replay, again)


def test_deterministic_resume_from_saved_files(kern, tmp_path):
    kern.deterministic = True
    over = dict(batch_size=4, R1_once_every=2, ema_kimg=0.002, ema_rampup=0.5, checkpoints_dir=str(tmp_path), name="ema")
    real = _real(4, 64)
    a = _trainer(TINY, **over)
    torch.manual_seed(5)
    for _ in range(5):
        a.train_one_step({"real_A": real}, 0)
    a.save(3000)
    rng = (torch.get_rng_state(), torch.cuda.get_rng_state())
    for _ in range(5):
        a.train_one_step({"real_A": real}, 0)
    b = _trainer(TINY, seed=77, **over)
    assert b.model.singlegpu_model.load(os.path.join(str(tmp_path), "ema", "3k_checkpoint.pth"))
    assert b.load()
    torch.set_rng_state(rng[0])
    torch.cuda.set_rng_state(rng[1])
    for _ in range(5):
        b.train_one_step({"real_A": real}, 0)
    assert int(b.ema.updates) == 5
    assert _same(_state(a), _state(b))


@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
def test_guard_drops_the_average_with_the_update(graphs):
    tr = _trainer(TINY, batch_size=4, R1_once_every=100, cuda_graphs=graphs, skip_nonfinite_steps=True, ema_kimg=0.01)
    name, p = next((n, p) for n, p in tr.model.singlegpu_model.named_parameters() if n.startswith("E."))
    flag = torch.zeros(1, dtype=torch.bool, device=DEV)
    val = torch.full((1,), float("inf"), device=DEV)

    def hook(param):
        with torch.no_grad():
            g0 = param.grad.view(-1)[:1]
            g0.copy_(torch.where(flag, val, g0))          # a device-side select: the same hook works inside a graph
    handle = p.register_post_accumulate_grad_hook(hook)
    real = _real(4, 64)
    for _ in range(8):                                    # warm-up, capture and replays of D and G
        tr.train_one_step({"real_A": real}, 0)
    assert int(tr.ema.updates) == 4
    before = _state(tr)
    flag.fill_(True)
    tr.train_one_step({"real_A": real}, 0)                # D: untouched by the poison (E is frozen)
    tr.train_one_step({"real_A": real}, 0)                # G: dropped
    flag.fill_(False)
    after = _state(tr)
    n_g = len(tr.Gparams)
    assert _same(after[-n_g - 1:], before[-n_g - 1:])     # shadow and counter
    assert tr.nonfinite_steps() == {"D": 0, "R1": 0, "G": 1} and tr.nonfinite_report("G") == {name: 1}
    tr.train_one_step({"real_A": real}, 0)
    tr.train_one_step({"real_A": real}, 0)
    assert int(tr.ema.updates) == 5
    handle.remove()
    if graphs:
        assert tr.graphs.disabled is None, (tr.graphs.disabled, tr.graphs.last_traceback)


@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
def test_micro_batches_average_once_per_update(kern, graphs):
    kern.deterministic = False
    batch, half_life, rampup = 4, 8.0, 1.0
    tr = _trainer(TINY, batch_size=batch, micro_batches=2, cuda_graphs=graphs, ema_kimg=half_life / 1000,
                  ema_rampup=rampup)
    real = _real(batch, 64)
    ref = [p.detach().clone() for p in tr.Gparams]
    n_g = 0
    for _ in range(8):
        g_step = tr.train_mode_counter == 1
        tr.train_one_step({"real_A": real}, 0)
        if g_step:                                        # B is the update's 4 images, not a micro-batch's 2
            ref = [_fma64(_beta(n_g, batch, half_life, rampup), s, p.detach()) for s, p in zip(ref, tr.Gparams)]
            n_g += 1
    torch.cuda.synchronize()
    assert n_g == 4 and int(tr.ema.updates) == 4
    assert max(_ulps(a, b) for a, b in zip(tr.ema.averaged(), ref)) <= 4.0
    if graphs:
        assert tr.graphs.disabled is None, (tr.graphs.disabled, tr.graphs.last_traceback)
        assert [k for k in tr.graphs.captured if k[0] == "G"][0][5:] == (2, ("ema", half_life, rampup))


def test_averaged_checkpoint_loads_into_an_inference_model(tmp_path):
    import swapping_autoencoder_pytorch_b200 as S
    tr = _trainer(TINY, batch_size=4, ema_kimg=0.005, checkpoints_dir=str(tmp_path), name="ema")
    real = _real(4, 64)
    for _ in range(6):
        tr.train_one_step({"real_A": real}, 0)
    tr.save(6000)
    torch.manual_seed(1234)
    model = S.create_model(default_options(**dict(TINY, num_gpus=1, isTrain=False, checkpoints_dir=str(tmp_path), name="ema",
                                                   resume_iter="latest_ema"))).singlegpu_model
    own = dict(model.named_parameters())
    for n, v in zip(tr.ema.names, tr.ema.averaged()):
        assert _bits(own[n].detach(), v), n
    with torch.no_grad():
        sp, gl = model(real, command="encode")
        out = model(sp, gl, command="decode")
    assert out.shape == real.shape and bool(torch.isfinite(out).all())
