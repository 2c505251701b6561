"""GPU (H100): gradient accumulation (opt.micro_batches; sae_bucket_accumulate).

* the kernel through the C ABI: bitwise torch's fp32 a + b for every size class (float4 body, scalar tail), gradient views at
  storage offset 1 (the element-by-element loop), null entries, n = 0, bad arguments, one tensor of 2^31 + 7 elements;
* deterministic mode, 256^2 default nets, batch 4, k = 2: D, D + R1 and G updates, eager and replayed, TF32 and fp32, bitwise
  equal to the trainer's bodies run eagerly with step=False per micro-batch, the gradients summed in order and one Adam step
  with grad_scale = 1 / 2;
* default (atomic) mode: the bucket Adam reads is bitwise the fp32 sum, in order, of the micro-batches' gradient buffers;
* two deterministic runs are bitwise identical;
* the non-finite guard drops an update poisoned in micro-batch 1 only, counts it once and names the tensor;
* with graphs: one graph per kind; an update is k replays, one sae_bucket_pack and k - 1 sae_bucket_accumulate issued
  after them, then Adam."""
import ctypes

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


def _accumulate(grads, sizes, bucket):
    """sae_bucket_accumulate of grads (None: a null entry of the given size) into bucket, in the layout of sae_bucket_pack"""
    offsets, o = [], 0
    for s in sizes:
        offsets.append(o)
        o += (s + 3) // 4 * 4
    assert bucket.numel() >= o
    tab = _i64(0 if g is None else g.data_ptr() for g in grads)
    offs, szs = _i64(offsets), _i64(sizes)
    _lib.check(_lib.load().sae_bucket_accumulate(_p(tab), _p(offs), _p(szs), len(grads), _p(bucket), bucket.numel(), _stream()),
               "sae_bucket_accumulate")
    torch.cuda.synchronize()
    return offsets


def _bits(a, b):
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


def _same(a, b):
    return len(a) == len(b) and all(_bits(x, y) for x, y in zip(a, b))


# ------------------------------------------------------------------------------------------------ kernel
def test_accumulate_is_fp32_add_bitwise():
    g = torch.Generator(DEV).manual_seed(11)
    grads, sizes = [], []
    for size in (1, 3, 4, 5, 4097, 1000003):
        grads.append(torch.randn(size, device=DEV, generator=g) * 1e-3)
        sizes.append(size)
    base = torch.randn(5002, device=DEV, generator=g)
    grads += [base[1:], base[1:4097]]                      # storage offset 1: the unaligned, element-by-element loop
    sizes += [5001, 4096]
    grads.insert(2, None)                                  # null entries: their segments are left alone
    sizes.insert(2, 17)
    grads.append(None)
    sizes.append(4)
    total = sum((s + 3) // 4 * 4 for s in sizes)
    bucket = torch.randn(total, device=DEV, generator=g)
    bucket[::7] = 0.0
    before = bucket.clone()
    offsets = _accumulate(grads, sizes, bucket)
    want = before.clone()
    for gr, o, s in zip(grads, offsets, sizes):
        if gr is not None:
            want[o:o + s] = before[o:o + s] + gr
    assert _bits(bucket, want)
    # twice more: a + b + c in order
    again = bucket.clone()
    _accumulate(grads, sizes, bucket)
    for gr, o, s in zip(grads, offsets, sizes):
        if gr is not None:
            again[o:o + s] = again[o:o + s] + gr
    assert _bits(bucket, again)


def test_accumulate_arguments():
    lib = _lib.load()
    assert lib.sae_bucket_accumulate(None, None, None, 0, None, 0, None) == 0
    t = torch.zeros(8, device=DEV)
    tab = _i64([t.data_ptr()])
    offs, szs = _i64([0]), _i64([8])
    assert lib.sae_bucket_accumulate(None, _p(offs), _p(szs), 1, _p(t), 8, None) == -1
    assert lib.sae_bucket_accumulate(_p(tab), None, _p(szs), 1, _p(t), 8, None) == -1
    assert lib.sae_bucket_accumulate(_p(tab), _p(offs), None, 1, _p(t), 8, None) == -1
    assert lib.sae_bucket_accumulate(_p(tab), _p(offs), _p(szs), 1, None, 8, None) == -1
    assert lib.sae_bucket_accumulate(_p(tab), _p(offs), _p(szs), -1, _p(t), 8, None) == -1
    assert lib.sae_bucket_accumulate(_p(tab), _p(offs), _p(szs), 1, _p(t), -1, None) == -1
    assert lib.sae_bucket_accumulate(_p(tab), _p(offs), _p(szs), 65536, _p(t), 8, None) == -3
    torch.cuda.synchronize()


def test_accumulate_beyond_2_31_elements():
    n = (1 << 31) + 7
    g = torch.Generator(DEV).manual_seed(12)
    bucket = torch.randn(n + 1, device=DEV, generator=g)
    grad = torch.randn(n, device=DEV, generator=g)
    want = bucket[:n] + grad
    _accumulate([grad], [n], bucket)
    assert _bits(bucket[:n], want)
    del want
    want = bucket[:n - 1] + grad[1:]                       # the unaligned loop over 2^31 + 6 elements
    _accumulate([grad[1:]], [n - 1], bucket)
    assert _bits(bucket[:n - 1], want)
    del bucket, grad, want
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


def _trainer(base, **over):
    import swapping_autoencoder_pytorch_b200 as S
    opt = default_options(**dict(base, num_gpus=1, **over))
    torch.manual_seed(0)
    return S.create_optimizer(opt, S.create_model(opt))


def _state(tr):
    out = [p.detach().clone() for p in tr.model.singlegpu_model.parameters()]
    for o in (tr.optimizer_G, tr.optimizer_D):
        st = o._state()
        out += [st.exp_avg.clone(), st.exp_avg_sq.clone(), st.steps.clone()]
    return out


def _real(n, size, seed=5):
    return torch.randn(n, 3, size, size, device=DEV, generator=torch.Generator(DEV).manual_seed(seed)).clamp(-1, 1)


def _compose_update(tr, kind, chunks):
    """one accumulated update written out: the body with step=False per micro-batch, gradients summed in order, one Adam step"""
    body = {"D": tr._discriminator_body, "R1": tr._r1_body, "G": tr._generator_body}[kind]
    optimizer = tr.optimizer_G if kind == "G" else tr.optimizer_D
    total, means = None, {}
    for chunk in chunks:
        out = body(chunk, step=False)
        for k, v in out.items():
            if not k.startswith("_"):
                means.setdefault(k, []).append(v.detach().mean())
        g = [None if p.grad is None else p.grad.clone() for p in optimizer.params]
        total = g if total is None else [None if a is None else a + b for a, b in zip(total, g)]
    optimizer.step(grads=total, grad_scale=1.0 / len(chunks))
    return {k: torch.stack(v).mean() for k, v in means.items()}


def _compose_half_step(tr, chunks):
    """train_one_step of the composition: the toggle, the lazy-R1 decision, the averaged losses"""
    if tr.toggle_training_mode() == "generator":
        tr.discriminator_iter_counter += 1
        losses = _compose_update(tr, "D", chunks)
        if tr.discriminator_iter_counter % tr.opt.R1_once_every == 0:
            losses.update(_compose_update(tr, "R1", chunks))
        losses["D_total"] = sum(v.mean() for v in losses.values())
    else:
        losses = _compose_update(tr, "G", chunks)
    return {k: float(v) for k, v in losses.items()}


@pytest.mark.parametrize("precision", ["tf32", "fp32"])
@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
def test_deterministic_updates_equal_the_composition(kern, monkeypatch, precision, graphs):
    kern.precision, kern.deterministic = precision, True
    extra = {}
    if graphs:
        _zero_noise(monkeypatch)
        extra = dict(lambda_PatchGAN=0.0, lambda_patch_R1=0.0)
    real = _real(4, 256)
    tr = _trainer({}, batch_size=4, micro_batches=2, R1_once_every=2, cuda_graphs=graphs, **extra)
    ref = _trainer({}, batch_size=4, R1_once_every=2, **extra)
    torch.manual_seed(123)
    rows = []
    for _ in range(8):                                  # D, G, D + R1, G, ...: with graphs every kind is captured and replayed
        rows.append({k: float(v) for k, v in tr.train_one_step({"real_A": real}, 0).items()})
    mine = _state(tr)
    torch.manual_seed(123)
    for i in range(8):
        want = _compose_half_step(ref, [real[:2], real[2:]])
        assert rows[i] == want, (i, rows[i], want)
    assert any("D_R1" in r for r in rows)
    assert _same(mine, _state(ref))
    if graphs:
        assert tr.graphs.disabled is None, (tr.graphs.disabled, tr.graphs.last_traceback)
        assert sorted(k[0] for k in tr.graphs.captured) == ["D", "G", "R1"]
        assert all(len(k) == 6 and k[5] == 2 for k in tr.graphs.captured)


@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
def test_bucket_is_the_fp32_sum_of_the_micro_batch_gradients(kern, graphs):
    kern.deterministic = False
    tr = _trainer(TINY, batch_size=4, micro_batches=2, R1_once_every=2, cuda_graphs=graphs)
    model = tr.model
    snaps, checked = [], []
    accumulate, reduce = model.accumulate_to_bucket, model.reduce_accumulated

    def snap_accumulate(params, j):
        if j == 0:
            snaps.clear()
        snaps.append([None if p.grad is None else p.grad.clone() for p in params])
        return accumulate(params, j)

    def check_reduce():
        views = reduce()
        want = [None if a is None else a + b for a, b in zip(*snaps)]
        checked.append(all((v is None and w is None) or _bits(v, w) for v, w in zip(views, want)))
        return views
    model.accumulate_to_bucket, model.reduce_accumulated = snap_accumulate, check_reduce
    real = _real(4, 64)
    for _ in range(12):
        tr.train_one_step({"real_A": real}, 0)
    torch.cuda.synchronize()
    assert len(checked) == 15 and all(checked), checked          # 6 D, 3 R1, 6 G updates
    if graphs:
        assert tr.graphs.disabled is None, (tr.graphs.disabled, tr.graphs.last_traceback)
        assert len(tr.graphs.captured) == 3


@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
def test_two_deterministic_runs_bitwise(kern, graphs):
    kern.deterministic = True
    real = _real(4, 64)
    runs = []
    for _ in range(2):
        tr = _trainer(TINY, batch_size=4, micro_batches=2, R1_once_every=2, cuda_graphs=graphs)
        torch.manual_seed(321)
        rows = []
        for _ in range(8 if graphs else 4):             # D, G, D + R1, G (, ... until every kind replays)
            rows.append(({k: float(v) for k, v in tr.train_one_step({"real_A": real}, 0).items()}, _state(tr)))
        runs.append(rows)
        if graphs:
            assert tr.graphs.disabled is None, (tr.graphs.disabled, tr.graphs.last_traceback)
    for i, (a, b) in enumerate(zip(*runs)):
        assert a[0] == b[0], i
        assert _same(a[1], b[1]), i


@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
def test_guard_drops_an_update_poisoned_in_one_micro_batch(graphs):
    tr = _trainer(TINY, batch_size=4, micro_batches=2, R1_once_every=100, cuda_graphs=graphs, skip_nonfinite_steps=True)
    named = dict(tr.model.singlegpu_model.named_parameters())
    flag = torch.zeros(1, dtype=torch.bool, device=DEV)
    val = torch.full((1,), float("nan"), device=DEV)
    targets, handles = {}, []
    for kind, net in (("D", "Dpatch"), ("G", "E")):
        name = next(n for n in named if n.startswith(net + "."))
        targets[kind] = name
        p = named[name]

        def hook(param):
            with torch.no_grad():
                g0 = param.grad.view(-1)[:1]
                g0.copy_(torch.where(flag, val, g0))      # a device-side select: the same hook works inside a graph
        frozen = not p.requires_grad
        handles.append(p.requires_grad_(True).register_post_accumulate_grad_hook(hook))
        p.requires_grad_(not frozen)
    armed = [False]
    accumulate = tr.model.accumulate_to_bucket

    def arm_after_first(params, j):
        out = accumulate(params, j)
        flag.fill_(armed[0] and j == 0)                   # only the backward of micro-batch 1 is poisoned
        return out
    tr.model.accumulate_to_bucket = arm_after_first
    real = _real(4, 64)
    for _ in range(6):                                    # warm-up, capture and replays of D and G
        tr.train_one_step({"real_A": real}, 0)
    for kind in ("D", "G"):
        armed[0] = True
        before = _state(tr)
        tr.train_one_step({"real_A": real}, 0)
        armed[0] = False
        assert _same(_state(tr), before), kind
        assert tr.nonfinite_steps()[kind] == 1
        assert tr.nonfinite_report(kind) == {targets[kind]: 1}
    for _ in range(2):
        before = _state(tr)
        tr.train_one_step({"real_A": real}, 0)
        assert not _same(_state(tr), before)
    assert tr.nonfinite_steps() == {"D": 1, "R1": 0, "G": 1}
    for h in handles:
        h.remove()
    if graphs:
        assert tr.graphs.disabled is None, (tr.graphs.disabled, tr.graphs.last_traceback)


def test_graph_update_launches(kern, monkeypatch):
    kern.deterministic = False
    tr = _trainer(TINY, batch_size=4, micro_batches=2, R1_once_every=2, cuda_graphs=True)
    calls = []                                            # (wrapper, library launches it made)

    def spy(name, orig):
        def call(*a, **kw):
            n = _lib.launch_count()
            out = orig(*a, **kw)
            calls.append((name, _lib.launch_count() - n))
            return out
        return call
    for name in ("bucket_pack", "bucket_accumulate", "adam_step"):
        monkeypatch.setattr(kern, name, spy(name, getattr(kern, name)))
    real = _real(4, 64)
    for _ in range(8):                                    # every kind captured (R1 on its second update)
        tr.train_one_step({"real_A": real}, 0)
    assert tr.graphs.disabled is None, (tr.graphs.disabled, tr.graphs.last_traceback)
    assert sorted(k[0] for k in tr.graphs.captured) == ["D", "G", "R1"]
    per_kind = {k[0]: v[3] for k, v in tr.graphs.captured.items()}
    for kind in ("D", "G"):                               # D update 5 (no R1), G update 5: both replayed
        calls.clear()
        n0, r0 = _lib.launch_count(), tr.graphs.replayed_launches
        tr.train_one_step({"real_A": real}, 0)
        torch.cuda.synchronize()
        assert tr.graphs.replayed_launches - r0 == 2 * per_kind[kind], kind
        assert [c[0] for c in calls] == ["bucket_pack", "bucket_accumulate", "adam_step"], (kind, calls)
        assert calls[0][1] == 1 and calls[1][1] == 1, (kind, calls)        # one launch each
        # nothing else is launched eagerly: the bucket launches and the Adam update's own kernels
        assert _lib.launch_count() - n0 == sum(c[1] for c in calls), (kind, calls)
