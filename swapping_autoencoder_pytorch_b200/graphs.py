"""CUDA-graph execution of the training half-steps (extension; SURVEY.md Appendix B "launch-count pressure").

One half-step of the reference optimizer (``optimizers/swapping_autoencoder_optimizer.py:67-111``) is ~1200 kernel
launches issued from Python through autograd; on the GPU the kernels of a 256x256 batch finish about as fast as the
host can issue them, and at the small per-GPU batches of the reference's own multi-GPU configurations the host is the
bottleneck outright.  The step has static shapes and no host-visible control flow between "images in" and "losses
out" — the lazy-R1 decision is a host counter, the D / G toggle too — so each body (D, G, R1) is captured ONCE into a
``torch.cuda.CUDAGraph`` (forward, backward, and at world size 1 the fused Adam step) and replayed afterwards with the
images copied into a static input buffer.

* The first ``warmup`` calls of every body run eagerly (lazy initialisation inside the kernels library, Adam state).
* All graphs share one memory pool: bodies never run concurrently.
* Random draws (NoiseInjection, crop windows) use torch's graph-safe Philox generator: every replay draws fresh numbers.
* Data parallel (world > 1): the graph holds forward + backward only; the gradient all-reduce (``parallel.py``) and the
  Adam step run eagerly after the replay on the graph's static gradient buffers — no NCCL call is captured.
* A body that fails to capture falls back to eager execution for the rest of the run (``self.disabled`` holds why).
"""
import gc
import os
import traceback
import warnings

import torch

from . import _lib, backend


class HalfStepGraphs:
    def __init__(self, trainer, warmup=2):
        self.trainer = trainer
        self.warmup = warmup
        self.calls = {}
        self.captured = {}        # (kind, input shape, kernel precision, deterministic) -> (graph, static_input, static_outputs, launches)
        self.pool = None
        self.stream = None             # side stream shared by the eager warm-up calls and every capture (see _side)
        self.disabled = None
        self.last_traceback = None
        self.replayed_launches = 0     # kernels of this library executed through graph replays (bench bookkeeping)
        self.enabled = True            # bench switches to eager for its per-launch instrumentation pass
        # data parallel, opt-in (SAE_GRAPH_NCCL=1): capture pack -> NCCL all-reduce -> Adam into the graph as well (one replay = one
        # whole half-step); falls back to the eager tail if the collective cannot be captured.  Default off: with the lazy loss
        # read-back the host already runs ahead, so the eager tail (3 launches + the collective) costs only its device time,
        # and a process that holds captured NCCL kernels can hang in destroy_process_group at exit.
        self.nccl_in_graph = os.environ.get("SAE_GRAPH_NCCL", "0") == "1"
        self.nccl_capture_error = None
        # bench.py sets this to a list to get (start, replay done, exchange + Adam done) CUDA events of every replayed half-step
        self.phase_events = None

    # ------------------------------------------------------------------
    def _wrapper(self):
        return self.trainer.model

    def _world(self):
        return getattr(self._wrapper(), "world", 1)

    def _optimizer(self, kind):
        return self.trainer.optimizer_G if kind == "G" else self.trainer.optimizer_D

    def _tail(self, kind):
        """world > 1: pack the static gradient buffers, all-reduce, Adam reading the bucket (optimizer.exchange_and_step)"""
        self.trainer.exchange_and_step(self._optimizer(kind), self._params(kind))

    def _side(self, fn):
        """Run ``fn`` on the capture stream.  The warm-up calls must run where the capture will: autograd remembers
        the stream a parameter's gradient-accumulation node was created on, and a capture that has to synchronise
        with the (non-capturing) default stream for such a node is invalid."""
        if self.stream is None:
            self.stream = torch.cuda.Stream()
        cur = torch.cuda.current_stream()
        self.stream.wait_stream(cur)
        with torch.cuda.stream(self.stream):
            out = fn()
        cur.wait_stream(self.stream)
        return out

    def _give_up(self, kind, err):
        self.disabled = "%s: %s" % (type(err).__name__, (str(err).splitlines() or ["?"])[0][:200])
        self.last_traceback = traceback.format_exc()
        warnings.warn("CUDA-graph capture of the %s half-step failed (%s); continuing eagerly\n%s"
                      % (kind, self.disabled, self.last_traceback))
        self._recover()

    def _recover(self):
        torch.cuda.synchronize()
        try:
            # a capture that died half-way can leave torch's CUDA generator in "capturing" state; one empty, successful
            # capture cycle resets it so that eager random draws work again
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                torch.zeros(1, device="cuda")
            del g
        except Exception:      # noqa: BLE001
            pass
        torch.cuda.synchronize()

    def run(self, kind, body, images):
        if self.disabled is not None or not self.enabled:
            return body(images)
        # a graph records the kernels of one precision mode (backend.CudaKernels.precision): switching the mode captures new
        # graphs, after warm-up calls of their own (the other mode's kernels initialise lazily, outside any capture).  The same
        # holds for the deterministic mode (backend.CudaKernels.deterministic_mode()), which records other kernels.
        k = backend.kernels()
        precision = getattr(k, "precision", "tf32")
        det = bool(getattr(k, "deterministic_mode", lambda: False)())
        n = self.calls.get((kind, precision, det), 0)
        self.calls[(kind, precision, det)] = n + 1
        key = (kind, tuple(images.shape), precision, det)
        hit = self.captured.get(key)
        if hit is None:
            if n < self.warmup:
                return self._side(lambda: body(images))
            try:
                try:
                    hit = self._capture(key, body, images, self.nccl_in_graph)
                except Exception as e:      # noqa: BLE001
                    if not (self.nccl_in_graph and self._world() > 1):
                        raise
                    # the collective could not be captured on this stack: keep the graph for forward + backward and run the
                    # exchange + Adam eagerly after every replay
                    self.nccl_in_graph = False
                    self.nccl_capture_error = "%s: %s" % (type(e).__name__, (str(e).splitlines() or ["?"])[0][:200])
                    self._recover()
                    hit = self._capture(key, body, images, False)
            except Exception as e:      # noqa: BLE001 — any capture failure means "run eagerly", never "stop training"
                self._give_up(kind, e)
                return body(images)
        graph, static_in, outputs, launches, grads, tail_captured = hit
        # host-side state the eager body would have left behind: which group is trainable, and which gradient buffers
        # the parameters point at (every graph owns its own static set)
        self._select_group(kind)
        for p, g in grads:
            p.grad = g
        with torch.no_grad():            # the R1 body marks its input as requiring grad
            static_in.copy_(images, non_blocking=True)
        ev = None
        if self.phase_events is not None:
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            ev[0].record()
        graph.replay()
        self.replayed_launches += launches
        if ev is not None:
            ev[1].record()
        if self._world() > 1 and not tail_captured:
            self._tail(kind)
        if ev is not None:
            ev[2].record()
            self.phase_events.append((kind, ev))
        return dict(outputs)

    def release(self):
        """drop every captured graph (call before tearing the process group down when collectives were captured)"""
        torch.cuda.synchronize()
        self.captured.clear()
        self.pool = None
        gc.collect()
        torch.cuda.synchronize()

    def describe(self, world):
        """one-line account of what a replay contains (bench.py reports it)"""
        if world == 1:
            return "forward+backward+Adam per replay"
        if self.nccl_in_graph:
            return "forward+backward+bucket pack+NCCL all-reduce+Adam per replay"
        return "forward+backward per replay; bucket pack, NCCL all-reduce and Adam (reading the bucket) issued after it%s" % (
            " (%s)" % self.nccl_capture_error if self.nccl_capture_error else "")

    def _select_group(self, kind):
        t = self.trainer
        t.set_requires_grad(t.Dparams, kind != "G")
        t.set_requires_grad(t.Gparams, kind == "G")

    def _params(self, kind):
        return self.trainer.Gparams if kind == "G" else self.trainer.Dparams

    def warm_up(self, images):
        """Run every body often enough that all three graphs exist (benchmarks call this before their timed region;
        it performs real optimizer steps, including extra R1 steps)."""
        t = self.trainer
        for _ in range(self.warmup + 1):
            for kind, body in (("D", t._discriminator_body), ("R1", t._r1_body), ("G", t._generator_body)):
                self.run(kind, body, images)
        torch.cuda.synchronize()

    def _capture(self, key, body, images, with_tail=False):
        kind = key[0]
        world = self._world()
        wrapper = self._wrapper()
        static_in = torch.empty_like(images).requires_grad_(False)
        with torch.no_grad():
            static_in.copy_(images)
        for p in self._params(kind):
            p.grad = None                    # gradients of the eager calls: the capture allocates its own static set
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        if self.stream is None:
            self.stream = torch.cuda.Stream()
        if self.pool is None:
            self.pool = torch.cuda.graph_pool_handle()
        n0 = _lib.launch_count()
        if world > 1:
            wrapper.suspend_reduce = True
        # no cyclic garbage collection while the stream is capturing: a collected object that owns device memory or an
        # older CUDA graph would issue cudaFree / cudaGraphExecDestroy in the middle of the capture and invalidate it
        gc.collect()
        gc_was_enabled = gc.isenabled()
        gc.disable()
        try:
            with torch.cuda.graph(graph, pool=self.pool, stream=self.stream):
                outputs = body(static_in, step=(world == 1))
                if world > 1 and with_tail:
                    self._tail(kind)
        finally:
            if gc_was_enabled:
                gc.enable()
            if world > 1:
                wrapper.suspend_reduce = False
        launches = _lib.launch_count() - n0
        outputs = {k: v for k, v in outputs.items() if torch.is_tensor(v)}
        grads = [(p, p.grad) for p in self._params(kind)]      # None where the body produces no gradient (R1: final bias)
        hit = (graph, static_in, outputs, launches, grads, bool(world > 1 and with_tail))
        self.captured[key] = hit
        return hit
