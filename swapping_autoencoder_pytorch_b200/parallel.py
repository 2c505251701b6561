"""Data-parallel execution: one process per GPU, one NCCL all-reduce of a flat gradient bucket per backward.

Replaces reference ``models/__init__.py:75-93`` (``MultiGPUModelWrapper`` over single-process
``nn.DataParallel``: per-call parameter broadcast, scatter/gather, reduce onto GPU 0) and keeps its call
surface: ``wrapper(*args, command=...)``, ``.singlegpu_model``, ``.get_parameters_for_mode``, ``.save``,
``.opt``.  Design (SURVEY.md §8(e)):

* the batch is partitioned by image across ranks (each rank is handed its own shard; per-rank batch even);
* parameters are replicated once (broadcast from rank 0 at construction), optimizer state is replicated;
* because ``requires_grad`` is toggled between the D and G half-steps (reference optimizer :44-49), stock DDP's
  fixed reducer does not fit; instead every parameter carries a post-accumulate hook that queues ONE
  end-of-backward callback; the callback packs the gradients that exist (the active group) into a persistent
  flat fp32 bucket with a single kernel, all-reduces it (sum) over NCCL / NVLink, and unpacks scaled by
  1/world — so ``loss.backward(); optimizer.step()`` in the unchanged optimizer sees averaged gradients;
* per-sample losses are means over the local shard; the average of equal-sized shard means equals the
  reference's mean over the gathered global batch (reference optimizer :75, :93).
"""
import os

import torch
import torch.distributed as dist

from . import backend


def init_distributed(backend_name=None):
    """Join the torchrun-provided process group (no-op for a single process).  Returns (rank, world, local_rank)."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        if backend_name is None:
            backend_name = "nccl" if torch.cuda.is_available() else "gloo"
        if backend_name == "nccl":
            torch.cuda.set_device(local)
        dist.init_process_group(backend=backend_name)
    return rank, world, local


class GradientBucket:
    """Persistent flat buffer + cached device tables for the gradient tensors of one parameter set."""

    def __init__(self, device):
        self.device = device
        self.flat = None
        self.layouts = {}     # tuple of sizes -> (offsets tensor, sizes tensor, total, offsets list)
        self.tables = None    # backend.PointerTables, created with the first CUDA bucket

    def _layout(self, grads):
        key = tuple(g.numel() for g in grads)
        hit = self.layouts.get(key)
        if hit is None:
            offsets, total = [], 0
            for s in key:
                offsets.append(total)
                total += (s + 3) // 4 * 4            # keep every segment 16-byte aligned
            dev = self.device
            hit = (torch.tensor(offsets, dtype=torch.int64, device=dev), torch.tensor(key, dtype=torch.int64, device=dev), total,
                   offsets)
            self.layouts[key] = hit
        return hit

    def reserve(self, total):
        if self.flat is None or self.flat.numel() < total:
            self.flat = torch.zeros(total, dtype=torch.float32, device=self.device)

    def fill(self, grads, micro_batch=0):
        """copy the given gradient tensors into the flat bucket (micro_batch 0: sae_bucket_pack), or add them to what it holds
        (a later micro-batch of the same update, same tensors: sae_bucket_accumulate); returns one bucket view per gradient"""
        offsets_t, sizes_t, total, offsets = self._layout(grads)
        self.reserve(total)
        flat = self.flat[:total]
        if self.tables is None:
            self.tables = backend.PointerTables(max(len(grads), 1024), self.device)
        ptrs = self.tables.get(tuple(g.data_ptr() for g in grads))
        k = backend.kernels()
        if micro_batch == 0:
            k.bucket_pack(ptrs, offsets_t, sizes_t, len(grads), flat)
        else:
            k.bucket_accumulate(ptrs, offsets_t, sizes_t, len(grads), flat)
        return [flat[o:o + g.numel()].view_as(g) for o, g in zip(offsets, grads)], (ptrs, offsets_t, sizes_t, flat)

    def pack_all_reduce(self, grads):
        """SUM over ranks of the given gradient tensors, left in the flat bucket; returns one bucket view per gradient"""
        views, info = self.fill(grads)
        dist.all_reduce(info[3])
        return views, info

    def all_reduce_mean(self, grads, world):
        if not grads:
            return
        if self.device.type != "cuda":
            # host path used by the gloo unit tests: same flatten / reduce / scatter-back arithmetic in torch
            flat = torch.cat([g.reshape(-1) for g in grads])
            dist.all_reduce(flat)
            flat.div_(world)
            o = 0
            for g in grads:
                g.copy_(flat[o:o + g.numel()].view_as(g))
                o += g.numel()
            return
        _, (ptrs, offsets_t, sizes_t, flat) = self.pack_all_reduce(grads)
        backend.kernels().bucket_unpack(ptrs, offsets_t, sizes_t, len(grads), flat, 1.0 / world)


class MultiGPUModelWrapper:
    def __init__(self, opt, model):
        self.opt = opt
        self.world = dist.get_world_size() if dist.is_initialized() else 1
        self.rank = dist.get_rank() if dist.is_initialized() else 0
        if opt.num_gpus > 0:
            model = model.to(torch.device("cuda", torch.cuda.current_device()))
        self.singlegpu_model = model
        self.parallelized_model = model          # attribute kept for callers of the reference wrapper
        self.device = next(model.parameters()).device
        self._pending = False
        self.suspend_reduce = False           # set while a half-step is being captured into a CUDA graph (graphs.py)
        # set by an optimizer that calls reduce_to_bucket() itself and reads the bucket (optimizer.py): the end-of-backward
        # callback, which averages INTO p.grad for a stock optimizer, is then not queued
        self.defer_to_optimizer = False
        self._bucket = GradientBucket(self.device)
        self._accumulated = None     # (flat, views, which params have a gradient) of the update being accumulated
        model(command="per_gpu_initialize")
        if self.world > 1:
            with torch.no_grad():
                for t in list(model.parameters()) + list(model.buffers()):
                    dist.broadcast(t, src=0)
            for p in model.parameters():
                p.register_post_accumulate_grad_hook(self._on_grad)

    # the hook fires once per parameter per backward; only the first one queues the callback
    def _on_grad(self, param):
        if self.suspend_reduce or self.defer_to_optimizer:
            return
        if not self._pending:
            self._pending = True
            torch.autograd.Variable._execution_engine.queue_callback(self._reduce_gradients)

    def _reduce_gradients(self):
        self._pending = False
        grads = [p.grad for p in self.singlegpu_model.parameters()
                 if p.requires_grad and p.grad is not None]
        self._bucket.all_reduce_mean(grads, self.world)

    def reduce_gradients_now(self):
        """explicit form of the end-of-backward callback (used after a CUDA-graph replay, where autograd does not run)"""
        if self.world > 1:
            self._reduce_gradients()

    def reduce_to_bucket(self, params):
        """Gradient exchange for an optimizer that reads the bucket directly (optimizer.MultiTensorAdam.step(grads=...)):
        packs the existing gradients of ``params``, all-reduces (SUM) and returns a list aligned with ``params`` of views
        into the flat bucket (None where a parameter has no gradient).  Nothing is written back to ``p.grad``: the 1/world
        factor is the optimizer's ``grad_scale``.  On a CPU group (gloo tests) the views hold the same sums."""
        present = [p for p in params if p.grad is not None]
        if not present:
            return [None] * len(params)
        if self.device.type != "cuda":
            flat = torch.cat([p.grad.reshape(-1) for p in present])
            dist.all_reduce(flat)
            views, o = [], 0
            for p in present:
                views.append(flat[o:o + p.numel()].view_as(p))
                o += p.numel()
        else:
            views, _ = self._bucket.pack_all_reduce([p.grad for p in present])
        it = iter(views)
        return [next(it) if p.grad is not None else None for p in params]

    def accumulate_to_bucket(self, params, micro_batch):
        """Gradient accumulation (opt.micro_batches > 1), called after each micro-batch's backward: micro-batch 0 packs the
        existing gradients of ``params`` into the flat bucket, every later one adds its gradients (the same tensors) to it, in
        micro-batch order.  At world size 1 the bucket is only this sum; D and G share it, as their updates never overlap.
        ``reduce_accumulated`` ends the update.  On a CPU device (the gloo tests) the same sums are formed in torch."""
        present = [p.grad is not None for p in params]
        grads = [p.grad for p in params if p.grad is not None]
        if micro_batch == 0:
            self._accumulated = None
        elif self._accumulated is None or self._accumulated[2] != present:
            raise RuntimeError("accumulate_to_bucket: micro-batch %d has other gradients than micro-batch 0" % micro_batch)
        if not grads:
            self._accumulated = (None, [], present)
            return
        if self.device.type != "cuda":
            flat = torch.cat([g.reshape(-1) for g in grads])
            if micro_batch == 0:
                views, o = [], 0
                for g in grads:
                    views.append(flat[o:o + g.numel()].view_as(g))
                    o += g.numel()
                self._accumulated = (flat, views, present)
            else:
                self._accumulated[0].add_(flat)
            return
        views, (_, _, _, flat) = self._bucket.fill(grads, micro_batch)
        self._accumulated = (flat, views, present)

    def reduce_accumulated(self):
        """the summed gradients of the update's micro-batches, all-reduced (SUM) once over the ranks when world > 1: a list
        aligned with the ``params`` given to ``accumulate_to_bucket`` of bucket views (None where a parameter has no gradient)"""
        flat, views, present = self._accumulated
        self._accumulated = None
        if self.world > 1 and flat is not None:
            dist.all_reduce(flat)
        it = iter(views)
        return [next(it) if has else None for has in present]

    def get_parameters_for_mode(self, mode):
        return self.singlegpu_model.get_parameters_for_mode(mode)

    def save(self, total_steps_so_far):
        if self.rank == 0:
            self.singlegpu_model.save(total_steps_so_far)

    def shard(self, batch):
        """This rank's slice of a global batch (dim 0), mirroring DataParallel's scatter."""
        if self.world == 1:
            return batch
        n = batch.shape[0]
        assert n % self.world == 0, "global batch must divide evenly across ranks"
        per = n // self.world
        return batch[self.rank * per:(self.rank + 1) * per]

    def __call__(self, *args, **kwargs):
        self._pending = False        # a backward that raised after queueing the callback must not block the next one
        return self.singlegpu_model(*args, **kwargs)
