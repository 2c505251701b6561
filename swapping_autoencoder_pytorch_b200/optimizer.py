"""Training driver of the hot path: alternating discriminator / generator half-steps with lazy R1.

Restates reference ``optimizers/swapping_autoencoder_optimizer.py:7-119`` (same public methods, same Adam
hyper-parameters and R1 schedule) for boxes without the reference checkout.  The data-parallel gradient
exchange is invisible here: ``MultiGPUModelWrapper`` (parallel.py) all-reduces the active parameter group at
the end of every ``backward()``.
"""
import math
import os

import torch

from . import _lib, augment, backend, util


class MultiTensorAdam:
    """``torch.optim.Adam`` for one parameter group as ONE kernel launch (``sae_adam_step``, SURVEY.md §8 f2) — the subset of
    the torch optimizer interface the reference driver uses (``zero_grad`` / ``step`` / ``state_dict`` / ``load_state_dict`` /
    ``param_groups``; reference optimizers/swapping_autoencoder_optimizer.py:34-42, :76, :94).  Same arithmetic and the same
    per-parameter semantics: a parameter without a gradient is skipped and keeps its own step count.  Moments live in two
    flat fp32 buffers, step counts on the device, so the update is capturable in a CUDA graph.  ``step(grads=...)`` lets the
    data-parallel path hand in views of the flat all-reduce bucket with ``grad_scale = 1 / world`` (no unpack pass)."""

    def __init__(self, params, lr, betas=(0.9, 0.999), eps=1e-8):
        self.params = list(params)
        self.param_groups = [dict(params=self.params, lr=float(lr), betas=(float(betas[0]), float(betas[1])), eps=float(eps),
                                  weight_decay=0, amsgrad=False, maximize=False)]
        sizes, offsets, total = [], [], 0
        for p in self.params:
            sizes.append(p.numel())
            offsets.append(total)
            total += (p.numel() + 3) // 4 * 4          # every segment 16-byte aligned
        self._sizes, self._offsets, self._total = sizes, offsets, total
        self._dev = None
        self._cache = None

    def _state(self):
        if self._dev is None:
            dev = self.params[0].device
            self.exp_avg = torch.zeros(self._total, dtype=torch.float32, device=dev)
            self.exp_avg_sq = torch.zeros(self._total, dtype=torch.float32, device=dev)
            self.steps = torch.zeros(len(self.params), dtype=torch.float32, device=dev)
            self.offsets_t = torch.tensor(self._offsets, dtype=torch.int64, device=dev)
            self.sizes_t = torch.tensor(self._sizes, dtype=torch.int64, device=dev)
            self._cache = backend.PointerTables(len(self.params), dev)
            self._dev = dev
        return self

    def zero_grad(self, set_to_none=True):
        for p in self.params:
            if set_to_none:
                p.grad = None
            elif p.grad is not None:
                p.grad.detach_().zero_()

    @torch.no_grad()
    def step(self, grads=None, grad_scale=1.0, guard=None):
        """guard: a ``NonfiniteGuard`` — scan the gradients this update reads and drop the update on the device when any
        element is not finite (opt.skip_nonfinite_steps).  Returns the guard's device skip word (None without a guard)."""
        st = self._state()
        g = self.param_groups[0]
        if grads is None:
            grads = [p.grad for p in self.params]
        grads = [None if t is None else (t if t.is_contiguous() else t.contiguous()) for t in grads]
        if all(t is None for t in grads):
            return
        params = self.params
        if st.exp_avg.dtype != params[0].dtype:           # fp64 runs of the CPU test-suite
            st.exp_avg, st.exp_avg_sq = st.exp_avg.to(params[0].dtype), st.exp_avg_sq.to(params[0].dtype)
        kw = {} if guard is None else {"skip": guard.scan(grads, st.sizes_t, self._cache)}
        backend.kernels().adam_step(params, grads, st.offsets_t, st.sizes_t, st.exp_avg, st.exp_avg_sq, st.steps, g["lr"],
                                    g["betas"][0], g["betas"][1], g["eps"], float(grad_scale), self._cache, **kw)
        return kw.get("skip")

    # torch.optim.Adam's on-disk format, so optimizer checkpoints interoperate with the stock optimizer
    def state_dict(self):
        st = self._state()
        state = {}
        for i, (o, n, p) in enumerate(zip(self._offsets, self._sizes, self.params)):
            if float(st.steps[i]) == 0.0:
                continue
            state[i] = {"step": st.steps[i].detach().clone().cpu(), "exp_avg": st.exp_avg[o:o + n].view_as(p).clone(),
                        "exp_avg_sq": st.exp_avg_sq[o:o + n].view_as(p).clone()}
        group = {k: v for k, v in self.param_groups[0].items() if k != "params"}
        group["params"] = list(range(len(self.params)))
        return {"state": state, "param_groups": [group]}

    def load_state_dict(self, sd):
        st = self._state()
        group = sd["param_groups"][0]
        assert len(group["params"]) == len(self.params), "optimizer state belongs to a different parameter list"
        for k in ("lr", "betas", "eps"):
            if k in group:
                self.param_groups[0][k] = tuple(group[k]) if k == "betas" else group[k]
        st.exp_avg.zero_()
        st.exp_avg_sq.zero_()
        st.steps.zero_()
        for i, entry in sd["state"].items():
            i = int(i)
            o, n = self._offsets[i], self._sizes[i]
            st.exp_avg[o:o + n].copy_(entry["exp_avg"].reshape(-1))
            st.exp_avg_sq[o:o + n].copy_(entry["exp_avg_sq"].reshape(-1))
            st.steps[i] = float(entry["step"])


class NonfiniteGuard:
    """Device state of the skip-on-non-finite guard for one kind of half-step (D, R1 or G).  ``scan`` counts the non-finite
    elements of the gradients Adam is about to read (one kernel) and returns the total as the ``skip`` argument of the
    guarded update; it also advances this kind's skip counter and, when the total is non-zero, keeps the per-tensor counts
    as the report.  All of it stays on the device, so it is capturable and costs no host sync."""

    def __init__(self, n, skipped):
        dev = skipped.device
        self.counts = torch.zeros(n + 1, dtype=torch.int64, device=dev)     # the latest scan: per tensor, then the total
        self.report = torch.zeros(n, dtype=torch.int64, device=dev)         # the latest scan with a non-zero total
        self.skipped = skipped                                              # one-element view of the trainer's counters

    def scan(self, grads, sizes, cache):
        self.counts.zero_()
        backend.kernels().nonfinite_count(grads, sizes, self.counts, cache)
        total = self.counts[-1:]
        bad = total != 0
        self.skipped.add_(bad)
        torch.where(bad, self.counts[:-1], self.report, out=self.report)
        return total


class ParameterEMA:
    """Exponential moving average of one parameter group (opt.ema_kimg; INTEGRATION.md §2f): a flat shadow in the layout of
    the group's ``MultiTensorAdam`` moments, initialised to a copy of the parameters, and the number of averaging updates
    made, both on the device.  ``update`` is one launch pair (sae_ema_update) that forms beta from that counter on the
    device, so it is capturable and one captured graph serves every step of the ramp."""

    def __init__(self, adam, names, half_life_images, rampup):
        self.adam = adam                      # layout (offsets_t, sizes_t) and pointer-table cache
        self.names = list(names)              # state_dict keys of adam.params
        self.half_life_images = float(half_life_images)
        self.rampup = float(rampup)
        adam._state()
        p0 = adam.params[0]
        self.shadow = torch.zeros(adam._total, dtype=p0.dtype, device=p0.device)
        self.updates = torch.zeros(1, dtype=torch.int64, device=p0.device)
        with torch.no_grad():
            for v, p in zip(self.averaged(), adam.params):
                v.copy_(p)

    def averaged(self):
        """one view of the shadow per parameter, shaped like it"""
        return [self.shadow[o:o + n].view_as(p) for o, n, p in zip(self.adam._offsets, self.adam._sizes, self.adam.params)]

    @torch.no_grad()
    def update(self, images_per_update, skip=None):
        """one averaging update after the group's Adam update; images_per_update: the update's global batch (rank's images
        times world); skip: the guard's device skip word of that Adam update (a dropped update drops this one too)"""
        st = self.adam._state()
        backend.kernels().ema_update(self.adam.params, st.offsets_t, st.sizes_t, self.shadow, self.updates,
                                     float(images_per_update), self.half_life_images, self.rampup, st._cache, skip=skip)

    def state_dict(self):
        return {"shadow": {n: v.detach().clone() for n, v in zip(self.names, self.averaged())}, "t": int(self.updates.item())}

    def load_state_dict(self, sd):
        """in place: captured graphs hold the shadow and the counter"""
        with torch.no_grad():
            for n, v in zip(self.names, self.averaged()):
                v.copy_(sd["shadow"][n])
            self.updates.fill_(int(sd["t"]))


NONFINITE_KINDS = ("D", "R1", "G")


# the discriminator logits the model hands to the statistics' sink (model.SwappingAutoencoderModel.score_sink), by half-step
STATS_SCORES = (("D", "real"), ("D", "rec"), ("D", "mix"), ("D", "patch_real"), ("D", "patch_mix"),
                ("G", "rec"), ("G", "mix"), ("G", "patch_mix"))
STATS_NORMS = ("grad_norm", "weight_norm", "update_norm")


class TrainingStats:
    """Training statistics accumulated on the device (opt.training_stats; INTEGRATION.md §2g).  One flat fp64 window holds,
    per kind of update (D, R1, G): the number of applied updates, then per tensor the squared L2 norms of the gradient Adam
    read (grad_scale included), of the parameter after the update and of the step Adam applied; after them four sums (score,
    sign, finite count, non-finite count) per discriminator logit tensor of ``STATS_SCORES``.  ``record_update`` is four
    launches (sae_sumsq, sae_adam_norms) after the group's Adam update and ``score`` one (sae_score_stats); none reads
    anything back, so both are capturable.  ``read`` is the only device-to-host transfer."""

    def __init__(self, groups, device, world=1):
        self.groups = groups                    # {kind: (MultiTensorAdam, state_dict keys of its params)}
        self.world = world
        self._at, o = {}, 0
        for kind in NONFINITE_KINDS:
            self._at[kind] = o                  # [updates, grad_sq[n], weight_sq[n], update_sq[n]]
            o += 1 + 3 * len(groups[kind][1])
        self._scores_at = o
        self.window = torch.zeros(o + 4 * len(STATS_SCORES), dtype=torch.float64, device=device)
        n = max(len(names) for _, names in groups.values())
        self.partials = torch.zeros(max(2 * n * _lib.SAE_STATS_BLOCKS, 1), dtype=torch.float64, device=device)
        self._score_index = {k: i for i, k in enumerate(STATS_SCORES)}

    def _views(self, kind):
        o, n = self._at[kind], len(self.groups[kind][1])
        w = self.window
        return w[o:o + 1], w[o + 1:o + 1 + n], w[o + 1 + n:o + 1 + 2 * n], w[o + 1 + 2 * n:o + 1 + 3 * n]

    @torch.no_grad()
    def record_update(self, kind, grads, grad_scale, skip=None):
        """after the Adam update of ``kind``: grads as that update read them (None: the parameters' .grad), grad_scale its
        factor, skip the guard's device skip word (a dropped update adds nothing, to the update count included)"""
        adam = self.groups[kind][0]
        if grads is None:
            grads = [p.grad for p in adam.params]
        grads = [None if t is None else (t if t.is_contiguous() else t.contiguous()) for t in grads]
        if all(t is None for t in grads):
            return                              # MultiTensorAdam.step made no update either
        st = adam._state()
        g = adam.param_groups[0]
        updates, grad_sq, weight_sq, update_sq = self._views(kind)
        k = backend.kernels()
        k.sumsq(grads, st.sizes_t, grad_sq, self.partials, st._cache, scale=float(grad_scale), skip=skip)
        k.adam_norms(adam.params, grads, st.offsets_t, st.sizes_t, st.exp_avg, st.exp_avg_sq, st.steps, g["lr"], g["betas"][0],
                     g["betas"][1], g["eps"], weight_sq, update_sq, updates, self.partials, st._cache, skip=skip)

    @torch.no_grad()
    def score(self, kind, name, logits):
        """the model's sink: add one discriminator logit tensor of the ``kind`` half-step to the window"""
        o = self._scores_at + 4 * self._score_index[(kind, name)]
        backend.kernels().score_stats(logits.detach(), self.window[o:o + 4])

    def read(self, reset=True, per_tensor=False):
        """the window as plain floats (see SwappingAutoencoderOptimizer.training_stats); one device-to-host copy.  With more
        than one rank the score sums are all-reduced first, so every rank must call this."""
        src = self.window
        if self.world > 1:
            import torch.distributed as dist
            scores = self.window[self._scores_at:].clone()
            dist.all_reduce(scores)
            src = torch.cat([self.window[:self._scores_at], scores])
        vals = src.cpu().tolist()
        if reset:
            self.window.zero_()                 # in place: captured graphs hold the window
        out, pt = {}, {}
        for kind in NONFINITE_KINDS:
            o, names = self._at[kind], self.groups[kind][1]
            n, u = len(names), vals[self._at[kind]]
            out[kind + "/updates"] = int(u)
            for j, stat in enumerate(STATS_NORMS):
                seg = vals[o + 1 + j * n:o + 1 + (j + 1) * n]
                out["%s/%s" % (kind, stat)] = math.sqrt(sum(seg) / u) if u else 0.0
                if per_tensor:
                    for key, v in zip(names, seg):
                        pt.setdefault(key, {})["%s/%s" % (kind, stat)] = math.sqrt(v / u) if u else 0.0
        for i, (kind, name) in enumerate(STATS_SCORES):
            s, sign, finite, bad = vals[self._scores_at + 4 * i:self._scores_at + 4 * i + 4]
            out["%s/scores/%s" % (kind, name)] = s / finite if finite else 0.0
            out["%s/signs/%s" % (kind, name)] = sign / finite if finite else 0.0
            out["%s/scores/%s/nonfinite" % (kind, name)] = int(bad)
        if per_tensor:
            out["per_tensor"] = pt
        return out


class SwappingAutoencoderOptimizer:
    @staticmethod
    def modify_commandline_options(parser, is_train):
        parser.add_argument("--lr", default=0.002, type=float)
        parser.add_argument("--beta1", default=0.0, type=float)
        parser.add_argument("--beta2", default=0.99, type=float)
        parser.add_argument("--R1_once_every", default=16, type=int,
                            help="lazy R1 regularization: the R1 loss is computed once every this many D iterations")
        parser.add_argument("--micro_batches", default=1, type=int,
                            help="gradient accumulation (extension): split each rank's batch into this many micro-batches and "
                                 "make one Adam update from their summed gradients")
        parser.add_argument("--ema_kimg", default=0.0, type=float,
                            help="weight averaging (extension): half-life, in thousands of images, of an exponential moving "
                                 "average of the E and G weights, saved as <N>k_ema_checkpoint.pth; 0 turns it off")
        parser.add_argument("--ema_rampup", default=0.05, type=float,
                            help="ramp-up of the average's half-life: at most this fraction of the images seen so far; "
                                 "0: no ramp")
        parser.add_argument("--training_stats", type=util.str2bool, nargs="?", const=True, default=False,
                            help="training statistics (extension): accumulate per-update gradient, weight and Adam-step norms "
                                 "and the discriminators' scores on the device; read them with trainer.training_stats()")
        parser.add_argument("--augment_p", default=0.0, type=float,
                            help="adaptive discriminator augmentation (extension): probability of each transform of D's inputs; "
                                 "the initial value when --ada_target > 0")
        parser.add_argument("--ada_target", default=0.0, type=float,
                            help="tune the augmentation probability on the device towards E[sign(D(real))] = this value "
                                 "(StyleGAN2-ADA uses 0.6); 0: no tuning")
        parser.add_argument("--ada_kimg", default=500.0, type=float,
                            help="thousands of images over which the tuned probability can move by one")
        parser.add_argument("--ada_interval", default=4, type=int, help="tune the probability every this many D updates")
        return parser

    def __init__(self, model):
        self.opt = opt = model.opt
        self.model = model
        self.train_mode_counter = 0
        self.discriminator_iter_counter = 0
        self.Gparams = model.get_parameters_for_mode("generator")
        self.Dparams = model.get_parameters_for_mode("discriminator")
        on_cuda = bool(self.Gparams and self.Gparams[0].is_cuda)
        # CUDA-graph execution of the half-steps (extension, ``opt.cuda_graphs``): see graphs.py
        self.graphs = None
        if on_cuda and getattr(opt, "cuda_graphs", False):
            from .graphs import HalfStepGraphs
            self.graphs = HalfStepGraphs(self)
        # data parallel: this driver exchanges the gradients itself and hands the flat bucket to Adam (no unpack pass, the
        # 1/world factor folded into the update); the wrapper's end-of-backward averaging into p.grad — what a stock optimizer
        # needs — is switched off
        self.world = getattr(model, "world", 1)
        if self.world > 1:
            model.defer_to_optimizer = True
        self.optimizer_G = MultiTensorAdam(self.Gparams, lr=opt.lr, betas=(opt.beta1, opt.beta2))
        # lazy regularisation correction of lr and betas (StyleGAN2 appendix B; reference :38-42)
        c = opt.R1_once_every / (1 + opt.R1_once_every)
        self.optimizer_D = MultiTensorAdam(self.Dparams, lr=opt.lr * c, betas=(opt.beta1 ** c, opt.beta2 ** c))
        # skip-on-non-finite guard (extension, ``opt.skip_nonfinite_steps``): created on first use
        self._nonfinite_skipped = None      # device int64 [3]: skipped half-steps per kind, NONFINITE_KINDS order
        self._nonfinite_guards = {}
        # weight averaging (extension, ``opt.ema_kimg`` > 0): the shadow is a copy of E and G as they are now, after any
        # continue_train checkpoint the model loaded
        self.ema = None
        ema_kimg, ema_rampup = float(getattr(opt, "ema_kimg", 0.0)), float(getattr(opt, "ema_rampup", 0.05))
        if not (ema_kimg >= 0.0 and ema_rampup >= 0.0):
            raise ValueError("opt.ema_kimg and opt.ema_rampup must be >= 0, got %r and %r" % (ema_kimg, ema_rampup))
        if ema_kimg > 0.0:
            names = {id(p): n for n, p in self._inner().named_parameters()}
            self.ema = ParameterEMA(self.optimizer_G, [names[id(p)] for p in self.Gparams], ema_kimg * 1000.0, ema_rampup)
        # training statistics (extension, ``opt.training_stats``): the window lives outside any graph pool, like the shadow
        self.stats = None
        if getattr(opt, "training_stats", False) and self.Gparams:
            names = {id(p): n for n, p in self._inner().named_parameters()}
            d_names, g_names = [names[id(p)] for p in self.Dparams], [names[id(p)] for p in self.Gparams]
            self.stats = TrainingStats({"D": (self.optimizer_D, d_names), "R1": (self.optimizer_D, d_names),
                                        "G": (self.optimizer_G, g_names)}, self.Gparams[0].device, world=self.world)
            inner = self._inner()
            if hasattr(inner, "score_sink"):    # this package's model; the reference's own model file has no sink
                inner.score_sink = self.stats.score
        # adaptive discriminator augmentation (extension, ``opt.augment_p`` > 0 or ``opt.ada_target`` > 0): p and the sign
        # sums live outside any graph pool, like the shadow
        self.augment = None
        ada = (float(getattr(opt, "augment_p", 0.0)), float(getattr(opt, "ada_target", 0.0)),
               float(getattr(opt, "ada_kimg", 500.0)), getattr(opt, "ada_interval", 4))
        if augment.check_options(*ada) and self.Gparams:
            self.augment = augment.AugmentPipe(*ada, self.Gparams[0].device, world=self.world)
            inner = self._inner()
            if hasattr(inner, "augment_pipe"):  # this package's model; the reference's own model file has no hook
                inner.augment_pipe = self.augment

    def _inner(self):
        return getattr(self.model, "singlegpu_model", self.model)

    def ema_key(self):
        """what a captured G graph bakes in of the average: () when it is off, so the graph keys stay as they were"""
        return () if self.ema is None else (("ema", self.ema.half_life_images, self.ema.rampup),)

    def stats_key(self):
        """what a captured graph bakes in of the statistics: () when they are off, so the graph keys stay as they were"""
        return () if self.stats is None else (("stats",),)

    def augment_key(self):
        """what a captured graph bakes in of the augmentation: () when it is off, so the graph keys stay as they were"""
        return () if self.augment is None else (("ada",),)

    def augment_p(self):
        """the current augmentation probability p (opt.augment_p, tuned with opt.ada_target > 0); one device-to-host read"""
        if self.augment is None:
            raise RuntimeError("no augmentation: opt.augment_p and opt.ada_target are 0")
        return self.augment.value()

    def training_stats(self, reset=True, per_tensor=False):
        """The statistics accumulated since the last reset (opt.training_stats; INTEGRATION.md §2g), as plain floats, with
        one device-to-host copy:
        * "<kind>/updates" for kind in D, R1, G: the applied updates (a dropped one is in ``nonfinite_steps()`` instead);
        * "<kind>/grad_norm", "/weight_norm", "/update_norm": the group's L2 norm of the gradient Adam read, of the parameters
          after the update and of the step Adam applied, root-mean-square over the window's updates (0.0 without updates);
        * "D/scores/<t>" and "D/signs/<t>" for t in real, rec, mix, patch_real, patch_mix, and "G/..." for rec, mix and
          patch_mix: the mean discriminator logit and mean sign over the finite elements, "…/scores/<t>/nonfinite" the
          number of NaN / Inf logits left out (these need this package's model: the reference's model file has no sink);
        * per_tensor=True: "per_tensor", {state_dict key: {"<kind>/<norm>": float}}.
        reset: clear the window afterwards.  With more than one rank this is a collective (one small all-reduce of the score
        sums): every rank must call it.  The norms are the same on every rank already."""
        if self.stats is None:
            raise RuntimeError("no training statistics: opt.training_stats is off")
        return self.stats.read(reset=reset, per_tensor=per_tensor)

    def ema_state_dict(self):
        """the inner model's full state_dict with every E. / G. parameter replaced by its average (copies): the reference's
        keys, shapes and dtypes, D, Dpatch and num_discriminator_iters live.  ``model.load`` takes it as it is."""
        if self.ema is None:
            raise RuntimeError("no weight average: opt.ema_kimg is 0")
        sd = self._inner().state_dict()
        for n, v in zip(self.ema.names, self.ema.averaged()):
            sd[n] = v.detach().clone()
        return sd

    def nonfinite_guard_on(self):
        return bool(getattr(self.opt, "skip_nonfinite_steps", False))

    def _nonfinite_counters(self):
        if self._nonfinite_skipped is None:
            self._nonfinite_skipped = torch.zeros(len(NONFINITE_KINDS), dtype=torch.int64, device=self.Gparams[0].device)
        return self._nonfinite_skipped

    def nonfinite_guard(self, kind):
        """the ``NonfiniteGuard`` of one kind of half-step ("D", "R1" or "G"), created on first use"""
        g = self._nonfinite_guards.get(kind)
        if g is None:
            i = NONFINITE_KINDS.index(kind)
            g = NonfiniteGuard(len(self.Gparams if kind == "G" else self.Dparams), self._nonfinite_counters()[i:i + 1])
            self._nonfinite_guards[kind] = g
        return g

    def nonfinite_steps(self):
        """{"D": n, "R1": n, "G": n}: half-steps of each kind whose update the guard dropped since construction (or as
        restored by ``load_state_dict``); one device-to-host read"""
        if self._nonfinite_skipped is None:
            return {k: 0 for k in NONFINITE_KINDS}
        return dict(zip(NONFINITE_KINDS, self._nonfinite_skipped.tolist()))

    def nonfinite_report(self, kind):
        """{state_dict key: non-finite element count} of the gradients of the most recent ``kind`` half-step that had any
        ({} if none had); one device-to-host read"""
        g = self._nonfinite_guards.get(kind)
        if g is None:
            if kind not in NONFINITE_KINDS:
                raise ValueError(kind)
            return {}
        inner = getattr(self.model, "singlegpu_model", self.model)
        names = {id(p): n for n, p in inner.named_parameters()}
        params = self.Gparams if kind == "G" else self.Dparams
        return {names[id(p)]: c for p, c in zip(params, g.report.tolist()) if c}

    def exchange_and_step(self, optimizer, params, kind=None, micro_batches=1, images=None):
        """optimizer step of one half-step; with more than one rank: pack -> all-reduce (SUM) -> Adam reading the bucket.
        With ``opt.skip_nonfinite_steps`` the gradients Adam reads (the reduced bucket with more than one rank: the same bytes
        on every rank) are scanned first and a non-finite one drops the update of the half-step ``kind``.
        micro_batches > 1: the gradients were summed into the bucket by ``accumulate_to_bucket`` after every micro-batch; one
        all-reduce (world > 1), one scan, one Adam update reading the bucket with grad_scale = 1 / (micro_batches * world).
        With ``opt.ema_kimg`` > 0 a G update is followed by one averaging update over ``images`` (this rank's images of the
        update) times world, dropped with the Adam update when the guard drops that.  With ``opt.training_stats`` the norms of
        the update are added to the statistics' window, from the gradients Adam read; a dropped update adds nothing."""
        guard = self.nonfinite_guard(kind) if kind is not None and self.nonfinite_guard_on() else None
        kw = {} if guard is None else {"guard": guard}
        if micro_batches > 1:
            grads, scale = self.model.reduce_accumulated(), 1.0 / (micro_batches * self.world)
        elif self.world > 1:
            grads, scale = self.model.reduce_to_bucket(params), 1.0 / self.world
        else:
            grads, scale = None, 1.0                # Adam reads the parameters' .grad
        skip = optimizer.step(grads=grads, grad_scale=scale, **kw)
        if self.stats is not None and kind is not None:
            self.stats.record_update(kind, grads, scale, skip=skip)
        if kind == "G" and self.ema is not None:
            if images is None:
                raise ValueError("exchange_and_step: a G update with weight averaging needs its image count")
            self.ema.update(images * self.world, skip=skip)

    @staticmethod
    def set_requires_grad(params, requires_grad):
        for p in params:
            p.requires_grad_(requires_grad)

    def prepare_images(self, data_i):
        return data_i["real_A"]

    def toggle_training_mode(self):
        modes = ["discriminator", "generator"]
        self.train_mode_counter = (self.train_mode_counter + 1) % len(modes)
        return modes[self.train_mode_counter]

    def train_one_step(self, data_i, total_steps_so_far=0):
        """One half-step.  The toggle returns "generator" first, which selects the *discriminator* update
        (reference :59-65) — strict D, G, D, G alternation starting with D."""
        images = self.prepare_images(data_i)
        self.split_micro_batches(images)            # a batch that does not split raises before the schedule moves
        if self.toggle_training_mode() == "generator":
            losses = self.train_discriminator_one_step(images)
        else:
            losses = self.train_generator_one_step(images)
        return util.to_numpy(losses, lazy=getattr(self.opt, "async_loss_readback", True))

    # ------------------------------------------------------------------ half-step bodies (eager or captured)
    def _generator_body(self, images, step=True):
        self.set_requires_grad(self.Dparams, False)
        self.set_requires_grad(self.Gparams, True)
        self.optimizer_G.zero_grad()
        g_losses, g_metrics = self.model(images, None, None, command="compute_generator_losses")
        sum(v.mean() for v in g_losses.values()).backward()
        if step:
            self.exchange_and_step(self.optimizer_G, self.Gparams, kind="G", images=images.shape[0])
        g_losses.update(g_metrics)
        return g_losses

    def _discriminator_body(self, images, step=True):
        self.set_requires_grad(self.Dparams, True)
        self.set_requires_grad(self.Gparams, False)
        self.optimizer_D.zero_grad()
        d_losses, d_metrics, sp, gl = self.model(images, command="compute_discriminator_losses")
        sum(v.mean() for v in d_losses.values()).backward()
        # extra outputs travel under "_"-prefixed keys so that eager and captured execution share one flat dict
        d_losses["_sp"], d_losses["_gl"] = sp.detach(), gl.detach()
        d_losses.update({"_metric:" + k: v for k, v in d_metrics.items()})
        if step:
            self.exchange_and_step(self.optimizer_D, self.Dparams, kind="D")
        return d_losses

    def _r1_body(self, images, step=True):
        self.set_requires_grad(self.Dparams, True)
        self.set_requires_grad(self.Gparams, False)
        self.optimizer_D.zero_grad()
        r1_losses = self.model(images, command="compute_R1_loss")
        (sum(v.mean() for v in r1_losses.values()) * self.opt.R1_once_every).backward()
        if step:
            self.exchange_and_step(self.optimizer_D, self.Dparams, kind="R1")
        return r1_losses

    # ------------------------------------------------------------------ gradient accumulation (extension, opt.micro_batches)
    def micro_batches(self):
        return getattr(self.opt, "micro_batches", 1)

    def split_micro_batches(self, images):
        """the rank's images [B, ...] as opt.micro_batches consecutive slices of B / k images along dim 0; ValueError unless
        k divides B into even micro-batches of at least 2 images (``swap`` pairs images).  k = 1: [images], unchecked."""
        k = self.micro_batches()
        if k == 1:
            return [images]
        if not isinstance(k, int) or isinstance(k, bool) or k < 1:
            raise ValueError("opt.micro_batches must be a positive integer, got %r" % (k,))
        n = images.shape[0]
        if n % k != 0 or (n // k) % 2 != 0 or n // k < 2:
            raise ValueError("a batch of %d images does not split into %d micro-batches of an even number of images" % (n, k))
        b = n // k
        return [images[j * b:(j + 1) * b] for j in range(k)]

    @staticmethod
    def _mean_outputs(parts):
        """one body's outputs over the micro-batches of an update: every value the mean of its k micro-batch means, formed on
        the device; the codes ("_sp", "_gl") concatenated, so they keep the full batch's shape"""
        out = {}
        for key in parts[0]:
            vals = [p[key] for p in parts]
            out[key] = torch.cat(vals) if key in ("_sp", "_gl") else torch.stack(vals).mean()
        return out

    def _run(self, kind, images):
        """Eager execution of one body, or — with ``opt.cuda_graphs`` on a CUDA device — replay of its CUDA graph.
        With opt.micro_batches = k > 1: the body once per micro-batch with step=False (eager or replayed), its gradients
        summed into the flat bucket after each, then one exchange and one Adam update (exchange_and_step)."""
        body = {"G": self._generator_body, "D": self._discriminator_body, "R1": self._r1_body}[kind]
        chunks = self.split_micro_batches(images)
        k = len(chunks)
        if k == 1:
            if self.graphs is not None and images.is_cuda:
                return self.graphs.run(kind, body, images)
            return body(images)
        params = self.Gparams if kind == "G" else self.Dparams
        parts = []
        for j, chunk in enumerate(chunks):
            if self.graphs is not None and chunk.is_cuda:
                out = self.graphs.run(kind, body, chunk, micro_batches=k)
            else:
                out = body(chunk, step=False)
            self.model.accumulate_to_bucket(params, j)
            # a replay's outputs are the graph's static buffers, which the next replay overwrites: reduce / copy them now
            with torch.no_grad():
                parts.append({key: (v.detach().clone() if key in ("_sp", "_gl") else v.detach().mean())
                              for key, v in out.items() if torch.is_tensor(v)})
        self.exchange_and_step(self.optimizer_G if kind == "G" else self.optimizer_D, params, kind=kind, micro_batches=k,
                               images=images.shape[0])
        return self._mean_outputs(parts)

    def train_generator_one_step(self, images):
        return self._run("G", images)

    def train_discriminator_one_step(self, images):
        opt = self.opt
        if opt.lambda_GAN == 0.0 and opt.lambda_PatchGAN == 0.0:
            return {}
        self.discriminator_iter_counter += 1
        d_losses = dict(self._run("D", images))
        micro = self.micro_batches()
        if micro > 1:
            # compute_discriminator_losses advanced the model's iteration buffer once per micro-batch; it counts D updates
            getattr(self.model, "singlegpu_model", self.model).num_discriminator_iters.sub_(micro - 1)
        self.previous_sp, self.previous_gl = d_losses.pop("_sp"), d_losses.pop("_gl")
        d_metrics = {k[len("_metric:"):]: d_losses.pop(k) for k in list(d_losses) if k.startswith("_metric:")}

        needs_r1 = (opt.lambda_R1 > 0.0 or opt.lambda_patch_R1 > 0.0) and \
            self.discriminator_iter_counter % opt.R1_once_every == 0
        if needs_r1:
            d_losses.update(self._run("R1", images))

        if self.augment is not None and self.augment.tuning() and self.discriminator_iter_counter % self.augment.interval == 0:
            # every ada_interval-th D update: fold the sign sums of D(aug(real)) into p (one launch, eager: the captured
            # D graph is the same on adjusting and non-adjusting steps)
            self.augment.adjust(images.shape[0])

        d_losses["D_total"] = sum(v.mean() for v in d_losses.values())
        d_losses.update(d_metrics)
        return d_losses

    def get_visuals_for_snapshot(self, data_i):
        with torch.no_grad():
            return self.model(self.prepare_images(data_i), command="get_visuals_for_snapshot")

    # ------------------------------------------------------------------ checkpointing (SURVEY.md §8 f3)
    def state_dict(self):
        """Adam state of both groups (torch.optim.Adam's format) + the schedule counters.  The reference never saves this
        (optimizers/base_optimizer.py has no state I/O): resuming there restarts Adam's moments from zero.  With
        ``opt.skip_nonfinite_steps`` the guard's skip counters (``nonfinite_steps()``) are saved as well, with ``opt.ema_kimg``
        > 0 the weight average under "ema" (``ParameterEMA.state_dict``: the shadow by state_dict key, and t), with the
        augmentation on its probability and sign sums under "ada" ({"p", "acc"})."""
        sd = {"optimizer_G": self.optimizer_G.state_dict(), "optimizer_D": self.optimizer_D.state_dict(),
              "train_mode_counter": self.train_mode_counter, "discriminator_iter_counter": self.discriminator_iter_counter}
        if self.nonfinite_guard_on():
            sd["nonfinite_steps"] = self.nonfinite_steps()
        if self.ema is not None:
            sd["ema"] = self.ema.state_dict()
        if self.augment is not None:
            sd["ada"] = self.augment.state_dict()
        return sd

    def load_state_dict(self, sd):
        self.optimizer_G.load_state_dict(sd["optimizer_G"])
        self.optimizer_D.load_state_dict(sd["optimizer_D"])
        self.train_mode_counter = int(sd.get("train_mode_counter", 0))
        self.discriminator_iter_counter = int(sd.get("discriminator_iter_counter", 0))
        if "nonfinite_steps" in sd:
            counts = [int(sd["nonfinite_steps"].get(k, 0)) for k in NONFINITE_KINDS]
            self._nonfinite_counters().copy_(torch.tensor(counts, dtype=torch.int64))     # in place: captured graphs hold it
        if self.ema is not None and "ema" in sd:
            self.ema.load_state_dict(sd["ema"])          # without one the construction-time copy stays
        if self.augment is not None and "ada" in sd:
            self.augment.load_state_dict(sd["ada"])      # in place: captured graphs hold p and the sign sums

    def _optimizer_path(self, total_steps_so_far=None, what="optimizer"):
        name = "latest_%s.pth" % what if total_steps_so_far is None else "%dk_%s.pth" % (total_steps_so_far // 1000, what)
        return os.path.join(self._inner()._checkpoint_dir(), name)

    @staticmethod
    def _save_with_link(obj, path, link):
        torch.save(obj, path)
        if os.path.lexists(link):
            os.remove(link)
        os.symlink(os.path.basename(path), link)

    def save(self, total_steps_so_far):
        """model checkpoint in the reference's format (models/base_model.py:33-41) + ``<N>k_optimizer.pth`` beside it; with
        ``opt.ema_kimg`` > 0 also ``<N>k_ema_checkpoint.pth`` (``ema_state_dict()``, the model checkpoint's format, so the
        reference's ``--resume_iter latest_ema`` loads it) and its ``latest_ema_checkpoint.pth`` link.  Rank 0 writes."""
        self.model.save(total_steps_so_far)
        if getattr(self.model, "rank", 0) == 0:
            self._save_with_link(self.state_dict(), self._optimizer_path(total_steps_so_far), self._optimizer_path(None))
            if self.ema is not None:
                self._save_with_link(self.ema_state_dict(), self._optimizer_path(total_steps_so_far, "ema_checkpoint"),
                                     self._optimizer_path(None, "ema_checkpoint"))

    def load(self, path=None):
        """restore the optimizer state written by ``save`` (missing file: keep the fresh state, like the reference)"""
        path = path or self._optimizer_path(None)
        if not os.path.exists(path):
            return False
        self.load_state_dict(torch.load(path, map_location=str(self.Gparams[0].device)))
        return True
