#!/usr/bin/env python
"""Debug aid: list the layout-conversion copies (.contiguous() on non-channels-last tensors) a D + G step performs."""
import collections
import os
import sys
import traceback

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import swapping_autoencoder_pytorch_b200 as S  # noqa: E402
import importlib  # noqa: E402
conv = importlib.import_module("swapping_autoencoder_pytorch_b200.stylegan2_op.conv")
fused_act = importlib.import_module("swapping_autoencoder_pytorch_b200.stylegan2_op.fused_act")
upfirdn2d = importlib.import_module("swapping_autoencoder_pytorch_b200.stylegan2_op.upfirdn2d")

log = collections.Counter()


def audit(name, fn):
    def wrapped(t):
        out = fn(t)
        if out.data_ptr() != t.data_ptr() and t.numel() > 1_000_000:
            st = traceback.extract_stack(limit=7)
            where = " < ".join("%s:%d" % (os.path.basename(f.filename), f.lineno) for f in st[:-1][-4:])
            log[(name, tuple(t.shape), tuple(t.stride()), where)] += t.numel() * 8
        return out
    return wrapped


for mod in (conv, upfirdn2d):
    mod.nhwc = audit(mod.__name__.split(".")[-1] + ".nhwc", mod.nhwc)
fused_act._cl = audit("fused_act._cl", fused_act._cl)

opt = S.default_options(num_gpus=1, batch_size=int(os.environ.get("B", "8")))
model = S.create_model(opt)
trainer = S.create_optimizer(opt, model)
real = torch.randn(opt.batch_size, 3, 256, 256, device="cuda").clamp(-1, 1)
trainer.train_one_step({"real_A": real}, 0)
trainer.train_one_step({"real_A": real}, 0)
log.clear()
trainer.train_one_step({"real_A": real}, 0)
trainer.train_one_step({"real_A": real}, 0)
torch.cuda.synchronize()
tot = sum(log.values())
print("total copy traffic %.1f MB over %d sites" % (tot / 1e6, len(log)))
for (name, shape, stride, where), b in log.most_common(25):
    print("%8.1f MB %-18s %-24s %-28s %s" % (b / 1e6, name, shape, stride, where))
