#!/usr/bin/env python
"""Per-kernel GPU time of ONE warm training step (CUPTI activity records through torch.profiler):
kernel name, launches, total time, share of the step -- as a markdown table on stdout.

CUPTI's activity trace costs little per launch and times the kernels warm, in the order and
overlap the step really has."""
import collections
import os
import re
import sys

import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from unflow_b200 import synthetic as synth  # noqa: E402
from unflow_b200.e2eflow.core import conv_ops  # noqa: E402
from unflow_b200.e2eflow.core.train import Trainer  # noqa: E402

conv_ops.set_mode(os.environ.get("UNFLOW_CONV_PRECISION", "3xtf32"))
torch.backends.cudnn.benchmark = True
dev = torch.device("cuda", 0)
tr = Trainer(dict(synth.KITTI_PARAMS, learning_rate=1e-5), synth.KITTI_NORMALIZATION, dev, seed=1)
im1, im2, _ = synth.image_pair(4, 384, 1280, seed=1)
im1, im2 = im1.to(dev), im2.to(dev)
for _ in range(4):
    tr.step(im1, im2)
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    tr.step(im1, im2)
    torch.cuda.synchronize()

agg = collections.OrderedDict()
for e in prof.events():
    if "cuda" not in str(getattr(e, "device_type", "")).lower():
        continue
    t = getattr(e, "device_time", None)
    if t is None:
        t = getattr(e, "cuda_time", 0.0)
    name = re.sub(r"^void ", "", e.name)
    name = re.sub(r"\(.*$", "", name)
    if len(name) > 110:
        name = name[:107] + "..."
    a = agg.setdefault(name, [0, 0.0])
    a[0] += 1
    a[1] += float(t)
total = sum(v[1] for v in agg.values())
ours = sum(v[1] for k, v in agg.items() if k.startswith(("unflow::", "ll::")) or "unflow" in k)
n = sum(v[0] for v in agg.values())
print("# CUPTI kernel times, one warm training step (%d launches, %.2f ms of kernel time)\n" % (n, total / 1e3))
print("B=4, 384x1280, FlowNetC, 3xTF32 conv path, cuDNN autotune, eager launch (no CUDA graph);"
      " hand-written kernels (`unflow::`, `ll::`) = %.1f %% of the kernel time\n" % (100.0 * ours / total))
print("| share | time (us) | launches | kernel |\n|---:|---:|---:|---|")
for k, v in sorted(agg.items(), key=lambda kv: -kv[1][1])[:45]:
    print("| %.2f %% | %.1f | %d | `%s` |" % (100.0 * v[1] / total, v[1], v[0], k))
