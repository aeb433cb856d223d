#!/usr/bin/env python
"""The narrow-conv kernels (flow heads) at the shapes of the benchmark step, one launch each, for
`ncu --set full`:

  ncu --set full --clock-control none --import-source on -k regex:"narrow_" \
      -o gpurun_out/prof_narrow python tools/profile_narrow.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from unflow_b200.e2eflow.core import conv_ops  # noqa: E402

conv_ops.set_mode('3xtf32')
torch.manual_seed(0)
for (N, C, H, W) in ((8, 194, 96, 320), (8, 386, 48, 160)):      # flow2, flow3 of a B=4 bidirectional step
    x = torch.randn(N, C, H, W, device="cuda").contiguous(memory_format=torch.channels_last).requires_grad_(True)
    w = (torch.randn(2, C, 3, 3, device="cuda") * 0.05).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    b = torch.zeros(2, device="cuda", requires_grad=True)
    y = conv_ops._NarrowConv3x3.apply(x, w, b)
    y.backward(torch.randn_like(y))
torch.cuda.synchronize()
