#!/usr/bin/env python
"""Run every hand-written kernel a few times at the shapes of the benchmark step, for ncu:

  ncu --set full --clock-control none --import-source on -k regex:unflow -o gpurun_out/prof \
      python tools/profile_kernels.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from unflow_b200 import synthetic as synth  # noqa: E402
from unflow_b200.e2eflow import ops  # noqa: E402
from unflow_b200.e2eflow.core import fused_loss  # noqa: E402
from unflow_b200.e2eflow.core.image_warp import image_warp  # noqa: E402
from unflow_b200 import _native  # noqa: E402


def main():
    reps = int(os.environ.get("REPS", "2"))
    torch.manual_seed(0)
    B, C, H, W = 4, 256, 48, 160
    a = torch.randn(B, C, H, W, device="cuda", requires_grad=True)
    b = torch.randn(B, C, H, W, device="cuda", requires_grad=True)
    for _ in range(reps):
        out = ops.correlation(a, b)
        out.backward(torch.ones_like(out))
    terms = ['occ', 'fb', 'ternary', 'smooth_2nd']
    for (Bl, h, w, d) in ((4, 96, 320, 3), (4, 384, 1280, 3)):
        im1, im2, ffw, fbw = synth.level_inputs(1, h, w, seed=3)
        im1, im2 = im1.cuda().repeat(Bl, 1, 1, 1), im2.cuda().repeat(Bl, 1, 1, 1)
        ffw = ffw.cuda().repeat(Bl, 1, 1, 1).requires_grad_(True)
        fbw = fbw.cuda().repeat(Bl, 1, 1, 1).requires_grad_(True)
        border = torch.ones(Bl, h, w, 1, device="cuda")
        for _ in range(reps):
            l = fused_loss.compute_losses_fused(im1, im2, ffw, fbw, border, 'fb', d, terms)
            (l['ternary'] + l['fb'] + l['smooth_2nd']).backward()
        for _ in range(reps):
            wv = image_warp(im1, ffw)
            wv.sum().backward()
            ops.backward_warp(im1, ffw.detach())
            ops.forward_warp(ffw.detach())
            ops.downsample(im1, 2 if h < 300 else 4)
    n = 39175300
    p, g, m, v = (torch.zeros(n, device="cuda") for _ in range(4))
    for t in range(1, reps + 1):
        _native.check(_native.lib().unflow_adam_step(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), n,
                                                     1e-4, 0.9, 0.999, 1e-8, t, 1.0, 1,
                                                     torch.cuda.current_stream().cuda_stream), "adam")
    torch.cuda.synchronize()


if __name__ == "__main__":
    main()
