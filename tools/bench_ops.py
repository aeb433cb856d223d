#!/usr/bin/env python
"""Op-level timing on one H100 (CUDA events, L2 flushed between iterations).

Prints one JSON line per kernel with the algorithmic bytes / FLOPs of SURVEY.md 8d and the
achieved fraction of the H100 SXM data-sheet peaks (or MEASURED_PEAKS.json where present)."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from unflow_b200.e2eflow import ops  # noqa: E402
from unflow_b200.e2eflow.core.image_warp import image_warp  # noqa: E402

PEAKS = {"hbm_gbs": 3350.0, "sm_max_mhz": 1980.0}      # H100 SXM data sheet
try:
    PEAKS.update(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))))
except Exception:
    pass
FMA_PEAK = 132 * 128 * 2 * PEAKS["sm_max_mhz"] * 1e6 / 1e12  # TFLOP/s fp32


def timeit(fn, iters=20, warmup=5, flush=True):
    scratch = torch.empty(256 * 1024 * 1024 // 4, device="cuda") if flush else None
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        if flush:
            scratch.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        times.append(s.elapsed_time(e) * 1e-3)
    times.sort()
    return times[len(times) // 2], times[0]


def report(name, t_med, t_min, nbytes, flops=None):
    rec = {"kernel": name, "ms_median": round(t_med * 1e3, 4), "ms_min": round(t_min * 1e3, 4),
           "alg_MB": round(nbytes / 1e6, 2), "GBs": round(nbytes / t_med / 1e9, 1),
           "hbm_frac": round(nbytes / t_med / 1e9 / PEAKS["hbm_gbs"], 4)}
    if flops:
        rec["TFLOPs"] = round(flops / t_med / 1e12, 2)
        rec["fma_frac"] = round(flops / t_med / 1e12 / FMA_PEAK, 4)
    print(json.dumps(rec), flush=True)


def main():
    torch.manual_seed(0)
    B, C, H, W = 8, 256, 48, 160
    a = torch.randn(B, C, H, W, device="cuda")
    b = torch.randn(B, C, H, W, device="cuda")
    D2 = 441
    nbytes = 4 * B * H * W * (2 * C + D2)
    flops = 2 * B * H * W * C * D2
    t = timeit(lambda: ops.correlation(a, b))
    report("correlation_fwd B8 256x48x160 d20", *t, nbytes, flops)

    ar, br = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
    out = ops.correlation(ar, br)
    g = torch.randn_like(out)
    t = timeit(lambda: torch.autograd.grad(out, (ar, br), g, retain_graph=True), iters=5, warmup=1)
    report("correlation_bwd B8", *t, 4 * B * H * W * (D2 + 4 * C), 2 * flops)

    Bl, h, w = 4, 384, 1280
    im = torch.rand(Bl, h, w, 3, device="cuda")
    # smooth flow (|f| <= 8 px), as the loss pyramid sees; i.i.d. random flows scatter every lane of a
    # warp to a different row and measure the L1, not the kernel
    sys.path.insert(0, ROOT)
    from unflow_b200 import synthetic
    fl = synthetic.image_pair(Bl, h, w, seed=3)[2].cuda().contiguous()
    t = timeit(lambda: image_warp(im, fl))
    report("image_warp fwd B4 384x1280x3", *t, 4 * Bl * h * w * (2 * 3 + 2))
    t = timeit(lambda: ops.backward_warp(im, fl))
    report("backward_warp fwd B4 384x1280x3", *t, 4 * Bl * h * w * (2 * 3 + 2))
    t = timeit(lambda: ops.forward_warp(fl))
    report("forward_warp fwd B4 384x1280", *t, 4 * Bl * h * w * 3)
    t = timeit(lambda: ops.downsample(im, 4))
    report("downsample x4 B4 384x1280x3", *t, 4 * Bl * 3 * (h * w + h * w // 16))
    flr = fl.clone().requires_grad_(True)
    imr = im.clone().requires_grad_(True)
    o = image_warp(imr, flr)
    go = torch.randn_like(o)
    t = timeit(lambda: torch.autograd.grad(o, (imr, flr), go, retain_graph=True))
    report("image_warp bwd (dflow+dimage) B4 384x1280x3", *t, 4 * Bl * h * w * (3 * 3 + 4))

    # flow heads at the shapes of the B=4 bidirectional step, input = channel slice of a pitch-padded NHWC buffer
    # (what the decoder's concat buffers are): the TMA-staged kernels (csrc/narrow_conv_tma.cu)
    from unflow_b200.e2eflow.core import conv_ops
    for (N, C, hh, ww, tag) in ((8, 194, 96, 320, "flow2"), (8, 386, 48, 160, "flow3")):
        buf = torch.randn(N, hh, ww, (C + 3) // 4 * 4, device="cuda")
        x = buf[..., :C].permute(0, 3, 1, 2)
        wgt = (torch.randn(2, C, 3, 3, device="cuda") * 0.05).contiguous(memory_format=torch.channels_last)
        bias = torch.zeros(2, device="cuda")
        g = torch.randn(N, 2, hh, ww, device="cuda").contiguous(memory_format=torch.channels_last)
        nbytes = 4 * N * hh * ww * (C + 2)
        flops = 2 * N * hh * ww * C * 18
        wr = wgt.clone().requires_grad_(True)
        with torch.no_grad():
            t = timeit(lambda: conv_ops._NarrowConv3x3.apply(x, wgt, bias))
        report("narrow_conv_fwd %s" % tag, *t, nbytes, flops)

        def fwd_bwd():
            y = conv_ops._NarrowConv3x3.apply(x, wr, bias)     # x needs no grad: wgrad + bias grad only
            y.backward(g)
        t = timeit(fwd_bwd)
        report("narrow_conv fwd+wgrad %s" % tag, *t, 2 * nbytes, 2 * flops)


if __name__ == "__main__":
    main()
