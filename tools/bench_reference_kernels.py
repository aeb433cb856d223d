#!/usr/bin/env python
"""Op-level timing of the reference's own CUDA kernels (oracle/_ref/libref_ops.so, see
oracle/ref_kernels.py) next to this repository's kernels, same inputs, one H100:

    python tools/bench_reference_kernels.py        (prints one JSON line per op)

CUDA events around each call, L2 flushed between iterations, median of 20.  The reference wrappers
synchronise inside each call (the kernels run on the legacy default stream), so their time is taken
with a host timer around the synchronous call and includes one launch latency."""
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_kernels as RK  # noqa: E402
from unflow_b200.e2eflow import ops  # noqa: E402


def med(fn, iters=20, warmup=3):
    scratch = torch.empty(256 * 1024 * 1024 // 4, device="cuda")
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        scratch.zero_()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    ts.sort()
    return ts[len(ts) // 2] * 1e3


def line(name, ref_ms, our_ms):
    print(json.dumps({"op": name, "reference_ms": round(ref_ms, 4), "ours_ms": round(our_ms, 4),
                      "speedup": round(ref_ms / our_ms, 2)}), flush=True)


def main():
    torch.manual_seed(0)
    B, C, H, W = 8, 256, 48, 160
    a, b = torch.randn(B, C, H, W, device="cuda"), torch.randn(B, C, H, W, device="cuda")
    line("correlation fwd B8 256x48x160 d20", med(lambda: RK.correlation(a, b)), med(lambda: ops.correlation(a, b)))
    out, p0, p1 = RK.correlation(a, b)
    go = torch.randn_like(out)
    ar, br = a.clone().requires_grad_(True), b.clone().requires_grad_(True)

    def ours_bwd():
        o = ops.correlation(ar, br)
        o.backward(go)
    t_fwd = med(lambda: ops.correlation(ar, br))
    line("correlation bwd (both gradients)", med(lambda: RK.correlation_grad(go, p0, p1, (B, C, H, W))),
         max(med(ours_bwd) - t_fwd, 1e-6))
    im = torch.rand(4, 384, 1280, 3, device="cuda")
    fl = torch.randn(4, 384, 1280, 2, device="cuda") * 3
    line("backward_warp fwd B4 384x1280x3", med(lambda: RK.backward_warp(im, fl)), med(lambda: ops.backward_warp(im, fl)))
    line("forward_warp fwd B4 384x1280", med(lambda: RK.forward_warp(fl)), med(lambda: ops.forward_warp(fl)))
    line("downsample x4 B4 384x1280x3", med(lambda: RK.downsample(im, 4)), med(lambda: ops.downsample(im, 4)))


if __name__ == "__main__":
    main()
