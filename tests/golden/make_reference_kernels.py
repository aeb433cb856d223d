"""Run the reference's own CUDA kernels (oracle/_ref/libref_ops.so, built by oracle/ref_kernels.py from
the reference tree) on the inputs of tests/test_reference_kernels.py and store what that test compares
against in tests/golden/reference_kernels.npz:

    python tests/golden/make_reference_kernels.py [OUT.npz]      (needs a GPU and oracle/_ref)

For every output tensor the file keeps its largest magnitude (the scale of the test's tolerance) and its
values at up to SAMPLE seeded flat positions; the correlation geometry table comes from the reference's
host code (CorrelationState).  The inputs are not stored: the test draws them from the same seeds."""
import itertools
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import ref_kernels as RK  # noqa: E402

SAMPLE = 4096
CORR_CASES = [(2, 32, 12, 20, dict(kernel_size=1, max_displacement=4, pad=4, stride_1=1, stride_2=2)),
              (1, 16, 10, 14, dict(kernel_size=3, max_displacement=3, pad=4, stride_1=2, stride_2=1)),
              (1, 256, 48, 160, dict(kernel_size=1, max_displacement=20, pad=20, stride_1=1, stride_2=2))]
GEOMETRY = list(itertools.product((48, 37), (160, 64), (1, 3), (20, 4, 0), (20, 4, 0), (1, 2), (1, 2)))


def sample_index(numel, key):
    """The flat positions kept of a tensor with ``numel`` elements (all of them when it is small)."""
    if numel <= SAMPLE:
        return np.arange(numel, dtype=np.int64)
    rng = np.random.default_rng(sum(map(ord, key)))
    return np.sort(rng.choice(numel, SAMPLE, replace=False)).astype(np.int64)


def corr_inputs(B, C, H, W):
    g = torch.Generator().manual_seed(C + H)
    a, b = torch.randn(B, C, H, W, generator=g), torch.randn(B, C, H, W, generator=g)
    return g, a, b


def warp_inputs():
    g = torch.Generator().manual_seed(3)
    im = torch.rand(2, 18, 26, 3, generator=g)
    fl = torch.randn(2, 18, 26, 2, generator=g) * 4
    return g, im, fl


def main(path):
    out = {}

    def put(key, t):
        v = t.detach().double().cpu().numpy().reshape(-1)
        idx = sample_index(v.size, key)
        out[key + "_shape"] = np.asarray(t.shape, dtype=np.int64)
        out[key + "_absmax"] = np.float64(np.abs(v).max())
        out[key + "_idx"] = idx
        out[key + "_val"] = v[idx]

    out["geometry"] = np.asarray([RK.correlation_out_shape(256, H, W, ks, md, pad, s1, s2)
                                  for H, W, ks, md, pad, s1, s2 in GEOMETRY], dtype=np.int64)
    for i, (B, C, H, W, attrs) in enumerate(CORR_CASES):
        g, a, b = corr_inputs(B, C, H, W)
        ref, p0, p1 = RK.correlation(a.cuda(), b.cuda(), **attrs)
        go = torch.randn(ref.shape, generator=g)
        r0, r1 = RK.correlation_grad(go.cuda(), p0, p1, (B, C, H, W), **attrs)
        put("corr%d_out" % i, ref)
        put("corr%d_d0" % i, r0)
        put("corr%d_d1" % i, r1)

    g, im, fl = warp_inputs()
    ref = RK.backward_warp(im.cuda(), fl.cuda())
    put("bwarp_out", ref)
    go = torch.randn(ref.shape, generator=g)
    put("bwarp_dflow", RK.backward_warp_grad(go.cuda(), im.cuda(), fl.cuda()))
    ref = RK.forward_warp(fl.cuda())
    put("fwarp_out", ref)
    go = torch.randn(ref.shape, generator=g)
    put("fwarp_dflow", RK.forward_warp_grad(go.cuda(), fl.cuda()))
    x = torch.rand(2, 16, 24, 3, generator=g)
    for scale in (2, 4):
        put("down%d_out" % scale, RK.downsample(x.cuda(), scale))
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "reference_kernels.npz"))
