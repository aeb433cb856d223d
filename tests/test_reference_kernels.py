"""The reference's own CUDA kernels as ground truth for the four custom ops, through the golden
vectors they produced (tests/golden/reference_kernels.npz, made by tests/golden/make_reference_kernels.py
from the reference kernels compiled against stand-in TensorFlow headers, oracle/ref_kernels.py).

* CPU part: the correlation geometry of the reference's ``CorrelationState`` host code -- compared with
  the oracle and with the product's C ABI.
* GPU part: the oracle's C restatement and the product's kernels are compared with the reference
  kernels' outputs on the same seeded inputs -- forward and gradients of all four ops, including
  displacement > 0 / C > 1 / K = 3 / strides, which the reference's own KATs never exercise
  (test/ops/correlation.py:30-89).  The file holds each reference output's largest magnitude and its
  values at a fixed sample of positions."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

from oracle import ops as oops

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
import make_reference_kernels as MK  # noqa: E402

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_kernels.npz"))


def test_correlation_geometry_from_the_reference_host_code():
    from unflow_b200 import _native
    lib = _native.lib()
    n = 0
    for (H, W, ks, md, pad, s1, s2), want in zip(MK.GEOMETRY, G["geometry"]):
        want = tuple(int(v) for v in want)
        oc, oh, ow = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        rc = oops.lib().oracle_correlation_shape(H, W, ks, md, pad, s1, s2, ctypes.byref(oc), ctypes.byref(oh), ctypes.byref(ow))
        c2, h2, w2 = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        rc2 = lib.unflow_correlation_out_shape(H, W, ks, md, pad, s1, s2, ctypes.byref(c2), ctypes.byref(h2),
                                               ctypes.byref(w2))
        shape = (c2.value, h2.value, w2.value)
        if want[1] <= 0 or want[2] <= 0:            # the reference op rejects these (correlation_op.cc:60-61)
            assert rc != 0 and rc2 != 0
            continue
        n += 1
        assert rc == 0 and (oc.value, oh.value, ow.value) == want, (H, W, ks, md, pad, s1, s2)
        assert rc2 == 0 and tuple(shape) == want, (H, W, ks, md, pad, s1, s2)
    assert n > 100


def _close(a, key, tol=1e-5):
    """``a`` against the reference output ``key``: max error at the stored positions <= tol * max|reference|."""
    a = a.detach().double().cpu()
    assert tuple(a.shape) == tuple(int(v) for v in G[key + "_shape"]), key
    got = a.reshape(-1).numpy()[G[key + "_idx"]]
    scale = max(float(G[key + "_absmax"]), 1e-12)
    err = float(np.abs(got - G[key + "_val"]).max())
    assert err <= tol * scale, (key, err / scale)


@pytest.mark.gpu
@pytest.mark.parametrize("B,C,H,W,attrs", MK.CORR_CASES)
def test_correlation_kernels(B, C, H, W, attrs):
    from unflow_b200.e2eflow import ops
    case = MK.CORR_CASES.index((B, C, H, W, attrs))
    g, a, b = MK.corr_inputs(B, C, H, W)
    key = "corr%d_" % case
    _close(oops.correlation(a, b, **attrs), key + "out")
    go = torch.randn(tuple(int(v) for v in G[key + "out_shape"]), generator=g)
    ao, bo = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
    oops.correlation(ao, bo, **attrs).backward(go)
    _close(ao.grad, key + "d0")
    _close(bo.grad, key + "d1")
    ac, bc = a.cuda().requires_grad_(True), b.cuda().requires_grad_(True)
    out = ops.correlation(ac, bc, **attrs)
    _close(out, key + "out")
    out.backward(go.cuda())
    _close(ac.grad, key + "d0", 2e-5)
    _close(bc.grad, key + "d1", 2e-5)


@pytest.mark.gpu
def test_warp_and_downsample_kernels():
    from unflow_b200.e2eflow import ops
    g, im, fl = MK.warp_inputs()
    _close(oops.backward_warp(im, fl), "bwarp_out")
    _close(ops.backward_warp(im.cuda(), fl.cuda()), "bwarp_out")
    go = torch.randn(tuple(int(v) for v in G["bwarp_out_shape"]), generator=g)
    fo = fl.clone().requires_grad_(True)
    oops.backward_warp(im, fo).backward(go)
    _close(fo.grad, "bwarp_dflow")
    fc = fl.cuda().requires_grad_(True)
    ops.backward_warp(im.cuda(), fc).backward(go.cuda())
    _close(fc.grad, "bwarp_dflow", 2e-5)

    _close(oops.forward_warp(fl), "fwarp_out", 1e-4)          # float atomics: order-dependent rounding
    _close(ops.forward_warp(fl.cuda()), "fwarp_out", 1e-4)
    go = torch.randn(tuple(int(v) for v in G["fwarp_out_shape"]), generator=g)
    fo = fl.clone().requires_grad_(True)
    oops.forward_warp(fo).backward(go)
    _close(fo.grad, "fwarp_dflow", 1e-4)
    fc = fl.cuda().requires_grad_(True)
    ops.forward_warp(fc).backward(go.cuda())
    _close(fc.grad, "fwarp_dflow", 1e-4)

    x = torch.rand(2, 16, 24, 3, generator=g)
    for scale in (2, 4):
        _close(oops.downsample(x, scale), "down%d_out" % scale)
        _close(ops.downsample(x.cuda(), scale), "down%d_out" % scale)
