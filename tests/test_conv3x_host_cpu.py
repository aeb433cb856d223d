"""Host logic of the tensor-core conv path (core/conv_ops.py) on the CPU: the space-to-depth form of the
first layers and the input copy in front of the kernels, against plain float64 autograd."""
import pytest
import torch
import torch.nn.functional as F

from unflow_b200.e2eflow.core import conv_ops as co


@pytest.mark.parametrize("C,H,W,k,pads", [(3, 16, 20, 7, (2, 3, 2, 3)), (6, 17, 21, 7, (3, 3, 3, 3)),
                                          (14, 12, 12, 7, (2, 3, 2, 3)), (3, 10, 14, 5, (1, 2, 1, 2))])
def test_space_to_depth_operands_are_the_same_convolution(C, H, W, k, pads):
    """7x7 stride-2 conv == 4x4 stride-1 conv over 2x2 pixel blocks (core/conv_ops.py), values and
    gradients."""
    g = torch.Generator().manual_seed(C + H)
    x = torch.randn(2, C, H, W, dtype=torch.float64, generator=g).requires_grad_(True)
    w = torch.randn(8, C, k, k, dtype=torch.float64, generator=g).requires_grad_(True)
    b = torch.randn(8, dtype=torch.float64, generator=g).requires_grad_(True)
    ref = F.leaky_relu(F.conv2d(F.pad(x, (pads[2], pads[3], pads[0], pads[1])), w, b, stride=2), co.LRELU_SLOPE)
    xs, ws = co.space_to_depth_operands(x, w, pads)
    m = (k + 1) // 2
    assert xs.shape == (2, 4 * C, ref.shape[2] + m - 1, ref.shape[3] + m - 1) and ws.shape == (8, 4 * C, m, m)
    assert co._use_space_to_depth(x, w, 2) and not co._use_space_to_depth(xs, ws, 1)
    go = torch.randn(ref.shape, dtype=torch.float64, generator=g)
    want = torch.autograd.grad(ref, (x, w, b), go)
    y = F.leaky_relu(F.conv2d(xs, ws, b), co.LRELU_SLOPE)
    assert y.shape == ref.shape and float((y - ref).abs().max()) < 1e-12
    got = torch.autograd.grad(y, (x, w, b), go)
    for a_, b_ in zip(got, want):
        assert a_.shape == b_.shape and float((a_ - b_).abs().max()) < 1e-10
    wide = torch.randn(8, 64, 5, 5, dtype=torch.float64)
    assert not co._use_space_to_depth(torch.zeros(1, 64, 8, 8), wide, 2)        # enough channels already


@pytest.mark.parametrize("stride,k,H,W,pads", [(2, 3, 21, 27, (1, 1, 1, 1)), (2, 3, 21, 27, (0, 0, 0, 0)),
                                               (2, 5, 20, 27, (1, 2, 2, 2)), (1, 3, 21, 27, (1, 1, 1, 1))])
def test_input_copy_leaves_the_convolution_unchanged(stride, k, H, W, pads):
    """conv_ops._tc_input: a conv over the copy (NHWC, pitch round4(C), a zero row / column appended where H / W
    is odd at stride 2) with the pads it returns is the conv over the original input, values and dL/dx."""
    g = torch.Generator().manual_seed(k * 100 + H + W)
    C = 5
    x = torch.randn(2, C, H, W, generator=g).requires_grad_(True)     # on the CPU every input is copied
    w = torch.randn(4, C, k, k, dtype=torch.float64, generator=g)
    xt, tp = co._tc_input(x, stride, pads)
    Hc, Wc = (H + H % 2, W + W % 2) if stride == 2 else (H, W)
    assert xt.shape == (2, C, Hc, Wc) and xt.stride() == (Hc * Wc * 8, 1, Wc * 8, 8)
    conv = lambda t, p: F.conv2d(F.pad(t.double().contiguous(), (p[2], p[3], p[0], p[1])), w, stride=stride)
    ref, got = conv(x, pads), conv(xt, tp)
    assert got.shape == ref.shape and torch.equal(got, ref)
    go = torch.randn(ref.shape, dtype=torch.float64, generator=g)
    want, = torch.autograd.grad(ref, x, go)
    have, = torch.autograd.grad(got, x, go)
    assert torch.equal(have, want)
