"""TensorFlow-1.x primitives the reference leans on, restated with torch on the CPU.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).  PARITY UNPINNED: the
reference has no test that pins any of these TF primitives and TF1 cannot be
run here, so each function restates the documented TF 1.x behaviour:

  * ``SAME`` padding (tensorflow/core/framework/common_shape_fns.cc,
    GetWindowedOutputSizeVerbose): out = ceil(in/stride),
    pad_total = max((out-1)*stride + k - in, 0), pad_before = pad_total // 2.
  * ``tf.image.resize_bilinear(align_corners=False)`` (legacy kernel,
    tensorflow/core/kernels/resize_bilinear_op.cc): src = dst * (in/out),
    no half-pixel offset, upper index clamped to in-1.
  * ``tf.image.resize_area`` (tensorflow/core/kernels/resize_area_op.cc).
  * ``tf.image.rgb_to_grayscale``: weights (0.2989, 0.5870, 0.1140).
  * ``slim.conv2d_transpose(k=4, stride=2, 'SAME')`` == gradient of a SAME
    stride-2 conv whose padding is (1, 1)  ->  ConvTranspose2d(padding=1).

Call sites in the reference: flownet.py:48,174-233; unsupervised.py:103-104;
losses.py:94,104,202-203; core/util.py:21-26.
"""
import math

import torch
import torch.nn.functional as F


def same_pad(in_size, k, stride):
    out = -(-in_size // stride)
    total = max((out - 1) * stride + k - in_size, 0)
    return total // 2, total - total // 2


def conv2d_same(x, w, b, stride):
    """NCHW conv with TF SAME padding. w is OIHW."""
    kh, kw = w.shape[2], w.shape[3]
    pt, pb = same_pad(x.shape[2], kh, stride)
    pl, pr = same_pad(x.shape[3], kw, stride)
    x = F.pad(x, (pl, pr, pt, pb))
    return F.conv2d(x, w, b, stride=stride)


def conv2d_transpose_same(x, w, b, stride=2):
    """NCHW transposed conv, TF SAME, k=4/stride=2 as used by the reference.

    w is torch layout [in, out, kh, kw]."""
    assert w.shape[2] == 4 and w.shape[3] == 4 and stride == 2
    return F.conv_transpose2d(x, w, b, stride=2, padding=1)


def resize_bilinear_legacy(x, size):
    """x: [B,H,W,C] -> [B,size[0],size[1],C]; TF1 align_corners=False.  The ratios, source positions and
    fractions are float32 as in TF's kernel; the interpolation runs in x's dtype, on x's device."""
    B, H, W, C = x.shape
    oh, ow = int(size[0]), int(size[1])
    dev = x.device
    hs = torch.tensor(H / oh, dtype=torch.float32, device=dev)
    ws = torch.tensor(W / ow, dtype=torch.float32, device=dev)
    iy = torch.arange(oh, dtype=torch.float32, device=dev) * hs
    ix = torch.arange(ow, dtype=torch.float32, device=dev) * ws
    y0 = iy.floor().long()
    y1 = torch.clamp(iy.ceil().long(), max=H - 1)
    x0 = ix.floor().long()
    x1 = torch.clamp(ix.ceil().long(), max=W - 1)
    ly = (iy - y0.float()).view(1, oh, 1, 1).to(x.dtype)
    lx = (ix - x0.float()).view(1, 1, ow, 1).to(x.dtype)
    top_rows = x[:, y0]
    bot_rows = x[:, y1]
    tl, tr = top_rows[:, :, x0], top_rows[:, :, x1]
    bl, br = bot_rows[:, :, x0], bot_rows[:, :, x1]
    top = tl + (tr - tl) * lx
    bot = bl + (br - bl) * lx
    return top + (bot - top) * ly


def resize_area(x, size):
    """tf.image.resize_area, x: [B,H,W,C]."""
    B, H, W, C = x.shape
    oh, ow = int(size[0]), int(size[1])

    def weights(n_in, n_out):
        scale = n_in / n_out
        m = torch.zeros(n_out, n_in, dtype=torch.float64)
        for o in range(n_out):
            start, end = o * scale, (o + 1) * scale
            j = int(math.floor(start))
            while j < math.ceil(end):
                lo, hi = max(start, j), min(end, j + 1)
                jj = min(max(j, 0), n_in - 1)
                if hi > lo:
                    m[o, jj] += hi - lo
                j += 1
        return (m / scale).to(torch.float32)

    wy = weights(H, oh)
    wx = weights(W, ow)
    out = torch.einsum("oh,bhwc->bowc", wy, x)
    return torch.einsum("pw,bowc->bopc", wx, out)


_GRAY = (0.2989, 0.5870, 0.1140)


def rgb_to_grayscale(x):
    """x: [B,H,W,3] -> [B,H,W,1]."""
    return (x[..., 0:1] * _GRAY[0] + x[..., 1:2] * _GRAY[1]) + x[..., 2:3] * _GRAY[2]


def conv2d_same_nhwc(x, w_hwio):
    """tf.nn.conv2d(x, w, [1,1,1,1], 'SAME') for NHWC x and HWIO weights (odd k)."""
    k = w_hwio.shape[0]
    w = w_hwio.permute(3, 2, 0, 1).contiguous().to(x)      # (constant filters: in x's dtype, on x's device)
    y = F.conv2d(x.permute(0, 3, 1, 2), w, None, stride=1, padding=k // 2)
    return y.permute(0, 2, 3, 1)
