"""Host side of csrc/tc_conv.cu: the hand-written wgmma (3xTF32, register accumulators) implicit-GEMM
convolution behind the conv / deconv stacks (reference slim.conv2d / slim.conv2d_transpose,
src/e2eflow/core/flownet.py:166-233, :89-155).

All tensors are NHWC in memory (what torch calls channels_last); a tensor may be a channel slice of
a wider buffer (a concat buffer): the kernels take the channel PITCH separately.  No fallback: the
functions raise when the CUDA library is missing or the shape is not served (``supported`` says which
shapes are)."""
import torch

from ... import _native
from ..._native import check


def _stream():
    return torch.cuda.current_stream().cuda_stream


def round4(c):
    return (c + 3) // 4 * 4


def nhwc_geometry(t):
    """(N, H, W, C, channel pitch) of an NCHW-shaped tensor whose memory is NHWC (channels_last),
    possibly a channel slice of a wider NHWC buffer; None when the memory is laid out otherwise."""
    if t.dim() != 4:
        return None
    N, C, H, W = t.shape
    sN, sC, sH, sW = t.stride()
    if C > 1 and sC != 1:
        return None
    pitch = sW if W > 1 else (sH if H > 1 else max(C, 1))
    if pitch < C or (W > 1 and sW != pitch) or (H > 1 and sH != W * pitch) or (N > 1 and sN != H * W * pitch):
        return None
    return N, H, W, C, pitch


def supported(x):
    """Tensors the tensor-core kernel reads or writes: NHWC memory, 16-byte aligned base, channel
    pitch a multiple of 4 floats."""
    g = nhwc_geometry(x)
    return (x.is_cuda and x.dtype == torch.float32 and g is not None and g[4] % 4 == 0
            and x.data_ptr() % 16 == 0)


class WeightPlanes:
    """hi / lo TF32 planes of one variable in the K-major layout [taps][rows][Cp] (rows = the GEMM's
    output channels, Cp = contraction channels rounded up to 4)."""

    def __init__(self, hi, lo, taps, rows, cols):
        self.hi, self.lo, self.taps, self.rows, self.cols = hi, lo, taps, rows, cols


def split_weights(w, transpose=False):
    """``w``: a conv variable [A, B, kh, kw] stored NHWC-ordered ([A][kh][kw][B] in memory -- OIHW
    convolution weights or IOHW transposed-convolution weights, core/flownet.py FlowNetVariables).
    Returns planes with rows = A and contraction = B (``transpose=False``) or rows = B and
    contraction = A (``transpose=True``)."""
    A, B, kh, kw = w.shape
    want = (kh * kw * B, 1, kw * B, B)
    assert all(n == 1 or s == t for n, s, t in zip(w.shape, w.stride(), want)), \
        "weights must be stored [A][kh][kw][B] (got strides %s)" % (w.stride(),)
    taps = kh * kw
    if transpose:
        rows, cols, s_t, s_r, s_c = B, A, B, 1, taps * B
    else:
        rows, cols, s_t, s_r, s_c = A, B, B, taps * B, 1
    cp = round4(cols)
    hi = torch.empty((taps, rows, cp), device=w.device, dtype=torch.float32)
    lo = torch.empty_like(hi)
    with torch.cuda.device(w.device):
        check(_native.lib().unflow_tc_wsplit(w.data_ptr(), hi.data_ptr(), lo.data_ptr(), taps, rows, cols,
                                             s_t, s_r, s_c, _stream()), "tc_wsplit")
    return WeightPlanes(hi, lo, taps, rows, cols)


def run(x, planes, out, *, mode, stride, kh, kw, pad_t, pad_l, bias=None, act=False, accumulate=False,
        slope=0.1):
    """out (+)= act(bias + conv(x)) -- ``x`` / ``out``: NCHW-shaped tensors with NHWC memory (channel
    slices allowed).  mode 0: convolution with offsets (pad_t, pad_l); mode 1: transposed convolution
    (o = stride * i - pad + k)."""
    gx, go = nhwc_geometry(x), nhwc_geometry(out)
    assert gx is not None and go is not None, "tc_conv needs NHWC (channels_last) memory"
    N, Hin, Win, Cin, xp = gx
    No, Hout, Wout, Cout, yp = go
    assert No == N and planes.rows == Cout and planes.cols == Cin and planes.taps == kh * kw
    from ..ops import kernel_timer
    pix = N * (Hin * Win if mode == 1 else Hout * Wout)       # positions each tap is applied to
    flops = 2 * pix * Cout * Cin * kh * kw            # nominal fp32 multiply-adds x 2 (executed as 3 TF32 MMAs each)
    with torch.cuda.device(x.device), kernel_timer.span("tc_conv", flops):
        check(_native.lib().unflow_tc_conv(
            x.data_ptr(), N, Hin, Win, Cin, xp, planes.hi.data_ptr(), planes.lo.data_ptr(),
            out.data_ptr(), Hout, Wout, Cout, yp, bias.data_ptr() if bias is not None else None,
            float(slope), 1 if act else 0, 1 if accumulate else 0, mode, stride, kh, kw,
            pad_t, pad_l, _stream()), "tc_conv")
    return out


def empty_nhwc(N, C, H, W, device):
    """An NCHW-shaped tensor with dense NHWC memory."""
    return torch.empty((N, H, W, C), device=device, dtype=torch.float32).permute(0, 3, 1, 2)


def wgrad(P, G, dw, *, stride, kh, kw, pad_t, pad_l):
    """dw[r, t, c] += sum_p P[p, r] * G[stride * p + (k - pad), c]  (csrc/tc_wgrad.cu).  ``P`` / ``G``:
    NCHW-shaped tensors with NHWC memory; ``dw``: a ZEROED (or to-be-accumulated) variable-shaped tensor
    [rows, cols, kh, kw] stored [rows][kh][kw][cols]."""
    gp, gg = nhwc_geometry(P), nhwc_geometry(G)
    assert gp is not None and gg is not None, "tc_wgrad needs NHWC (channels_last) memory"
    N, Hp, Wp, R, pp = gp
    Ng, Hg, Wg, C, gpitch = gg
    A, B, k1, k2 = dw.shape
    assert (A, B, k1, k2) == (R, C, kh, kw) and Ng == N
    want = (kh * kw * C, 1, kw * C, C)
    assert all(n == 1 or s == t for n, s, t in zip(dw.shape, dw.stride(), want)), "dw must be stored [rows][kh][kw][cols]"
    from ..ops import kernel_timer
    with torch.cuda.device(P.device), kernel_timer.span("tc_wgrad", 2 * N * Hp * Wp * R * C * kh * kw):
        check(_native.lib().unflow_tc_wgrad(P.data_ptr(), N, Hp, Wp, R, pp, G.data_ptr(), Hg, Wg, C, gpitch,
                                            dw.data_ptr(), kh * kw * C, C, stride, kh, kw, pad_t, pad_l,
                                            _stream()), "tc_wgrad")
    return dw


# ---- first layers in the row-window form (unflow_tc_conv_window / unflow_tc_wgrad_window) ----------
def window_channels(c):
    """Padded channel count (floats per pixel) of the row-window input: 4, 8 or 16; None if c > 16."""
    for cp in (4, 8, 16):
        if c <= cp:
            return cp
    return None


def window_input(x, pad_l, stride, wout):
    """x: NCHW-shaped [N,C,H,W] (any strides) -> the zero-padded NHWC buffer [N,H,Wp,Cp] the window kernels
    read: pad_l zero pixels on the left, zeros on the right up to the end of the last 8-pixel window."""
    N, C, H, W = x.shape
    cp = window_channels(C)
    wp = max(W + pad_l, stride * (wout - 1) + 8)
    buf = torch.zeros((N, H, wp, cp), device=x.device, dtype=torch.float32)
    buf[:, :, pad_l:pad_l + W, :C].copy_(x.permute(0, 2, 3, 1))
    return buf


def window_weights(w, cp):
    """[Co, Ci, kh, kw] variable (memory [Co][kh][kw][Ci]) -> the differentiable row-window form
    [Co, 8*cp, kh, 1] (memory [Co][kh][1][8*cp], column kx*cp + c; zero for kx >= kw, c >= Ci)."""
    Co, Ci, kh, kw = w.shape
    assert kw <= 8 and Ci <= cp
    wn = torch.nn.functional.pad(w.permute(0, 2, 3, 1), (0, cp - Ci, 0, 8 - kw))       # [Co, kh, 8, cp]
    return wn.reshape(Co, kh, 1, 8 * cp).permute(0, 3, 1, 2)


def run_window(xp, planes, out, *, kh, stride, pad_t, bias=None, act=False, slope=0.1):
    N, H, Wp, Cp = xp.shape
    go = nhwc_geometry(out)
    No, Hout, Wout, Cout, yp = go
    assert No == N and planes.rows == Cout and planes.cols == 8 * Cp and planes.taps == kh and xp.is_contiguous()
    from ..ops import kernel_timer
    with torch.cuda.device(xp.device), kernel_timer.span("tc_conv", 2 * N * Hout * Wout * Cout * 8 * Cp * kh):
        check(_native.lib().unflow_tc_conv_window(
            xp.data_ptr(), N, H, Wp, Cp, planes.hi.data_ptr(), planes.lo.data_ptr(), out.data_ptr(), Hout, Wout,
            Cout, yp, bias.data_ptr() if bias is not None else None, float(slope), 1 if act else 0, kh, stride,
            pad_t, _stream()), "tc_conv_window")
    return out


def wgrad_window(P, xp, dw, *, kh, stride, pad_t):
    """dw [Co, 8*Cp, kh, 1] (memory [Co][kh][1][8*Cp], zeroed) += the row-window weight gradient."""
    N, Ho, Wo, R, pp = nhwc_geometry(P)
    Nx, H, Wp, Cp = xp.shape
    assert Nx == N and tuple(dw.shape) == (R, 8 * Cp, kh, 1) and xp.is_contiguous()
    want = (kh * 8 * Cp, 1, 8 * Cp, 8 * Cp)
    assert all(n == 1 or s == t for n, s, t in zip(dw.shape, dw.stride(), want))
    from ..ops import kernel_timer
    with torch.cuda.device(P.device), kernel_timer.span("tc_wgrad", 2 * N * Ho * Wo * R * 8 * Cp * kh):
        check(_native.lib().unflow_tc_wgrad_window(P.data_ptr(), N, Ho, Wo, R, pp, xp.data_ptr(), H, Wp, Cp,
                                                   dw.data_ptr(), kh, stride, pad_t, _stream()), "tc_wgrad_window")
    return dw
