"""The 3xTF32 tensor-core conv path (core/conv_ops.py): accuracy against float64 and end-to-end parity of
the model against the fp32 oracle at the same tolerances as plain fp32.  No library convolution runs on a
CUDA tensor in this mode: the ``mode3x`` fixture makes them raise."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import flownet as oflownet
from oracle import unsupervised as ounsup
import synth
from test_gpu_step_launches import count_input_copies


def _no_library_conv(name, real):
    def call(*args, **kw):
        if any(isinstance(a, torch.Tensor) and a.is_cuda for a in args[:2]):
            raise AssertionError("library convolution %s on a CUDA tensor in 3xtf32 mode" % name)
        return real(*args, **kw)
    return call


@pytest.fixture
def mode3x(monkeypatch):
    # importing flownet sets the mode from UNFLOW_CONV_PRECISION: before set_mode, so that a test which is the first
    # to import it still runs in 3xtf32
    from unflow_b200.e2eflow.core import conv_ops, flownet  # noqa: F401
    for mod, name in ((F, "conv2d"), (F, "conv_transpose2d"), (torch.nn.grad, "conv2d_weight")):
        monkeypatch.setattr(mod, name, _no_library_conv(name, getattr(mod, name)))
    old = conv_ops.get_mode()
    conv_ops.set_mode('3xtf32')
    yield
    conv_ops.set_mode(old)


def rel(a, b):
    return float((a.double() - b).norm() / b.norm())


def on_gpu(x, layout):
    """``x`` (NCHW, CPU) on the GPU: 'nchw' contiguous; 'nhwc' dense NHWC; 'offset' a channel slice of an NHWC
    buffer starting at channel 1, so its base is 4 bytes past a 16-byte boundary (pitch C + 4); 'pitch' a channel
    slice of an NHWC buffer of pitch C + 2 (not a multiple of 4 for C % 4 == 0)."""
    if layout == "nchw":
        return x.cuda()
    before, after = {"nhwc": (0, 0), "offset": (1, 3), "pitch": (0, 2)}[layout]
    N, C, H, W = x.shape
    buf = torch.zeros(N, H, W, before + C + after)
    buf[..., before:before + C] = x.permute(0, 2, 3, 1)
    return buf.cuda()[..., before:before + C].permute(0, 3, 1, 2)


# (stride, k, pads, H, W, layout).  None of these inputs can be read in place by the tensor-core kernels, so each
# layer copies its input once (conv_ops._tc_input): NCHW memory, odd extents at stride 2 (the input gradient is a
# transposed launch and needs even ones; VALID padding shrinks the bottom / right pads below zero), a base that is
# not 16-byte aligned, a pixel pitch that is not a multiple of 4 floats.
CONV_CASES = {
    "1-3-pads0": (1, 3, (1, 1, 1, 1), 20, 28, "nchw"),
    "2-5-pads1": (2, 5, (1, 2, 1, 2), 20, 28, "nchw"),
    "2-7-pads2": (2, 7, (2, 3, 2, 3), 20, 28, "nchw"),
    "odd-2-3": (2, 3, (1, 1, 1, 1), 21, 27, "nhwc"),
    "odd-2-3-valid": (2, 3, (0, 0, 0, 0), 21, 27, "nhwc"),
    "unaligned-1-3": (1, 3, (1, 1, 1, 1), 20, 28, "offset"),
    "pitch-2-3": (2, 3, (0, 1, 0, 1), 20, 28, "pitch"),
}


@pytest.mark.parametrize("case", list(CONV_CASES))
def test_conv3x_matches_float64(mode3x, monkeypatch, case):
    from unflow_b200.e2eflow.core import conv_ops
    stride, k, pads, H, W, layout = CONV_CASES[case]
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 24, H, W, generator=g)
    w = torch.randn(16, 24, k, k, generator=g) * 0.1
    b = torch.randn(16, generator=g)
    xd = F.pad(x.double(), (pads[2], pads[3], pads[0], pads[1])).requires_grad_(True)
    wd, bd = w.double().requires_grad_(True), b.double().requires_grad_(True)
    yd = F.conv2d(xd, wd, bd, stride=stride)
    go = torch.randn(yd.shape, generator=g)
    yd.backward(go.double())
    xc, wc, bc = on_gpu(x, layout).requires_grad_(True), w.cuda().requires_grad_(True), b.cuda().requires_grad_(True)
    copies = count_input_copies(monkeypatch, conv_ops)
    y = conv_ops.conv2d(xc, wc, bc, stride, pads)
    y.backward(go.cuda())
    assert copies == [(2, 24, H, W)]
    gx_ref = xd.grad[:, :, pads[0]:pads[0] + H, pads[2]:pads[2] + W]
    for got, want, name in ((y, yd, "y"), (xc.grad, gx_ref, "dx"), (wc.grad, wd.grad, "dw"), (bc.grad, bd.grad, "db")):
        assert got.shape == want.shape, name
        e = rel(got.detach().cpu(), want.detach())
        assert e < 3e-5, "%s: rel err %.2e" % (name, e)   # measured: 2e-6 (3x3), 1e-5 (strided 5x5/7x7); 1xTF32 gives ~5e-4


@pytest.mark.parametrize("shape,stride", [((16, 24, 3, 5), 1), ((16, 24, 9, 9), 1), ((16, 24, 1, 1), 2)])
def test_conv3x_rejects_filters_the_kernels_do_not_take(mode3x, shape, stride):
    from unflow_b200.e2eflow.core import conv_ops
    x = torch.zeros(2, 24, 20, 28, device="cuda").contiguous(memory_format=torch.channels_last)
    with pytest.raises(ValueError, match="square k x k filters with stride <= k <= 8"):
        conv_ops.conv2d(x, torch.zeros(shape, device="cuda"), None, stride, (0, 0, 0, 0))


def test_deconv3x_matches_float64(mode3x):
    from unflow_b200.e2eflow.core import conv_ops
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 20, 9, 11, generator=g)
    w = torch.randn(20, 12, 4, 4, generator=g) * 0.1
    b = torch.randn(12, generator=g)
    xd, wd, bd = (t.double().requires_grad_(True) for t in (x, w, b))
    yd = F.conv_transpose2d(xd, wd, bd, stride=2, padding=1)
    go = torch.randn(yd.shape, generator=g)
    yd.backward(go.double())
    xc, wc, bc = x.cuda().requires_grad_(True), w.cuda().requires_grad_(True), b.cuda().requires_grad_(True)
    y = conv_ops.conv_transpose2d(xc, wc, bc)
    y.backward(go.cuda())
    for got, want, name in ((y, yd, "y"), (xc.grad, xd.grad, "dx"), (wc.grad, wd.grad, "dw"), (bc.grad, bd.grad, "db")):
        e = rel(got.detach().cpu(), want.detach())
        assert e < 2e-6, "%s: rel err %.2e" % (name, e)


def test_unsupervised_loss_3xtf32_vs_oracle(mode3x):
    """Same bar as the fp32 path: loss 2e-4, final flows 1e-4 relative, gradients in L2."""
    from unflow_b200.e2eflow.core.flownet import FlowNetVariables
    from unflow_b200.e2eflow.core.unsupervised import unsupervised_loss
    params = dict(synth.KITTI_PARAMS)
    tfv = oflownet.init_variables('C', False, seed=11)
    for k in tfv:
        tfv[k] = tfv[k].clone().requires_grad_(True)
    v = FlowNetVariables('C', False, seed=0).load_tf_dict({k: t.detach() for k, t in tfv.items()}).cuda()
    im1, im2, _ = synth.image_pair(1, 128, 256, seed=21)
    want_loss, want_fw, want_bw = ounsup.unsupervised_loss(tfv, (im1, im2), params, synth.KITTI_NORMALIZATION,
                                                           augment=False, return_flow=True)
    got_loss, got_fw, got_bw = unsupervised_loss((im1.cuda(), im2.cuda()), params, synth.KITTI_NORMALIZATION,
                                                 augment=False, return_flow=True, variables=v)
    assert abs(float(got_loss) - float(want_loss)) / abs(float(want_loss)) < 2e-4
    for g_, w_ in ((got_fw, want_fw), (got_bw, want_bw)):
        np.testing.assert_allclose(g_.detach().cpu().numpy(), w_.detach().numpy(), rtol=1e-4,
                                   atol=1e-4 * float(w_.abs().max()))
    want_loss.backward()
    got_loss.backward()
    for scope in v.kinds:
        w, _ = v.weights(scope)
        want = tfv[scope + '/weights'].grad.permute(3, 2, 0, 1)
        err = float((w.grad.cpu() - want).norm() / want.norm().clamp_min(1e-20))
        assert err < 5e-3, "%s: relative L2 gradient error %.3e" % (scope, err)


@pytest.mark.parametrize("deconv", [False, True])
def test_fused_bias_leaky_relu_layer_matches_float64(mode3x, deconv):
    """conv (+bias +leaky ReLU fused in the kernel's epilogue) and its backward (activation derivative and
    bias gradient in one pass over the incoming gradient) against float64."""
    from unflow_b200.e2eflow.core import conv_ops
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 12, 10, 14, generator=g)
    w = torch.randn(12, 8, 4, 4, generator=g) * 0.2 if deconv else torch.randn(8, 12, 3, 3, generator=g) * 0.2
    b = torch.randn(8, generator=g) * 0.5
    xd, wd, bd = (t.double().requires_grad_(True) for t in (x, w, b))
    yd = F.conv_transpose2d(xd, wd, bd, stride=2, padding=1) if deconv else F.conv2d(xd, wd, bd, padding=1)
    ad = F.leaky_relu(yd, 0.1)
    go = torch.randn(ad.shape, generator=g)
    ad.backward(go.double())
    xc, wc = x.cuda().requires_grad_(True), w.cuda().requires_grad_(True)
    # parameters are views into the flat buffer: only 4-byte aligned
    bc = torch.cat([torch.zeros(1), b]).cuda()[1:].detach().requires_grad_(True)
    assert bc.data_ptr() % 16 != 0
    a = (conv_ops.conv_transpose2d(xc, wc, bc, act=True) if deconv
         else conv_ops.conv2d(xc, wc, bc, 1, (1, 1, 1, 1), act=True))
    # feed the gradient through a channel-sliced, strided view like the concat backward does
    gbuf = torch.zeros(a.shape[0], a.shape[2], a.shape[3], a.shape[1] + 3, device="cuda")
    gview = gbuf.permute(0, 3, 1, 2)[:, 2:2 + a.shape[1]]
    gview.copy_(go.cuda())
    a.backward(gview)
    for got, want, name in ((a, ad, "a"), (xc.grad, xd.grad, "dx"), (wc.grad, wd.grad, "dw"), (bc.grad, bd.grad, "db")):
        e = rel(got.detach().cpu(), want.detach())
        assert e < 3e-5, "%s: rel err %.2e" % (name, e)


@pytest.mark.parametrize("N,C,H,W", [(2, 194, 37, 70), (1, 18, 16, 32), (3, 16, 5, 33), (1, 386, 48, 160)])
def test_narrow_flow_head_and_input_gradient_match_float64(mode3x, N, C, H, W):
    """csrc/narrow_conv.cu (the 2-channel 3x3 flow heads): forward, weight and bias gradients in
    exact fp32 against float64; ragged tiles, channel-chunk tails, strided incoming gradient,
    bit-identical repeats (fixed-order reduction).  The input gradient runs on the tensor-core kernel at
    every pixel pitch of the input, including pitches that are not a multiple of 4 (C = 194, 18, 386)."""
    from unflow_b200.e2eflow.core import conv_ops
    gen = torch.Generator().manual_seed(C * 1000 + H)
    x = torch.randn(N, C, H, W, generator=gen)
    w = torch.randn(2, C, 3, 3, generator=gen) * 0.1
    b = torch.randn(2, generator=gen)
    # the gradient arrives as a channel slice of a wider NHWC buffer (what the concat backward hands out)
    gwide = torch.randn(N, H, W, 5, generator=gen)
    xd, wd, bd = x.double().requires_grad_(True), w.double().requires_grad_(True), b.double().requires_grad_(True)
    yd = F.conv2d(xd, wd, bd, padding=1)
    gd = gwide.permute(0, 3, 1, 2)[:, 1:3].double()
    yd.backward(gd)

    xc = x.cuda().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    wc = w.cuda().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    bc = b.cuda().requires_grad_(True)
    y = conv_ops._NarrowConv3x3.apply(xc, wc, bc)
    assert y.shape == (N, 2, H, W) and y.stride() == (H * W * 4, 1, W * 4, 4)   # NHWC, 4 floats per pixel (TMA-readable)
    gc = gwide.cuda().permute(0, 3, 1, 2)[:, 1:3]
    y.backward(gc)
    assert rel(y.detach().cpu(), yd.detach()) < 2e-6
    assert rel(wc.grad.cpu(), wd.grad) < 2e-6
    assert rel(bc.grad.cpu(), bd.grad) < 2e-6
    assert rel(xc.grad.cpu(), xd.grad) < 3e-5                    # input gradient on the tensor-core kernel
    # the weight gradient is a fixed-order two-pass reduction: a second evaluation gives the same bits; the
    # forward is bit-repeatable when one CTA owns a tile (the full-size heads), while small images split the
    # channels over CTAs whose partial sums meet through atomics (order free, values within rounding)
    wc2 = wc.detach().clone().requires_grad_(True)
    y2 = conv_ops._NarrowConv3x3.apply(xc.detach(), wc2, bc.detach())
    y2.backward(gc)
    assert torch.equal(wc2.grad, wc.grad)
    if N * ((H + 15) // 16) * ((W + 31) // 32) >= 2 * 132:      # 132 SMs (H100 SXM)
        assert torch.equal(y2, y)
    else:
        assert rel(y2.detach().cpu(), y.detach().cpu()) < 1e-6
    # no bias, and the dispatch rule of conv2d
    y3 = conv_ops._NarrowConv3x3.apply(xc.detach(), wc.detach(), None)
    assert rel((y3 + bc.detach().view(1, 2, 1, 1)).cpu(), yd.detach()) < 2e-6
    assert conv_ops._use_narrow(xc, wc, 1, (1, 1, 1, 1))
    assert not conv_ops._use_narrow(xc, wc, 2, (1, 1, 1, 1)) and not conv_ops._use_narrow(xc, wc, 1, (0, 1, 0, 1))


@pytest.mark.parametrize("N,C,H,W", [(2, 194, 37, 70), (1, 386, 48, 160), (2, 1026, 6, 20), (1, 20, 16, 32)])
@pytest.mark.parametrize("path", ["tma", "cp_async"])
def test_narrow_flow_head_tma_and_cp_async_kernels(mode3x, N, C, H, W, path):
    """Both implementations of the flow-head kernels (csrc/narrow_conv_tma.cu: TMA-staged NHWC tiles;
    csrc/narrow_conv.cu: cp.async staging, the fallback for pixel pitches TMA cannot address) on an input that is
    a channel slice of a pitch-padded NHWC buffer, as the decoder's concat buffers are; against float64.  The
    launcher picks the kernels from the pitch: a multiple of 4 floats takes TMA, any other the cp.async kernels."""
    from torch.profiler import ProfilerActivity, profile
    from unflow_b200.e2eflow.core import conv_ops
    tma = path == "tma"
    gen = torch.Generator().manual_seed(C + 7 * H)
    pitch, c0 = ((C + 3) // 4 * 4 + 4, 4) if tma else ((C if C % 4 == 2 else C + 2), 0)
    buf = torch.randn(N, H, W, pitch, generator=gen)
    x = buf[..., c0:c0 + C].permute(0, 3, 1, 2)
    w = torch.randn(2, C, 3, 3, generator=gen) * 0.1
    b = torch.randn(2, generator=gen)
    g = torch.randn(N, 2, H, W, generator=gen)
    xd, wd, bd = x.double(), w.double().requires_grad_(True), b.double().requires_grad_(True)
    yd = F.conv2d(xd, wd, bd, padding=1)
    yd.backward(g.double())
    xc = buf.cuda()[..., c0:c0 + C].permute(0, 3, 1, 2)
    wc = w.cuda().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    bc = b.cuda().requires_grad_(True)
    gc = g.cuda()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.ones(4, device="cuda").add_(1)          # a session can miss the activity issued right at its start
        y = conv_ops._NarrowConv3x3.apply(xc, wc, bc)
        y.backward(gc)
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    ran = {k: any(k in nm for nm in names) for k in ("narrow_fwd_tma_kernel", "narrow_wgrad_tma_kernel",
                                                     "narrow_fwd_kernel", "narrow_wgrad_kernel")}
    assert ran == {"narrow_fwd_tma_kernel": bool(tma), "narrow_wgrad_tma_kernel": bool(tma),
                   "narrow_fwd_kernel": not tma, "narrow_wgrad_kernel": not tma}, (ran, sorted(names))
    assert rel(y.detach().cpu(), yd.detach()) < 2e-6
    assert rel(wc.grad.cpu(), wd.grad) < 2e-6
    assert rel(bc.grad.cpu(), bd.grad) < 2e-6


def test_narrow_conv_rejects_other_shapes():
    from unflow_b200 import _native
    x = torch.zeros(1, 4, 4, 6, device="cuda")
    y = torch.zeros(1, 4, 4, 2, device="cuda")
    w = torch.zeros(2, 3, 3, 6, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    lib = _native.lib()
    assert lib.unflow_conv3x3_narrow_fwd(x.data_ptr(), 6, w.data_ptr(), None, y.data_ptr(), 2, 1, 4, 4, 6, 4, s) == 1
    assert "2 output channels" in _native.lib().unflow_last_error().decode()
    assert lib.unflow_conv3x3_narrow_fwd(x.data_ptr(), 6, w.data_ptr(), None, y.data_ptr(), 2, 1, 4, 4, 5, 2, s) == 1
    assert lib.unflow_conv3x3_narrow_fwd(x.data_ptr(), 4, w.data_ptr(), None, y.data_ptr(), 2, 1, 4, 4, 6, 2, s) == 1   # pitch < C
    assert lib.unflow_conv3x3_narrow_fwd(x.data_ptr(), 6, w.data_ptr(), None, y.data_ptr(), 3, 1, 4, 4, 6, 2, s) == 1   # odd y pitch
    assert lib.unflow_conv3x3_narrow_wgrad_workspace_bytes(2, 16, 32, 6) == 2 * 18 * 6 * 4
    assert lib.unflow_conv3x3_narrow_wgrad_workspace_bytes(2, 17, 33, 6) == 8 * 18 * 6 * 4


def test_narrow_conv_on_a_channel_slice_of_a_wider_buffer(mode3x):
    """The flow heads read their input in place from the (pitch-padded) concat buffers: a channel slice
    with a larger pixel pitch must give the same results as the dense copy."""
    from unflow_b200.e2eflow.core import conv_ops
    gen = torch.Generator().manual_seed(3)
    buf = torch.randn(2, 37, 70, 200, generator=gen).cuda()
    xs = buf[..., 4:198].permute(0, 3, 1, 2)                            # 194 channels, pitch 200
    xd = xs.contiguous(memory_format=torch.channels_last)
    w = (torch.randn(2, 194, 3, 3, generator=gen) * 0.1).cuda().contiguous(memory_format=torch.channels_last)
    b = torch.randn(2, generator=gen).cuda()
    g = torch.randn(2, 2, 37, 70, generator=gen).cuda()
    outs = []
    for x in (xd, xs):
        wr = w.clone().requires_grad_(True)
        y = conv_ops._NarrowConv3x3.apply(x, wr, b)
        y.backward(g)
        outs.append((y.detach().clone(), wr.grad.clone()))
    # 18 tiles < 2 x 132 SMs: the forward splits the channels over several CTAs that add their parts with
    # atomics (order not fixed), the weight gradient splits them into disjoint ranges (bit-identical)
    # (the dense copy has a pixel pitch of 194 floats, which TMA cannot address: it runs on the cp.async kernels,
    # the pitch-200 slice on the TMA-staged ones -- same sums in another order)
    assert (outs[0][1] - outs[1][1]).abs().max().item() < 2e-5 * outs[0][1].abs().max().item()
    assert (outs[0][0] - outs[1][0]).abs().max().item() < 1e-5 * outs[0][0].abs().max().item()


@pytest.mark.parametrize("cin,hw", [(3, (20, 28)), (14, (22, 26)), (6, (21, 27))])
def test_first_layer_space_to_depth_matches_float64(mode3x, cin, hw):
    """7x7 stride-2 first layers run as 4x4 stride-1 convs over 2x2 pixel blocks (conv_ops.
    space_to_depth_operands); against the direct float64 convolution with TF SAME padding."""
    from unflow_b200.e2eflow.core import conv_ops
    from unflow_b200.e2eflow.core.flownet import _same_pad
    g = torch.Generator().manual_seed(cin)
    H, W = hw
    x = torch.randn(2, cin, H, W, generator=g)
    w = torch.randn(16, cin, 7, 7, generator=g) * 0.1
    b = torch.randn(16, generator=g)
    pads = _same_pad(H, 7, 2) + _same_pad(W, 7, 2)
    xd = F.pad(x.double(), (pads[2], pads[3], pads[0], pads[1])).requires_grad_(True)
    wd, bd = w.double().requires_grad_(True), b.double().requires_grad_(True)
    yd = F.leaky_relu(F.conv2d(xd, wd, bd, stride=2), 0.1)
    go = torch.randn(yd.shape, generator=g)
    yd.backward(go.double())
    xc = x.cuda().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    wc, bc = w.cuda().requires_grad_(True), b.cuda().requires_grad_(True)
    assert conv_ops._use_space_to_depth(xc, wc, 2)
    y = conv_ops.conv2d(xc, wc, bc, 2, pads, act=True)
    y.backward(go.cuda())
    gx_ref = xd.grad[:, :, pads[0]:pads[0] + H, pads[2]:pads[2] + W]
    for got, want, name in ((y, yd, "y"), (xc.grad, gx_ref, "dx"), (wc.grad, wd.grad, "dw"), (bc.grad, bd.grad, "db")):
        e = rel(got.detach().cpu(), want.detach())
        assert got.shape == want.shape and e < 1e-4, "%s: rel err %.2e" % (name, e)
