"""The 3xTF32 tensor-core conv path (core/conv_ops.py + csrc/split.cu): accuracy against float64
and end-to-end parity of the model against the fp32 oracle at the same tolerances as plain fp32."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import flownet as oflownet
from oracle import unsupervised as ounsup
import synth


@pytest.fixture
def mode3x():
    from unflow_b200.e2eflow.core import conv_ops
    old = conv_ops.get_mode()
    conv_ops.set_mode('3xtf32')
    yield
    conv_ops.set_mode(old)


def rel(a, b):
    return float((a.double() - b).norm() / b.norm())


def test_operand_kernel_exact():
    """csrc/split.cu: exact hi/lo decomposition, channel / batch concatenation, zero padding of
    channels, items and the TF-SAME border, arbitrary source strides."""
    from unflow_b200.e2eflow.core.conv_ops import _operand
    base = torch.randn(3, 7, 9, 6, device="cuda") * 100          # NHWC memory
    x = base.permute(0, 3, 1, 2)[:, :5]                           # [3,5,7,9] channel-sliced channels_last view
    s = _operand(x, 0, c_pad=8, pads=(1, 2, 0, 1))               # -> [3, 24, 10, 10]
    assert s.shape == (3, 24, 10, 10) and s.is_contiguous(memory_format=torch.channels_last)
    hi, hi2, lo = s[:, 0:8], s[:, 8:16], s[:, 16:24]
    assert torch.equal(hi, hi2)
    inner = (slice(None), slice(0, 5), slice(1, 8), slice(0, 9))
    assert torch.equal((hi + lo)[inner], x)                       # exact decomposition
    assert int((hi.contiguous().view(torch.int32) & 0x1FFF).abs().max()) == 0   # hi is a TF32 number
    total = (hi + lo)
    mask = torch.zeros_like(total, dtype=torch.bool)
    mask[inner] = True
    assert float(total[~mask].abs().max()) == 0.0                 # channel pad + spatial border are zeros
    assert float((lo[inner].abs() / x.abs()).max()) <= 2.0 ** -11
    # batch concat, order (hi;lo;hi), extra zero items, NCHW-contiguous source (weights)
    w = torch.randn(5, 3, 4, 4, device="cuda")
    b = _operand(w, 1, concat_batch=True, c_pad=4, n_out=8)      # -> [24, 4, 4, 4]
    assert b.shape == (24, 4, 4, 4)
    h0, l0, h1 = b[0:8], b[8:16], b[16:24]
    assert torch.equal(h0, h1) and torch.equal((h0 + l0)[:5, :3], w)
    assert float(h0[5:].abs().max()) == 0.0 and float(h0[:, 3:].abs().max()) == 0.0


@pytest.mark.parametrize("stride,k,pads", [(1, 3, (1, 1, 1, 1)), (2, 5, (1, 2, 1, 2)), (2, 7, (2, 3, 2, 3))])
def test_conv3x_matches_float64(mode3x, stride, k, pads):
    from unflow_b200.e2eflow.core import conv_ops
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 24, 20, 28, generator=g)
    w = torch.randn(16, 24, k, k, generator=g) * 0.1
    b = torch.randn(16, generator=g)
    xd = F.pad(x.double(), (pads[2], pads[3], pads[0], pads[1])).requires_grad_(True)
    wd, bd = w.double().requires_grad_(True), b.double().requires_grad_(True)
    yd = F.conv2d(xd, wd, bd, stride=stride)
    go = torch.randn(yd.shape, generator=g)
    yd.backward(go.double())
    xc, wc, bc = x.cuda().requires_grad_(True), w.cuda().requires_grad_(True), b.cuda().requires_grad_(True)
    y = conv_ops.conv2d(xc, wc, bc, stride, pads)
    y.backward(go.cuda())
    H, W = x.shape[2], x.shape[3]
    gx_ref = xd.grad[:, :, pads[0]:pads[0] + H, pads[2]:pads[2] + W]
    for got, want, name in ((y, yd, "y"), (xc.grad, gx_ref, "dx"), (wc.grad, wd.grad, "dw"), (bc.grad, bd.grad, "db")):
        e = rel(got.detach().cpu(), want.detach())
        assert e < 3e-5, "%s: rel err %.2e" % (name, e)   # measured: 2e-6 (3x3), 1e-5 (strided 5x5/7x7); 1xTF32 gives ~5e-4


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
    """conv (+bias +leaky ReLU fused in one pass) and its backward (activation derivative folded into
    the operand kernel, masked bias gradient) against float64."""
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
def test_narrow_flow_head_matches_float64(mode3x, N, C, H, W):
    """csrc/narrow_conv.cu (the 2-channel 3x3 flow heads): forward, weight and bias gradients in
    exact fp32 against float64; ragged tiles, channel-chunk tails, strided incoming gradient,
    bit-identical repeats (fixed-order reduction)."""
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
    tiles = N * ((H + 15) // 16) * ((W + 31) // 32)
    assert conv_ops._use_narrow(xc, wc, 1, (1, 1, 1, 1)) == (tiles >= conv_ops.NARROW_MIN_TILES)
    assert not conv_ops._use_narrow(xc, wc, 2, (1, 1, 1, 1)) and not conv_ops._use_narrow(xc, wc, 1, (0, 1, 0, 1))


@pytest.mark.parametrize("N,C,H,W", [(2, 194, 37, 70), (1, 386, 48, 160), (2, 1026, 6, 20), (1, 20, 16, 32)])
@pytest.mark.parametrize("tma", [1, 0])
def test_narrow_flow_head_tma_and_cp_async_kernels(mode3x, N, C, H, W, tma):
    """Both implementations of the flow-head kernels (csrc/narrow_conv_tma.cu: TMA-staged NHWC tiles;
    csrc/narrow_conv.cu: cp.async staging, the fallback for pitches TMA cannot address) on an input that is a
    channel slice of a pitch-padded NHWC buffer, as the decoder's concat buffers are; against float64."""
    from unflow_b200 import _native
    from unflow_b200.e2eflow.core import conv_ops
    gen = torch.Generator().manual_seed(C + 7 * H)
    pitch = (C + 3) // 4 * 4 + 4
    buf = torch.randn(N, H, W, pitch, generator=gen)
    x = buf[..., 4:4 + C].permute(0, 3, 1, 2)
    w = torch.randn(2, C, 3, 3, generator=gen) * 0.1
    b = torch.randn(2, generator=gen)
    g = torch.randn(N, 2, H, W, generator=gen)
    xd, wd, bd = x.double(), w.double().requires_grad_(True), b.double().requires_grad_(True)
    yd = F.conv2d(xd, wd, bd, padding=1)
    yd.backward(g.double())
    lib = _native.lib()
    assert lib.unflow_set_int_option(b"narrow_fwd_tma", tma) == 0
    try:
        xc = buf.cuda()[..., 4:4 + C].permute(0, 3, 1, 2)
        wc = w.cuda().contiguous(memory_format=torch.channels_last).requires_grad_(True)
        bc = b.cuda().requires_grad_(True)
        y = conv_ops._NarrowConv3x3.apply(xc, wc, bc)
        y.backward(g.cuda())
        torch.cuda.synchronize()
    finally:
        lib.unflow_set_int_option(b"narrow_fwd_tma", 1)
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
