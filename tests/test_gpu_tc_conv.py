"""The hand-written wgmma convolution kernels (csrc/tc_conv.cu, csrc/tc_wgrad.cu) through the C ABI
against float64 convolutions: every mode the FlowNet stacks use -- slim.conv2d with TF SAME padding at
stride 1 / 2, slim.conv2d_transpose (k4 s2), the input gradients of both, the weight gradients, the
row-window form of the 7x7 first layers -- including ragged channel counts, channel-sliced (pitched)
inputs and outputs, bias / leaky ReLU / accumulate epilogues.  Reference layers:
src/e2eflow/core/flownet.py:166-233 and :89-155.

Tolerance: 5e-6 of max|y| (3xTF32 split + fp32 register accumulation; measured ~1e-6, an fp32 FMA
loop over the same K is ~2e-5 at K = 9216)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL = 5e-6


def T():
    from unflow_b200.e2eflow.core import tc_conv
    return tc_conv


def rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))


def pitched(N, C, H, W, pitch, seed, fill=7.25):
    """NCHW-shaped view of an NHWC buffer with `pitch` floats per pixel; slack channels poisoned."""
    g = torch.Generator().manual_seed(seed)
    buf = torch.full((N, H, W, pitch), fill, device="cuda")
    v = buf[..., :C].permute(0, 3, 1, 2)
    v.copy_(torch.randn(N, C, H, W, generator=g).cuda())
    return v, buf


def cl(t):
    return t.contiguous(memory_format=torch.channels_last)


CONV = [  # N, Cin, Cout, H, W, k, stride, pads, x pitch, bias, act, accumulate
    (1, 32, 32, 8, 16, 1, 1, (0, 0, 0, 0), 32, False, False, False),
    (2, 64, 128, 16, 24, 3, 1, (1, 1, 1, 1), 64, True, True, False),
    (2, 70, 50, 13, 21, 3, 1, (1, 1, 1, 1), 80, True, True, False),
    (2, 64, 96, 12, 20, 3, 1, (1, 1, 1, 1), 64, False, False, True),
    (2, 64, 128, 16, 24, 3, 2, (0, 1, 0, 1), 64, True, True, False),
    (2, 40, 64, 16, 24, 5, 2, (1, 2, 1, 2), 40, True, True, False),
    (1, 473, 256, 12, 20, 3, 1, (1, 1, 1, 1), 476, True, True, False),
]


@pytest.mark.parametrize("N,Cin,Cout,H,W,k,stride,pads,xp,bias,act,accum", CONV)
def test_conv_forward(N, Cin, Cout, H, W, k, stride, pads, xp, bias, act, accum):
    t = T()
    pt, pb, pl, pr = pads
    x, _ = pitched(N, Cin, H, W, xp, seed=Cin + H)
    g = torch.Generator().manual_seed(Cout + k)
    w = cl((torch.randn(Cout, Cin, k, k, generator=g) * (2.0 / (Cin * k * k)) ** 0.5).cuda())
    b = (torch.randn(Cout + 1, generator=g) * 0.1).cuda()[1:] if bias else None       # 4-byte aligned only
    ref = F.conv2d(F.pad(x.double(), (pl, pr, pt, pb)), w.double(), b.double() if bias else None, stride=stride)
    if act:
        ref = F.leaky_relu(ref, 0.1)
    Ho, Wo = ref.shape[2:]
    out, obuf = pitched(N, Cout, Ho, Wo, t.round4(Cout) + 4, seed=1, fill=-3.5)
    if accum:
        ref = ref + out.double()
    else:
        out.fill_(float("nan"))
    t.run(x, t.split_weights(w), out, mode=0, stride=stride, kh=k, kw=k, pad_t=pt, pad_l=pl, bias=b, act=act,
          accumulate=accum)
    assert rel(out, ref) < TOL
    assert bool((obuf[..., Cout:] == -3.5).all())          # nothing written past C_out


@pytest.mark.parametrize("bias_act,accum,dense", [(True, False, True), (False, True, False), (False, False, False)])
def test_conv_k_slices(bias_act, accum, dense):
    """Few tiles, long K loop (the conv6 / conv6_1 shape of the step): the K loop of a tile is cut into slices
    on different CTAs whose partial sums meet in the output through atomics (zeroed first unless accumulating),
    bias + leaky ReLU as a separate pass.  Same result as the float64 convolution; slack channels untouched."""
    from unflow_b200 import _native
    t = T()
    N, Cin, Cout, H, W, k = 2, 1024, 256, 6, 20, 3
    x, _ = pitched(N, Cin, H, W, Cin, seed=5)
    g = torch.Generator().manual_seed(11)
    w = cl((torch.randn(Cout, Cin, k, k, generator=g) * (2.0 / (Cin * k * k)) ** 0.5).cuda())
    b = (torch.randn(Cout + 1, generator=g) * 0.1).cuda()[1:] if bias_act else None
    ref = F.conv2d(F.pad(x.double(), (1, 1, 1, 1)), w.double(), b.double() if bias_act else None)
    if bias_act:
        ref = F.leaky_relu(ref, 0.1)
    out, obuf = pitched(N, Cout, H, W, Cout if dense else Cout + 4, seed=1, fill=-3.5)
    if accum:
        ref = ref + out.double()
    else:
        out.fill_(float("nan"))
    planes = t.split_weights(w)
    res = {}
    for ks in (1, 0):
        assert _native.lib().unflow_set_int_option(b"tc_ksplit", ks) == 0
        o2 = out.clone() if not dense else None
        dst, dbuf = (out, obuf) if ks == 1 else pitched(N, Cout, H, W, Cout if dense else Cout + 4, seed=1, fill=-3.5)
        if ks == 0 and not accum:
            dst.fill_(float("nan"))
        t.run(x, planes, dst, mode=0, stride=1, kh=k, kw=k, pad_t=1, pad_l=1, bias=b, act=bias_act, accumulate=accum)
        res[ks] = dst.clone()
        assert rel(dst, ref) < TOL, ks
        if not dense:
            assert bool((dbuf[..., Cout:] == -3.5).all())
    _native.lib().unflow_set_int_option(b"tc_ksplit", 1)
    assert rel(res[1], res[0].double()) < 1e-5


DECONV = [  # N, Cin, Cout, H, W, k, stride, pad, out_hw, x pitch, bias+act
    (2, 64, 128, 6, 10, 4, 2, 1, None, 64, True),            # deconvN forward
    (2, 130, 64, 6, 20, 4, 2, 1, None, 132, True),
    (2, 128, 64, 8, 12, 3, 2, 0, (16, 24), 128, False),      # input gradient of 3x3 s2 SAME(0,1)
    (2, 128, 64, 8, 12, 5, 2, 1, (16, 24), 128, False),      # input gradient of 5x5 s2 SAME(1,2)
    (2, 128, 70, 9, 14, 3, 1, 1, None, 128, False),          # input gradient of 3x3 s1
]


@pytest.mark.parametrize("N,Cin,Cout,H,W,k,stride,pad,out_hw,xp,ba", DECONV)
def test_transposed_conv(N, Cin, Cout, H, W, k, stride, pad, out_hw, xp, ba):
    t = T()
    x, _ = pitched(N, Cin, H, W, xp, seed=Cin + W)
    g = torch.Generator().manual_seed(Cout + 3 * k)
    w = cl((torch.randn(Cin, Cout, k, k, generator=g) * (2.0 / (Cin * k * k / stride ** 2)) ** 0.5).cuda())
    b = (torch.randn(Cout, generator=g) * 0.1).cuda() if ba else None
    Ho, Wo = (H - 1) * stride - 2 * pad + k, (W - 1) * stride - 2 * pad + k
    oph = opw = 0
    if out_hw:
        oph, opw = out_hw[0] - Ho, out_hw[1] - Wo
        Ho, Wo = out_hw
    ref = F.conv_transpose2d(x.double(), w.double(), b.double() if ba else None, stride=stride, padding=pad,
                             output_padding=(max(oph, 0), max(opw, 0)))[:, :, :Ho, :Wo]
    if ba:
        ref = F.leaky_relu(ref, 0.1)
    out, obuf = pitched(N, Cout, Ho, Wo, t.round4(Cout) + 4, seed=2, fill=-3.5)
    out.fill_(float("nan"))
    t.run(x, t.split_weights(w, transpose=True), out, mode=1, stride=stride, kh=k, kw=k, pad_t=pad, pad_l=pad,
          bias=b, act=ba)
    assert rel(out, ref) < TOL
    assert bool((obuf[..., Cout:] == -3.5).all())


WGRAD = [  # N, Cin, Cout, H, W, k, stride, pads, x pitch
    (1, 32, 128, 8, 16, 1, 1, (0, 0, 0, 0), 32),
    (2, 64, 128, 16, 24, 3, 1, (1, 1, 1, 1), 64),
    (2, 70, 50, 13, 21, 3, 1, (1, 1, 1, 1), 80),
    (2, 64, 128, 16, 24, 3, 2, (0, 1, 0, 1), 64),
    (2, 24, 64, 16, 24, 5, 2, (1, 2, 1, 2), 24),
]


@pytest.mark.parametrize("N,Cin,Cout,H,W,k,stride,pads,xp", WGRAD)
def test_conv_weight_gradient(N, Cin, Cout, H, W, k, stride, pads, xp):
    t = T()
    pt, pb, pl, pr = pads
    x, _ = pitched(N, Cin, H, W, xp, seed=Cin + 1)
    Ho, Wo = (H + pt + pb - k) // stride + 1, (W + pl + pr - k) // stride + 1
    gy, _ = pitched(N, Cout, Ho, Wo, t.round4(Cout), seed=Cout + 2)
    ref = torch.nn.grad.conv2d_weight(F.pad(x.double(), (pl, pr, pt, pb)), (Cout, Cin, k, k), gy.double(), stride=stride)
    dw = cl(torch.zeros(Cout, Cin, k, k, device="cuda"))
    t.wgrad(gy, x, dw, stride=stride, kh=k, kw=k, pad_t=pt, pad_l=pl)
    assert rel(dw, ref) < TOL
    t.wgrad(gy, x, dw, stride=stride, kh=k, kw=k, pad_t=pt, pad_l=pl)        # accumulates (split-K atomics)
    assert rel(dw, 2 * ref) < TOL


def test_deconv_weight_gradient():
    t = T()
    N, Ci, Co, H, W = 2, 130, 64, 6, 10
    x, _ = pitched(N, Ci, H, W, 132, seed=3)
    gy, _ = pitched(N, Co, 2 * H, 2 * W, Co, seed=4)
    xr = x.double().clone().requires_grad_(True)
    wr = torch.zeros(Ci, Co, 4, 4, device="cuda", dtype=torch.float64, requires_grad=True)
    F.conv_transpose2d(xr, wr, stride=2, padding=1).backward(gy.double())
    dw = cl(torch.zeros(Ci, Co, 4, 4, device="cuda"))
    t.wgrad(x, gy, dw, stride=2, kh=4, kw=4, pad_t=1, pad_l=1)
    assert rel(dw, wr.grad) < TOL


@pytest.mark.parametrize("Ci,H,W", [(3, 24, 40), (6, 20, 28), (14, 16, 24)])
def test_first_layer_row_window_form(Ci, H, W):
    """7x7 stride-2 SAME(2,3) first layers: forward and weight gradient in the row-window form against
    the plain float64 convolution."""
    t = T()
    N, Co, k = 2, 64, 7
    g = torch.Generator().manual_seed(Ci)
    x = (torch.rand(N, Ci, H, W, generator=g) - 0.4).cuda()
    w = cl((torch.randn(Co, Ci, k, k, generator=g) * 0.05).cuda()).requires_grad_(True)
    b = (torch.randn(Co, generator=g) * 0.1).cuda()
    xd, wd = x.double(), w.detach().double().requires_grad_(True)
    ref = F.leaky_relu(F.conv2d(F.pad(xd, (2, 3, 2, 3)), wd, b.double(), stride=2), 0.1)
    Ho, Wo = ref.shape[2:]
    cp = t.window_channels(Ci)
    xp = t.window_input(x, 2, 2, Wo)
    w_rw = t.window_weights(w, cp)
    out = t.empty_nhwc(N, Co, Ho, Wo, x.device)
    t.run_window(xp, t.split_weights(w_rw.detach()), out, kh=k, stride=2, pad_t=2, bias=b, act=True)
    assert rel(out, ref) < TOL
    gy = torch.randn(N, Co, Ho, Wo, generator=g).cuda()
    gpre = cl(gy * torch.where(ref > 0, 1.0, 0.1).float())
    dw = torch.zeros((Co, k, 1, 8 * cp), device="cuda").permute(0, 3, 1, 2)
    t.wgrad_window(gpre, xp, dw, kh=k, stride=2, pad_t=2)
    w_rw.backward(dw)                                    # back through the pad / reshape to the variable
    ref.backward(gy.double())
    assert rel(w.grad, wd.grad) < TOL


def test_conv_ops_layers_run_on_the_tensor_core_kernels():
    """conv_ops.conv2d / conv_transpose2d in 3xTF32 mode: values and all three gradients of a conv and a
    deconv layer against float64 autograd, and the launch counter proves the wgmma kernels ran."""
    from unflow_b200 import _native
    from unflow_b200.e2eflow.core import conv_ops
    prev = conv_ops.get_mode()
    conv_ops.set_mode("3xtf32")
    try:
        g = torch.Generator().manual_seed(0)
        x = cl(torch.randn(2, 64, 16, 24, generator=g).cuda()).requires_grad_(True)
        w = cl((torch.randn(128, 64, 3, 3, generator=g) * 0.05).cuda()).requires_grad_(True)
        b = torch.zeros(128, device="cuda", requires_grad=True)
        wd = cl((torch.randn(128, 32, 4, 4, generator=g) * 0.05).cuda()).requires_grad_(True)
        bd = torch.zeros(32, device="cuda", requires_grad=True)
        n0 = _native.launch_count()
        y = conv_ops.conv2d(x, w, b, 2, (0, 1, 0, 1), act=True)
        z = conv_ops.conv_transpose2d(y, wd, bd, act=True)
        go = torch.randn(z.shape, generator=g).cuda()
        z.backward(go)
        assert _native.launch_count() - n0 >= 6
        xs, ws, bs, wds, bds = (t_.detach().double().requires_grad_(True) for t_ in (x, w, b, wd, bd))
        yr = F.leaky_relu(F.conv2d(F.pad(xs, (0, 1, 0, 1)), ws, bs, stride=2), 0.1)
        zr = F.leaky_relu(F.conv_transpose2d(yr, wds, bds, stride=2, padding=1), 0.1)
        zr.backward(go.double())
        assert rel(z, zr) < TOL
        for got, want in ((x.grad, xs.grad), (w.grad, ws.grad), (b.grad, bs.grad), (wd.grad, wds.grad), (bd.grad, bds.grad)):
            assert rel(got, want) < 2e-5
    finally:
        conv_ops.set_mode(prev)


@pytest.mark.parametrize("C,hw,act_pitch", [(4, (5, 7), 8), (32, (9, 11), 36), (64, (13, 21), 196), (128, (6, 10), 128),
                                            (200, (7, 9), 204), (2, (5, 6), 4)])
def test_lrelu_bwd_bias_pass(C, hw, act_pitch):
    """gpre = g * lrelu'(act) and the bias gradient in one pass (csrc/split.cu), for channel counts that fill
    a quarter / half / whole warp of float4 lanes and for the scalar path (C = 2); act is a channel slice
    of a wider NHWC buffer."""
    from unflow_b200.e2eflow.core import conv_ops
    N, (H, W) = 3, hw
    gen = torch.Generator().manual_seed(C)
    g = torch.randn(N, H, W, C, generator=gen).cuda().permute(0, 3, 1, 2)
    abuf = torch.randn(N, H, W, act_pitch, generator=gen).cuda()
    act = abuf[..., 1:1 + C].permute(0, 3, 1, 2) if act_pitch > C + 1 and C % 4 else abuf[..., :C].permute(0, 3, 1, 2)
    gpre, gb = conv_ops._lrelu_bwd_bias(g, act, True)
    want = g.double() * torch.where(act.double() > 0, 1.0, conv_ops.LRELU_SLOPE)
    assert float((gpre.double() - want).abs().max()) <= 1e-6 * float(want.abs().max())
    wb = want.sum((0, 2, 3))
    assert float((gb.double() - wb).abs().max()) <= 2e-6 * float(want.abs().sum((0, 2, 3)).max())


def test_launch_from_a_fresh_host_thread():
    """A host thread whose first CUDA call is one of the library's launchers -- autograd's backward worker running
    the correlation gradient, for one -- has no current context until something binds the device's primary
    context; the tensor-map encode inside the launcher has to do that itself (it failed with
    CUDA_ERROR_INVALID_CONTEXT).  Everything is prepared on the main thread, the launch happens on a new one."""
    import threading
    from unflow_b200 import _native
    tc = T()
    N, C, H, W = 2, 64, 16, 24
    g = torch.Generator().manual_seed(17)
    x = tc.empty_nhwc(N, C, H, W, "cuda")
    x.copy_(torch.randn(N, C, H, W, generator=g))
    w = torch.randn(C, 3, 3, C, generator=g).permute(0, 3, 1, 2).cuda()        # [Co][kh][kw][Ci] memory
    planes = tc.split_weights(w)
    want, got = tc.empty_nhwc(N, C, H, W, "cuda"), tc.empty_nhwc(N, C, H, W, "cuda")
    tc.run(x, planes, want, mode=0, stride=1, kh=3, kw=3, pad_t=1, pad_l=1)
    torch.cuda.synchronize()
    lib = _native.lib()
    xp, yp = tc.nhwc_geometry(x)[4], tc.nhwc_geometry(got)[4]
    result = {}

    def launch():
        result["rc"] = lib.unflow_tc_conv(x.data_ptr(), N, H, W, C, xp, planes.hi.data_ptr(), planes.lo.data_ptr(),
                                          got.data_ptr(), H, W, C, yp, None, 0.1, 0, 0, 0, 1, 3, 3, 1, 1, None)
        result["err"] = _native.last_error()
    t = threading.Thread(target=launch)
    t.start()
    t.join()
    assert result["rc"] == 0, result["err"]
    torch.cuda.synchronize()
    assert torch.equal(got, want)
