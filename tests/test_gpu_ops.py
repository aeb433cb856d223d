"""GPU parity of the four custom ops, called through the reference-style Python surface
(unflow_b200.e2eflow.ops -> ctypes -> C ABI -> sm_90a kernels), against the CPU oracle on the
same seeded inputs and against the reference's own known-answer vectors."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import ops as oops
from oracle.image_warp import image_warp as oimage_warp


def _ops():
    from unflow_b200.e2eflow import ops
    return ops


def rnd(shape, seed, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


def t(a):
    return torch.tensor(np.asarray(a), dtype=torch.float32)


def close(got, want, rtol=1e-4, atol_rel=1e-5):
    want = want.detach().cpu()
    got = got.detach().cpu()
    atol = atol_rel * max(float(want.abs().max()), 1e-12)
    np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=rtol, atol=atol)


# ------------------------------------------------------------------ reference KATs
@pytest.mark.parametrize("name", ["test_correlation_trivial", "test_correlation_batch"])
def test_correlation_reference_kats(kats, arr, name):
    call = kats["correlation"][name]["calls"][0]
    in0, in1, expected = (arr(a) for a in call["args"])
    out = _ops().correlation(t(in0).cuda(), t(in1).cuda(), **call["kwargs"])
    np.testing.assert_allclose(out.cpu().numpy(), expected, rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("name", ["test_move", "test_batches", "test_interpolate"])
def test_backward_warp_reference_kats(kats, arr, name):
    call = kats["backward_warp"][name]["calls"][0]
    first, second, flow = (arr(a) for a in call["args"])
    pred = _ops().backward_warp(t(second).cuda(), t(flow).cuda())
    np.testing.assert_allclose(pred.cpu().numpy(), first, rtol=1e-6, atol=1e-6)


def test_downsample_reference_kat(kats, arr):
    v = kats["downsample"]["test_downsample"]["vars"]
    first = t(arr(v["first"]).reshape(1, 4, 4, 1)).cuda()
    np.testing.assert_allclose(_ops().downsample(first, 2).cpu().numpy(),
                               arr(v["second"]).reshape(1, 2, 2, 1), rtol=1e-6, atol=1e-6)


# ------------------------------------------------------------------ correlation vs oracle
CORR_CASES = [
    # generic path
    dict(shape=(2, 5, 7, 9), kernel_size=1, max_displacement=4, pad=4, stride_1=1, stride_2=2),
    dict(shape=(1, 3, 6, 8), kernel_size=1, max_displacement=3, pad=3, stride_1=1, stride_2=1),
    dict(shape=(1, 4, 9, 10), kernel_size=3, max_displacement=2, pad=3, stride_1=1, stride_2=1),
    dict(shape=(2, 2, 9, 11), kernel_size=3, max_displacement=2, pad=3, stride_1=2, stride_2=2),
    dict(shape=(1, 3, 8, 9), kernel_size=1, max_displacement=4, pad=2, stride_1=1, stride_2=2),
    # tiled TMA path (K=1, s1=1, s2=2, pad==md, H even, W%4==0, W>=16)
    dict(shape=(2, 16, 8, 16), kernel_size=1, max_displacement=4, pad=4, stride_1=1, stride_2=2),
    dict(shape=(1, 13, 10, 20), kernel_size=1, max_displacement=20, pad=20, stride_1=1, stride_2=2),
    dict(shape=(2, 32, 12, 40), kernel_size=1, max_displacement=20, pad=20, stride_1=1, stride_2=2),
    dict(shape=(1, 64, 48, 64), kernel_size=1, max_displacement=20, pad=20, stride_1=1, stride_2=2),
    dict(shape=(1, 8, 6, 36), kernel_size=1, max_displacement=7, pad=7, stride_1=1, stride_2=2),
    # tiled backward: two channel slabs (one partial), H % 4 != 0, partial column tile
    dict(shape=(1, 130, 6, 24), kernel_size=1, max_displacement=20, pad=20, stride_1=1, stride_2=2),
    dict(shape=(2, 40, 14, 72), kernel_size=1, max_displacement=8, pad=8, stride_1=1, stride_2=2),
]


@pytest.mark.parametrize("case", CORR_CASES)
def test_correlation_fwd_bwd_vs_oracle(case):
    case = dict(case)
    shape = case.pop("shape")
    a, b = rnd(shape, 11), rnd(shape, 12)
    ao, bo = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
    ag, bg = a.cuda().requires_grad_(True), b.cuda().requires_grad_(True)
    want = oops.correlation(ao, bo, **case)
    got = _ops().correlation(ag, bg, **case)
    assert got.shape == want.shape
    close(got, want)
    w = rnd(tuple(want.shape), 13)
    (want * w).sum().backward()
    (got * w.cuda()).sum().backward()
    close(ag.grad, ao.grad)
    close(bg.grad, bo.grad)


def test_correlation_path_selection():
    from unflow_b200 import _native
    lib = _native.lib()
    assert lib.unflow_correlation_fwd_path(256, 48, 160, 1, 20, 20, 1, 2) == 1
    assert lib.unflow_correlation_fwd_path(256, 48, 160, 3, 20, 20, 1, 2) == 0


def test_correlation_flownetc_shape_subset():
    """configs[1] geometry (C=256, 48x160, d=20) on one item; oracle runs in seconds."""
    shape = (1, 256, 48, 160)
    a, b = rnd(shape, 21), rnd(shape, 22)
    want = oops.correlation(a, b)
    got = _ops().correlation(a.cuda(), b.cuda())
    close(got, want)


def test_correlation_full_size_properties():
    """BASELINE configs[1] full size (B=8): size-independent properties instead of the oracle."""
    ops = _ops()
    B, C, H, W = 8, 256, 48, 160
    g = torch.Generator(device="cuda").manual_seed(5)
    a = torch.randn(B, C, H, W, device="cuda", generator=g)
    b = torch.randn(B, C, H, W, device="cuda", generator=g)
    out = ops.correlation(a, b)
    assert out.shape == (B, 441, H, W)
    # (1) centre displacement == mean over channels of the product
    torch.testing.assert_close(out[:, 220], (a * b).mean(1), rtol=1e-4, atol=1e-5)
    # (2) symmetry: corr(b,a)[(-p,-o)](y+2p, x+2o) == corr(a,b)[(p,o)](y,x)
    rev = ops.correlation(b, a)
    for (p, o) in [(-10, -10), (3, -7), (10, 10), (0, 5)]:
        tc, tcr = (p + 10) * 21 + (o + 10), (-p + 10) * 21 + (-o + 10)
        ys = slice(max(0, -2 * p), min(H, H - 2 * p))
        xs = slice(max(0, -2 * o), min(W, W - 2 * o))
        ys2 = slice(ys.start + 2 * p, ys.stop + 2 * p)
        xs2 = slice(xs.start + 2 * o, xs.stop + 2 * o)
        torch.testing.assert_close(out[:, tc, ys, xs], rev[:, tcr, ys2, xs2], rtol=1e-4, atol=1e-5)
    # (3) zero padding: displaced row outside the image -> exact zeros
    assert float(out[:, 0, :20, :].abs().max()) == 0.0
    # (4) linearity in the second argument
    out2 = ops.correlation(a, 2.0 * b)
    torch.testing.assert_close(out2, 2.0 * out, rtol=1e-5, atol=1e-6)
    # (5) batch independence
    single = ops.correlation(a[3:4].contiguous(), b[3:4].contiguous())
    assert torch.equal(single[0], out[3])


@pytest.mark.parametrize("shape,md", [((2, 48, 20, 56), 20), ((1, 24, 12, 32), 8), ((4, 256, 48, 160), 20)])
def test_correlation_bidirectional_one_pass(shape, md):
    """Both cost volumes of the bidirectional pass from ONE forward launch (the reverse volume is a
    re-indexing of the forward accumulators, flownet.py:34-44 / SURVEY.md H1b): forward bit-identical to
    two launches, gradients equal to the sum autograd forms from the two separate ops."""
    ops = _ops()
    kw = dict(pad=md, kernel_size=1, max_displacement=md, stride_1=1, stride_2=2)
    a, b = rnd(shape, 41).cuda().requires_grad_(True), rnd(shape, 42).cuda().requires_grad_(True)
    ab, ba = ops.correlation_bidir(a, b, **kw)
    a2, b2 = a.detach().clone().requires_grad_(True), b.detach().clone().requires_grad_(True)
    ab2, ba2 = ops.correlation(a2, b2, **kw), ops.correlation(b2, a2, **kw)
    assert torch.equal(ab, ab2) and torch.equal(ba, ba2)
    gab, gba = rnd(tuple(ab.shape), 43).cuda(), rnd(tuple(ab.shape), 44).cuda()
    (ab * gab).sum().add((ba * gba).sum()).backward()
    (ab2 * gab).sum().add((ba2 * gba).sum()).backward()
    for got, want in ((a.grad, a2.grad), (b.grad, b2.grad)):
        scale = float(want.abs().max())
        assert float((got - want).abs().max()) <= 2e-6 * scale


@pytest.mark.parametrize("B,C,P,pitch,c0", [(2, 5, 37, 12, 3), (3, 441, 48 * 160, 476, 32), (2, 256, 24 * 20, 256, 0)])
def test_relayout_planar_interleaved(B, C, P, pitch, c0):
    """csrc/relayout.cu: the tiled transposes between the correlation op's NCHW tensors and channel slices of
    the NHWC concat buffers -- exact copies, accumulate adds, the slack channels stay untouched."""
    from unflow_b200 import _native
    lib = _native.lib()
    st = torch.cuda.current_stream().cuda_stream
    src = rnd((B, C, P), 7).cuda()
    buf = torch.full((B + 1, P, pitch), -3.5, device="cuda")
    dst = buf[1:]                                       # a batch slice too
    assert lib.unflow_planar_to_interleaved(src.data_ptr(), C * P, dst.data_ptr() + 4 * c0, P * pitch, pitch,
                                            B, C, P, 0, st) == 0
    assert torch.equal(dst[:, :, c0:c0 + C], src.permute(0, 2, 1))
    untouched = torch.ones(pitch, dtype=torch.bool); untouched[c0:c0 + C] = False
    assert bool((dst[:, :, untouched.cuda()] == -3.5).all()) and bool((buf[0] == -3.5).all())
    assert lib.unflow_planar_to_interleaved(src.data_ptr(), C * P, dst.data_ptr() + 4 * c0, P * pitch, pitch,
                                            B, C, P, 1, st) == 0
    assert torch.equal(dst[:, :, c0:c0 + C], 2 * src.permute(0, 2, 1))
    back = torch.empty_like(src)
    assert lib.unflow_interleaved_to_planar(dst.data_ptr() + 4 * c0, P * pitch, pitch, back.data_ptr(), C * P,
                                            B, C, P, st) == 0
    assert torch.equal(back, 2 * src)
    assert lib.unflow_planar_to_interleaved(src.data_ptr(), C * P, dst.data_ptr(), P * pitch, C - 1, B, C, P, 0, st) == 1


def test_flownetc_fused_trunk_input_matches_unfused():
    """concat([conv_redir, corr]) of both directions written into one NHWC buffer (ops.
    _CorrelationBidirConcat) against the unfused correlation_bidir + concat: same flows, same gradients."""
    from unflow_b200.e2eflow.core import flownet as F
    v = F.FlowNetVariables('C', False, seed=3).cuda()
    g = torch.Generator().manual_seed(5)
    im1 = (torch.rand(2, 128, 192, 3, generator=g) - 0.5).cuda()
    im2 = (torch.rand(2, 128, 192, 3, generator=g) - 0.5).cuda()
    res = {}
    try:
        for fused in (True, False):
            F.FUSED_TRUNK_INPUT = fused
            for p in v.parameters():
                p.grad = None
            fw, bw = F.flownet(im1, im2, 'C', backward_flow=True, variables=v)
            loss = sum((f * f).sum() * (i + 1) for i, f in enumerate(fw[0] + bw[0]))
            loss.backward()
            res[fused] = ([f.detach().clone() for f in fw[0] + bw[0]],
                          {k: p.grad.detach().clone() for k, p in v.named_parameters()})
    finally:
        F.FUSED_TRUNK_INPUT = True
    # (not bit-identical: the split-K weight gradients and the channel-split flow heads add with atomics in an
    # order that changes from run to run -- the same tolerance holds between two runs of either variant)
    for a, b in zip(res[True][0], res[False][0]):
        assert float((a - b).abs().max()) <= 2e-5 * float(b.abs().max())
    for k, want in res[False][1].items():
        got = res[True][1][k]
        assert float((got - want).abs().max()) <= 1e-4 * float(want.abs().max()) + 1e-12, k


def test_correlation_bidir_falls_back_for_other_attributes():
    ops = _ops()
    a, b = rnd((1, 8, 10, 14), 1).cuda(), rnd((1, 8, 10, 14), 2).cuda()
    kw = dict(pad=4, kernel_size=3, max_displacement=3, stride_1=2, stride_2=1)      # generic kernel
    ab, ba = ops.correlation_bidir(a, b, **kw)
    assert torch.equal(ab, ops.correlation(a, b, **kw)) and torch.equal(ba, ops.correlation(b, a, **kw))


def test_correlation_errors():
    ops = _ops()
    a = rnd((1, 2, 4, 4), 1).cuda()
    with pytest.raises(ValueError):
        ops.correlation(a, a, kernel_size=2)
    with pytest.raises(ValueError):
        ops.correlation(a, rnd((1, 2, 4, 5), 2).cuda())
    with pytest.raises(ValueError):
        ops.correlation(a, a, max_displacement=8, pad=0)
    with pytest.raises(RuntimeError):
        ops.correlation(a.cpu(), a.cpu())


# ------------------------------------------------------------------ warps
@pytest.mark.parametrize("C", [1, 2, 3, 5])
@pytest.mark.parametrize("scale", [0.7, 4.0])
def test_backward_warp_vs_oracle(C, scale):
    im, fl = rnd((2, 9, 13, C), 1), rnd((2, 9, 13, 2), 2, scale)
    flo = fl.clone().requires_grad_(True)
    flg = fl.cuda().requires_grad_(True)
    want = oops.backward_warp(im, flo)
    got = _ops().backward_warp(im.cuda(), flg)
    close(got, want, atol_rel=1e-6)
    w = rnd(tuple(want.shape), 3)
    (want * w).sum().backward()
    (got * w.cuda()).sum().backward()
    close(flg.grad, flo.grad, atol_rel=1e-5)


@pytest.mark.parametrize("C", [1, 2, 3, 5])
@pytest.mark.parametrize("scale", [0.7, 4.0])
def test_image_warp_vs_oracle(C, scale):
    from unflow_b200.e2eflow.core.image_warp import image_warp
    im, fl = rnd((2, 9, 13, C), 4), rnd((2, 9, 13, 2), 5, scale)
    imo, flo = im.clone().requires_grad_(True), fl.clone().requires_grad_(True)
    img, flg = im.cuda().requires_grad_(True), fl.cuda().requires_grad_(True)
    want = oimage_warp(imo, flo)
    got = image_warp(img, flg)
    close(got, want, atol_rel=1e-6)
    w = rnd(tuple(want.shape), 6)
    (want * w).sum().backward()
    (got * w.cuda()).sum().backward()
    close(flg.grad, flo.grad, atol_rel=1e-5)
    close(img.grad, imo.grad, atol_rel=1e-5)


def test_warp_empty_and_errors():
    ops = _ops()
    e = ops.backward_warp(torch.zeros(0, 4, 4, 3, device="cuda"), torch.zeros(0, 4, 4, 2, device="cuda"))
    assert e.shape == (0, 4, 4, 3)
    with pytest.raises(ValueError):
        ops.backward_warp(torch.zeros(1, 4, 4, 3, device="cuda"), torch.zeros(1, 4, 5, 2, device="cuda"))


def test_forward_warp_vs_oracle():
    for scale, shape in ((1.5, (2, 17, 23)), (9.0, (1, 40, 70)), (40.0, (1, 12, 12))):
        fl = rnd(shape + (2,), 7, scale)
        flo = fl.clone().requires_grad_(True)
        flg = fl.cuda().requires_grad_(True)
        want = oops.forward_warp(flo)
        got = _ops().forward_warp(flg)
        close(got, want, rtol=1e-5, atol_rel=1e-6)
        w = rnd(tuple(want.shape), 8)
        (want * w).sum().backward()
        (got * w.cuda()).sum().backward()
        close(flg.grad, flo.grad, rtol=1e-4, atol_rel=1e-5)


def test_forward_warp_disocclusion_mask_exact_outside_ties():
    """The binary disocclusion mask (forward_warp < 0.8, losses.py:28-29) must match the oracle
    except inside a tie band around the threshold (atomic summation order, SURVEY.md H4/H5)."""
    fl = rnd((2, 48, 64, 2), 9, 3.0)
    want = oops.forward_warp(fl)
    got = _ops().forward_warp(fl.cuda()).cpu()
    band = (want - 0.8).abs() < 1e-4
    assert torch.equal((got < 0.8)[~band], (want < 0.8)[~band])
    assert band.float().mean() < 0.01


@pytest.mark.parametrize("shape,scale", [((2, 8, 12, 3), 2), ((2, 8, 12, 3), 4), ((1, 384, 1280, 1), 4),
                                         ((3, 6, 10, 5), 1)])
def test_downsample_vs_oracle(shape, scale):
    im = rnd(shape, 3)
    close(_ops().downsample(im.cuda(), scale), oops.downsample(im, scale), rtol=1e-6, atol_rel=1e-7)


def test_downsample_errors():
    with pytest.raises(ValueError):
        _ops().downsample(torch.zeros(1, 6, 9, 1, device="cuda"), 2)


def test_native_library_is_loaded_and_counts_launches():
    from unflow_b200 import _native
    _native.reset_launch_count()
    _ops().downsample(torch.zeros(1, 4, 4, 1, device="cuda"), 2)
    assert _native.launch_count() == 1
