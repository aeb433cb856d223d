"""unflow_tc_conv on contractions over at most 4 channels, which it runs on the FMA pipes (csrc/conv_fma.cu), against
float64: both modes and strides, 1 to 4 input channels, kernels up to 8x8 (64 taps), output channel counts with every
tail mod 4, odd extents, channel-sliced inputs and outputs, every epilogue, and the launches of a FlowNetC training
step at 384x1280 (both directions of a batch of 4: 8 images).

The bound is elementwise and exact-fp32: a sequential FMA chain of n = taps x Cin products, then the bias, the
activation and the add of the old value, is off by at most (n + 2) 2^-24 A, where A is the same computation on the
absolute values of every operand."""
import pytest
import torch

from test_gpu_tc_conv import pitched
from test_gpu_tc_step_launches import planes_f64, ref_conv

pytestmark = pytest.mark.gpu

CANARY = -3.5


def T():
    from unflow_b200.e2eflow.core import tc_conv
    return tc_conv


def sliced(N, C, H, W, off, pitch, seed):
    """NCHW-shaped view of channels [off, off + C) of an NHWC buffer of `pitch` floats per pixel; the other
    channels hold NaN, which must never reach a result."""
    g = torch.Generator().manual_seed(seed)
    buf = torch.full((N, H, W, pitch), float("nan"), device="cuda")
    v = buf[..., off:off + C].permute(0, 3, 1, 2)
    v.copy_(torch.randn(N, C, H, W, generator=g).cuda())
    return v


def setup(mode, N, Cin, Cout, Hin, Win, k, stride, pad, *, bias, act, accum, x_off=0, y_off=0, seed=0):
    """Operands of one call: returns (launch(), out view, out buffer, ref, bound)."""
    t = T()
    if mode == 0:
        Hout, Wout = -(-Hin // stride), -(-Win // stride)
    else:
        Hout, Wout = stride * Hin, stride * Win
    x = sliced(N, Cin, Hin, Win, x_off, t.round4(x_off + Cin), seed)
    g = torch.Generator().manual_seed(seed + 1)
    shape = (Cout, Cin, k, k) if mode == 0 else (Cin, Cout, k, k)
    w = (torch.randn(*shape, generator=g) / (Cin * k * k) ** 0.5).cuda().contiguous(memory_format=torch.channels_last)
    planes = t.split_weights(w, transpose=mode == 1)
    b = (torch.randn(Cout + 1, generator=g) * 0.1).cuda()[1:] if bias else None       # 4-byte aligned only
    out, obuf = pitched(N, Cout, Hout, Wout, t.round4(y_off + Cout) + 4, seed=seed + 2, fill=CANARY)
    if y_off:                                        # the slice starts at channel y_off; canaries on both sides
        obuf.fill_(CANARY)
        out = obuf[..., y_off:y_off + Cout].permute(0, 3, 1, 2)
        out.copy_(torch.randn(N, Cout, Hout, Wout, generator=g).cuda())
    start = obuf.clone()

    x64, wt = x.double(), planes_f64(planes)
    ref = ref_conv(x64, wt, mode, stride, k, k, pad, pad, Hout, Wout)
    A = ref_conv(x64.abs(), wt.abs(), mode, stride, k, k, pad, pad, Hout, Wout)
    if bias:
        ref = ref + b.double().view(1, -1, 1, 1)
        A = A + b.double().abs().view(1, -1, 1, 1)
    if act:
        ref = torch.nn.functional.leaky_relu(ref, 0.1)
    if accum:
        ref = ref + out.double()
        A = A + out.double().abs()
    bound = (k * k * Cin + 2) * 2.0 ** -24 * A

    def launch():
        obuf.copy_(start)
        if not accum:
            out.fill_(float("nan"))
        t.run(x, planes, out, mode=mode, stride=stride, kh=k, kw=k, pad_t=pad, pad_l=pad, bias=b, act=act,
              accumulate=accum)
    return launch, out, obuf, start, (y_off, Cout), ref, bound


def check(out, obuf, start, cols, ref, bound):
    y_off, Cout = cols
    err = (out.double() - ref).abs()
    worst = float((err - bound).max())
    assert worst <= 0, "error exceeds (n + 2) 2^-24 A by %g" % worst
    keep = torch.ones(obuf.shape[-1], dtype=torch.bool, device="cuda")
    keep[y_off:y_off + Cout] = False
    assert torch.equal(obuf[..., keep], start[..., keep]), "a channel outside the output slice was written"


CASES = {  # mode, N, Cin, Cout, Hin, Win, k, stride, pad, x channel offset, y channel offset
    "conv_1x1_cin1_cout1": (0, 1, 1, 1, 7, 9, 1, 1, 0, 0, 0),
    "conv_3x3_cin2_cout5": (0, 3, 2, 5, 13, 11, 3, 1, 1, 4, 0),
    "conv_4x4_s2_cin3_cout3": (0, 2, 3, 3, 15, 21, 4, 2, 1, 0, 4),
    "conv_7x7_s2_cin4_cout194": (0, 2, 4, 194, 11, 17, 7, 2, 3, 8, 0),
    "conv_8x8_cin2_cout2": (0, 5, 2, 2, 9, 13, 8, 1, 3, 0, 0),
    "conv_8x8_s2_cin1_cout386": (0, 1, 1, 386, 10, 14, 8, 2, 3, 4, 4),
    "deconv_3x3_cin2_cout386": (1, 8, 2, 386, 7, 9, 3, 1, 1, 0, 4),
    "deconv_4x4_s2_cin2_cout2": (1, 4, 2, 2, 9, 11, 4, 2, 1, 4, 0),
    "deconv_3x3_s2_cin1_cout1026": (1, 2, 1, 1026, 5, 7, 3, 2, 1, 0, 0),
    "deconv_8x8_s2_cin4_cout5": (1, 3, 4, 5, 6, 9, 8, 2, 3, 4, 0),
    "deconv_7x7_cin3_cout3": (1, 6, 3, 3, 11, 5, 7, 1, 3, 0, 4),
    "deconv_1x1_cin4_cout1": (1, 7, 4, 1, 3, 5, 1, 1, 0, 0, 0),
}
EPILOGUES = {"plain": (False, False, False), "bias_act": (True, True, False), "accum": (False, False, True),
             "bias_act_accum": (True, True, True), "bias": (True, False, False)}


@pytest.mark.parametrize("epi", sorted(EPILOGUES))
@pytest.mark.parametrize("case", sorted(CASES))
def test_few_channel_conv_against_float64(case, epi):
    mode, N, Cin, Cout, H, W, k, stride, pad, x_off, y_off = CASES[case]
    bias, act, accum = EPILOGUES[epi]
    launch, out, obuf, start, cols, ref, bound = setup(mode, N, Cin, Cout, H, W, k, stride, pad, bias=bias, act=act,
                                                       accum=accum, x_off=x_off, y_off=y_off, seed=Cin * 7 + Cout)
    launch()
    check(out, obuf, start, cols, ref, bound)


def test_repeats_and_graph_replay_are_bit_identical():
    launch, out, obuf, start, cols, ref, bound = setup(1, 4, 2, 194, 24, 40, 3, 1, 1, bias=True, act=True,
                                                       accum=True, y_off=4, seed=5)
    launch()
    first = obuf.clone()
    launch()
    assert torch.equal(obuf, first)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        launch()                                     # warm-up outside the capture
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            launch()
    torch.cuda.current_stream().wait_stream(s)
    obuf.fill_(0.0)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(obuf, first)
    check(out, obuf, start, cols, ref, bound)


# The 13 launches of a FlowNetC training step at 384x1280 (8 images): the flow heads' input gradients (2 -> the
# concat's channels, the first head writes, the others add to what the decoder's deconvs left) and the up-sampling
# deconvs flowN_up, forward (bias, no activation) and input gradient (added to the flow's gradient).
STEP = {  # mode, Cout, Hin, Win, k, stride, pad, bias, accumulate
    "flow2_dx": (1, 194, 96, 320, 3, 1, 1, False, False),
    "flow3_dx": (1, 386, 48, 160, 3, 1, 1, False, True),
    "flow4_dx": (1, 770, 24, 80, 3, 1, 1, False, True),
    "flow5_dx": (1, 1026, 12, 40, 3, 1, 1, False, True),
    "flow6_dx": (1, 1024, 6, 20, 3, 1, 1, False, True),
    "flow6_up5": (1, 2, 6, 20, 4, 2, 1, True, False),
    "flow5_up4": (1, 2, 12, 40, 4, 2, 1, True, False),
    "flow4_up3": (1, 2, 24, 80, 4, 2, 1, True, False),
    "flow3_up2": (1, 2, 48, 160, 4, 2, 1, True, False),
    "flow6_up5_dx": (0, 2, 12, 40, 4, 2, 1, False, True),
    "flow5_up4_dx": (0, 2, 24, 80, 4, 2, 1, False, True),
    "flow4_up3_dx": (0, 2, 48, 160, 4, 2, 1, False, True),
    "flow3_up2_dx": (0, 2, 96, 320, 4, 2, 1, False, True),
}


@pytest.mark.parametrize("layer", sorted(STEP))
def test_step_launches_at_bench_geometry(layer):
    mode, Cout, H, W, k, stride, pad, bias, accum = STEP[layer]
    launch, out, obuf, start, cols, ref, bound = setup(mode, 8, 2, Cout, H, W, k, stride, pad, bias=bias, act=False,
                                                       accum=accum, y_off=4 if Cout == 2 else 0, seed=Cout)
    launch()
    check(out, obuf, start, cols, ref, bound)
