"""The stream-K tails of tc_conv_kernel (csrc/tc_schedule.h, csrc/tc_conv.cu: sk_fixup) against float64.

Launches whose last work items are cut into K ranges that several CTAs run: the warp that finishes a tile last adds
the other CTAs' partial sums and runs the epilogue.  Each case checks one launch of the C ABI against float64 (the
tolerance of test_gpu_tc_conv.py), that two launches are bit-identical (the partial sums are added in a fixed
order), and that the fixup counters are back at zero after eager launches and after CUDA graph replays."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from float64_refs import view

pytestmark = pytest.mark.gpu

TOL = 5e-6
SMS = 132


def T():
    from unflow_b200.e2eflow.core import tc_conv
    return tc_conv


def lib():
    from unflow_b200 import _native
    return _native.lib()


def plan(N, Hin, Win, Cin, Hout, Wout, Cout, mode, stride, k, pad_t, pad_l):
    buf = (ctypes.c_int * 1024)()
    n = lib().unflow_tc_conv_plan(N, Hin, Win, Cin, Hout, Wout, Cout, mode | 4, stride, k, k, pad_t, pad_l, buf, 1024)
    assert n > 0, n
    nt = buf[14]
    cs = list(buf[15:15 + buf[0] + 1])
    items = buf[0] * buf[8] * buf[9] * buf[10] * buf[11]
    return dict(items=items, taps=[cs[c + 1] - cs[c] for c in range(buf[0])], kblocks=buf[13],
                pair_px=buf[28 + 3 * nt])


def nhwc(N, C, H, W, pitch, seed):
    g = torch.Generator().manual_seed(seed)
    buf = torch.zeros((N, H, W, pitch), device="cuda")
    v = buf[..., :C].permute(0, 3, 1, 2)
    v.copy_(torch.randn(N, C, H, W, generator=g).cuda())
    return v


# mode, N, Cin, Cout, H, W, k, stride, pad, bias + act, accumulate; the output pitch is Cout + 4, so no launch is
# cut into K slices (they add their parts with red.add and need no fixup)
CASES = {
    # 6 tiles of 72 K blocks over 132 CTAs: every tile split into 9 chunk-long segments, most CTAs idle
    "bias_act_few_tiles": (0, 2, 256, 128, 16, 24, 3, 1, 1, True, False),
    # 300 tiles: one DP wave, 168 tiles in the stream-K tail
    "bias_act_dp_and_sk": (0, 8, 256, 96, 48, 100, 3, 1, 1, True, False),
    "accumulate": (0, 4, 320, 128, 16, 24, 3, 1, 1, True, True),
    # k4 s2 transposed, 64 channels: two parity classes per tile
    "pair_px": (1, 4, 256, 64, 12, 40, 4, 2, 1, True, False),
    # 5x5 s2 transposed, 96 channels: four classes with 9 / 6 / 6 / 4 taps
    "unequal_classes": (1, 4, 256, 96, 12, 40, 5, 2, 2, True, False),
}


def setup(case):
    t = T()
    mode, N, Cin, Cout, H, W, k, stride, pad, ba, accum = CASES[case]
    x = nhwc(N, Cin, H, W, t.round4(Cin), seed=Cin + k)
    g = torch.Generator().manual_seed(Cout + k)
    if mode == 0:
        w = (torch.randn(Cout, Cin, k, k, generator=g) * (2.0 / (Cin * k * k)) ** 0.5).cuda()
        ref = F.conv2d(F.pad(x.double(), (pad, pad, pad, pad)), w.double(), stride=stride)
        Hout, Wout = ref.shape[2:]
        planes = t.split_weights(w.contiguous(memory_format=torch.channels_last))
        p = plan(N, H, W, Cin, Hout, Wout, Cout, 0, stride, k, pad, pad)
    else:
        w = (torch.randn(Cin, Cout, k, k, generator=g) * (2.0 / (Cin * k * k)) ** 0.5).cuda()
        Hout, Wout = stride * H, stride * W
        ref = F.conv_transpose2d(x.double(), w.double(), stride=stride, padding=pad,
                                 output_padding=(Hout - ((H - 1) * stride - 2 * pad + k), Wout - ((W - 1) * stride - 2 * pad + k)))
        planes = t.split_weights(w.contiguous(memory_format=torch.channels_last), transpose=True)
        p = plan(N, H, W, Cin, Hout, Wout, Cout, 1, stride, k, pad, pad)
    b = (torch.randn(Cout, generator=g) * 0.1).cuda() if ba else None
    if ba:
        ref = F.leaky_relu(ref + b.double().view(1, -1, 1, 1), 0.1)
    out = nhwc(N, Cout, Hout, Wout, t.round4(Cout) + 4, seed=3)
    start = out.clone()
    if accum:
        ref = ref + start.double()

    def launch():
        out.copy_(start)
        t.run(x, planes, out, mode=mode, stride=stride, kh=k, kw=k, pad_t=pad, pad_l=pad, bias=b, act=ba,
              accumulate=accum)
    return launch, out, ref, p


def counters():
    """The fixup counters of the current device, through the role-timer hook (which also reports them)."""
    dbg = torch.zeros(16, dtype=torch.int64, device="cuda")
    x = torch.zeros((1, 32, 1, 8), device="cuda").contiguous(memory_format=torch.channels_last)
    y = torch.empty_like(x)
    t = T()
    lib().unflow_tc_conv_debug(dbg.data_ptr())
    try:
        t.run(x, t.split_weights(torch.zeros(32, 32, 1, 1, device="cuda").contiguous(memory_format=torch.channels_last)),
              y, mode=0, stride=1, kh=1, kw=1, pad_t=0, pad_l=0)
    finally:
        lib().unflow_tc_conv_debug(None)
    torch.cuda.synchronize()
    ptr, n = int(dbg[8]), int(dbg[9])
    assert ptr and n > 0
    return view(ptr, (n,)).clone()


@pytest.mark.parametrize("case", sorted(CASES))
def test_stream_k_tail_against_float64(case):
    launch, out, ref, p = setup(case)
    tail = p["items"] % SMS
    assert p["items"] < SMS or tail, "the case must leave a stream-K tail"
    if case == "pair_px":
        assert p["pair_px"] == 1
    if case == "unequal_classes":
        assert p["taps"] == [9, 6, 6, 4] and p["pair_px"] == 0
    launch()
    first = out.clone()
    err = float((first.double() - ref).abs().max() / ref.abs().max())
    assert err < TOL, err
    launch()
    assert torch.equal(out, first), "two launches differ"
    assert bool((counters() == 0).all())


def test_counters_zero_after_graph_replays():
    launch, out, ref, _ = setup("bias_act_few_tiles")
    launch()
    eager = out.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=side):
            for _ in range(3):
                launch()
        for _ in range(4):
            g.replay()
            side.synchronize()
            assert torch.equal(out, eager)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    del g
    assert bool((counters() == 0).all())
