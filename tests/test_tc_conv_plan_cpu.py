"""Host logic of csrc/tc_conv.cu on the CPU: the tap / output-class / tile plan the launcher builds
(unflow_tc_conv_plan) is executed here with plain tensor ops -- exactly the sum the kernel's
producer / MMA / epilogue roles implement, including the tile boxes and their masking -- and must
reproduce torch's conv2d / conv_transpose2d (the layers of reference flownet.py:166-233, :89-155 with
TF SAME padding, and their input gradients).  No GPU, no kernel launch."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from unflow_b200 import _native


def plan(N, Hin, Win, Cin, Hout, Wout, Cout, mode, stride, kh, kw, pt, pl):
    buf = (ctypes.c_int * 640)()
    n = _native.lib().unflow_tc_conv_plan(N, Hin, Win, Cin, Hout, Wout, Cout, mode, stride, kh, kw, pt, pl, buf, 640)
    assert n > 0, n
    v = list(buf[:n])
    keys = ["n_classes", "s_in", "s_out", "Hit", "Wit", "TW", "TH", "TN", "tiles_x", "tiles_y", "tiles_n",
            "n_blocks", "BN", "kblocks", "ntaps"]
    p = dict(zip(keys, v[:15]))
    p["class_start"] = v[15:20]
    p["class_pxy"] = [(v[20 + 2 * i], v[21 + 2 * i]) for i in range(4)]
    p["taps"] = [tuple(v[28 + 3 * i: 31 + 3 * i]) for i in range(p["ntaps"])]
    tail = v[28 + 3 * p["ntaps"]:]
    p["pair_px"] = tail[0]
    p["widx2"] = tail[1:1 + p["ntaps"]]
    p["ksplit"] = tail[1 + p["ntaps"]]
    assert len(tail) == 2 + p["ntaps"]
    return p


def execute(p, x, w_taps, N, Hout, Wout, Cout):
    """x [N,Hin,Win,Cin] (NHWC), w_taps [taps][Cout][Cin]; tile by tile like the kernel."""
    _, Hin, Win, Cin = x.shape
    out = torch.full((N, Hout, Wout, Cout), float("nan"), dtype=x.dtype)
    written = torch.zeros((N, Hout, Wout), dtype=torch.int32)
    TW, TH, TN = p["TW"], p["TH"], p["TN"]
    assert TW * TH * TN <= 128
    for cls in range(p["n_classes"]):
        px, py = p["class_pxy"][cls]
        taps = p["taps"][p["class_start"][cls]:p["class_start"][cls + 1]]
        for tn in range(p["tiles_n"]):
            for ty in range(p["tiles_y"]):
                for tx in range(p["tiles_x"]):
                    n0, iy0, ix0 = tn * TN, ty * TH, tx * TW
                    acc = torch.zeros((TN, TH, TW, Cout), dtype=x.dtype)
                    for (dx, dy, widx) in taps:
                        # the TMA box: element stride s_in, zero fill outside the tensor
                        box = torch.zeros((TN, TH, TW, Cin), dtype=x.dtype)
                        for a in range(TN):
                            for b in range(TH):
                                for c in range(TW):
                                    n, yy, xx = n0 + a, p["s_in"] * (iy0 + b) + dy, p["s_in"] * (ix0 + c) + dx
                                    if n < N and 0 <= yy < Hin and 0 <= xx < Win:
                                        box[a, b, c] = x[n, yy, xx]
                        acc += box @ w_taps[widx].t()
                    for a in range(TN):
                        for b in range(TH):
                            for c in range(TW):
                                n, iy, ix = n0 + a, iy0 + b, ix0 + c
                                if n < N and iy < p["Hit"] and ix < p["Wit"]:
                                    oy, ox = p["s_out"] * iy + py, p["s_out"] * ix + px
                                    out[n, oy, ox] = acc[a, b, c]
                                    written[n, oy, ox] += 1
    assert int(written.min()) == 1 and int(written.max()) == 1     # every output exactly once
    return out


CONV = [(2, 5, 9, 11, 7, 3, 1, (1, 1, 1, 1)), (1, 4, 6, 10, 12, 1, 1, (0, 0, 0, 0)),
        (2, 3, 8, 12, 5, 3, 2, (0, 1, 0, 1)), (1, 3, 8, 12, 4, 5, 2, (1, 2, 1, 2)),
        (1, 2, 12, 16, 3, 7, 2, (2, 3, 2, 3)), (3, 2, 6, 20, 70, 3, 1, (1, 1, 1, 1))]


@pytest.mark.parametrize("N,Cin,H,W,Cout,k,stride,pads", CONV)
def test_conv_plan(N, Cin, H, W, Cout, k, stride, pads):
    pt, pb, pl, pr = pads
    g = torch.Generator().manual_seed(k * 7 + Cin)
    x = torch.randn(N, Cin, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(Cout, Cin, k, k, generator=g, dtype=torch.float64)
    ref = F.conv2d(F.pad(x, (pl, pr, pt, pb)), w, stride=stride)
    Ho, Wo = ref.shape[2], ref.shape[3]
    p = plan(N, H, W, Cin, Ho, Wo, Cout, 0, stride, k, k, pt, pl)
    assert p["n_classes"] == 1 and p["ntaps"] == k * k and p["BN"] in (32, 64, 128)
    assert p["n_blocks"] * p["BN"] >= Cout > (p["n_blocks"] - 1) * p["BN"]
    w_taps = w.permute(2, 3, 0, 1).reshape(k * k, Cout, Cin)
    got = execute(p, x.permute(0, 2, 3, 1), w_taps, N, Ho, Wo, Cout)
    torch.testing.assert_close(got.permute(0, 3, 1, 2), ref, rtol=1e-12, atol=1e-12)


DECONV = [(2, 5, 3, 5, 7, 4, 2, 1, None), (1, 6, 4, 6, 3, 3, 2, 0, (8, 12)), (1, 4, 4, 6, 3, 5, 2, 1, (8, 12)),
          (1, 4, 6, 8, 3, 7, 2, 2, (12, 16)), (2, 4, 5, 7, 6, 3, 1, 1, None), (1, 3, 5, 7, 2, 1, 1, 0, None)]


@pytest.mark.parametrize("N,Cin,H,W,Cout,k,stride,pad,out_hw", DECONV)
def test_transposed_plan(N, Cin, H, W, Cout, k, stride, pad, out_hw):
    """deconvN forward (k4 s2 p1) and the input gradients of the stride-2 / stride-1 convolutions (the
    cropped transposed convolution: TF SAME's bottom / right padding rows are never produced)."""
    g = torch.Generator().manual_seed(k * 5 + Cout)
    x = torch.randn(N, Cin, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(Cin, Cout, k, k, generator=g, dtype=torch.float64)
    Ho, Wo = (H - 1) * stride - 2 * pad + k, (W - 1) * stride - 2 * pad + k
    oph = opw = 0
    if out_hw:
        oph, opw = out_hw[0] - Ho, out_hw[1] - Wo
        Ho, Wo = out_hw
    ref = F.conv_transpose2d(x, w, stride=stride, padding=pad, output_padding=(max(oph, 0), max(opw, 0)))[:, :, :Ho, :Wo]
    if Ho % stride or Wo % stride:
        assert _native.lib().unflow_tc_conv_plan(N, H, W, Cin, Ho, Wo, Cout, 1, stride, k, k, pad, pad, None, 0) == -1
        return
    p = plan(N, H, W, Cin, Ho, Wo, Cout, 1, stride, k, k, pad, pad)
    assert p["n_classes"] == stride * stride and p["ntaps"] == k * k
    w_taps = w.permute(2, 3, 1, 0).reshape(k * k, Cout, Cin)
    got = execute(p, x.permute(0, 2, 3, 1), w_taps, N, Ho, Wo, Cout)
    torch.testing.assert_close(got.permute(0, 3, 1, 2), ref, rtol=1e-12, atol=1e-12)


def test_plan_tiles_of_the_flownet_shapes():
    """Tile boxes at the FlowNetC geometry (2B = 8 samples): utilisation of the 128 MMA rows."""
    for (H, W, want) in [(48, 160, 1.0), (24, 80, 1.0), (12, 40, 0.93), (6, 20, 0.93)]:
        p = plan(8, H, W, 64, H, W, 64, 0, 1, 3, 3, 1, 1)
        tiles = p["tiles_x"] * p["tiles_y"] * p["tiles_n"]
        util = 8 * H * W / (tiles * 128.0)
        assert util >= want - 1e-9, (H, W, p["TW"], p["TH"], p["TN"], util)


def test_k_slices_of_the_flownet_shapes():
    """The K-slice decision at the FlowNetC geometry (2B = 8 samples): conv6_1 (1024 -> 1024 channels, 3x3 at
    6x20) has 8 tiles x 8 column blocks = 64 work items for 132 SMs and 288 K blocks per tile, so each tile is cut
    into two slices; conv3 (128 -> 256 channels, 5x5 stride 2 at 48x160) fills the GPU with tiles alone.
    tc_ksplit = 0 switches slicing off."""
    lib = _native.lib()
    conv6_1 = (8, 6, 20, 1024, 6, 20, 1024, 0, 1, 3, 3, 1, 1)
    conv3 = (8, 96, 320, 128, 48, 160, 256, 0, 2, 5, 5, 1, 1)
    assert plan(*conv6_1)["ksplit"] == 2
    assert plan(*conv3)["ksplit"] == 1
    try:
        assert lib.unflow_set_int_option(b"tc_ksplit", 0) == 0
        assert plan(*conv6_1)["ksplit"] == 1
    finally:
        lib.unflow_set_int_option(b"tc_ksplit", 1)


def test_tensor_core_options_reject_values_out_of_range():
    """unflow_set_int_option accepts tc_chunk 1..64 and tc_pair_px / tc_ksplit 0 / 1; anything else is
    UNFLOW_EINVAL and leaves the setting alone (the plan of conv6_1 keeps its two K slices)."""
    lib = _native.lib()
    for name, bad in ((b"tc_chunk", 0), (b"tc_chunk", 65), (b"tc_chunk", -1), (b"tc_pair_px", 2),
                      (b"tc_pair_px", -1), (b"tc_ksplit", 2), (b"tc_ksplit", -1)):
        assert lib.unflow_set_int_option(name, bad) == _native.UNFLOW_EINVAL, (name, bad)
        assert name.decode() in _native.last_error()
    assert plan(8, 6, 20, 1024, 6, 20, 1024, 0, 1, 3, 3, 1, 1)["ksplit"] == 2
    for name, good, default in ((b"tc_chunk", 1, 8), (b"tc_chunk", 64, 8), (b"tc_pair_px", 0, 1), (b"tc_ksplit", 0, 1)):
        assert lib.unflow_set_int_option(name, good) == _native.UNFLOW_OK
        assert lib.unflow_set_int_option(name, default) == _native.UNFLOW_OK


def test_plan_rejects_bad_arguments():
    lib = _native.lib()
    assert lib.unflow_tc_conv_plan(1, 8, 8, 4, 8, 8, 4, 0, 3, 3, 3, 1, 1, None, 0) == -1      # stride 3
    assert lib.unflow_tc_conv_plan(1, 8, 8, 4, 8, 8, 4, 2, 1, 3, 3, 1, 1, None, 0) == -1      # mode 2
    assert lib.unflow_tc_conv_plan(1, 8, 8, 4, 8, 8, 4, 0, 1, 9, 9, 4, 4, None, 0) == -1      # 81 taps
    assert lib.unflow_tc_conv_plan(1, 8, 8, 4, 8, 8, 4, 0, 1, 3, 3, 1, 1, None, 0) < -1       # needs a buffer


# ---------------------------------------------------------------------------------------------
# weight gradient (csrc/tc_wgrad.cu): the K-block pixel boxes / split-K plan executed on the CPU
# ---------------------------------------------------------------------------------------------
def wgrad_plan(N, Hp, Wp, R, C, stride, kh, kw, pt, pl):
    buf = (ctypes.c_int * 15)()
    assert _native.lib().unflow_tc_wgrad_plan(N, Hp, Wp, R, C, stride, kh, kw, pt, pl, buf) == 15
    keys = ["TW", "TH", "TN", "tiles_x", "tiles_y", "tiles_n", "n_ptiles", "kc", "n_chunks", "r_blocks",
            "c_blocks", "BN", "taps", "cgroups", "vgroups"]
    return dict(zip(keys, list(buf)))


def execute_wgrad(p, P, G, stride, kh, kw, pt, pl):
    """P [N,Hp,Wp,R], G [N,Hg,Wg,C] (NHWC) -> dw [R, taps, C], K block by K block, chunk by chunk."""
    N, Hp, Wp, R = P.shape
    _, Hg, Wg, C = G.shape
    assert p["TW"] * p["TH"] * p["TN"] == 32
    assert p["n_ptiles"] == p["tiles_x"] * p["tiles_y"] * p["tiles_n"]
    assert (p["n_chunks"] - 1) * p["kc"] < p["n_ptiles"] <= p["n_chunks"] * p["kc"]
    dw = torch.zeros(R, kh * kw, C, dtype=P.dtype)
    assert p["cgroups"] == -(-C // 32) and p["vgroups"] == kh * kw * p["cgroups"]
    gpb = p["BN"] // 32                                  # (tap, 32-channel group) pairs per column block
    assert p["c_blocks"] == -(-p["vgroups"] // gpb) and p["r_blocks"] == -(-R // 128)
    for chunk in range(p["n_chunks"]):
        for cb in range(p["c_blocks"]):
            groups = []
            for j in range(gpb):
                v = cb * gpb + j
                if v < p["vgroups"]:
                    tap, cg = divmod(v, p["cgroups"])
                    groups.append((tap, cg))
            parts = {g_: torch.zeros(R, 32, dtype=P.dtype) for g_ in groups}
            for kb in range(chunk * p["kc"], min((chunk + 1) * p["kc"], p["n_ptiles"])):
                q = kb
                px = (q % p["tiles_x"]) * p["TW"]; q //= p["tiles_x"]
                py = (q % p["tiles_y"]) * p["TH"]; q //= p["tiles_y"]
                pn = q * p["TN"]
                pb = torch.zeros(32, R, dtype=P.dtype)
                gbs = {g_: torch.zeros(32, 32, dtype=P.dtype) for g_ in groups}
                i = 0
                for a in range(p["TN"]):
                    for b in range(p["TH"]):
                        for c in range(p["TW"]):
                            n, y, x = pn + a, py + b, px + c
                            if n < N and y < Hp and x < Wp:
                                pb[i] = P[n, y, x]
                            for (tap, cg) in groups:
                                ky, kx = divmod(tap, kw)
                                gy, gx = stride * y + ky - pt, stride * x + kx - pl
                                if n < N and 0 <= gy < Hg and 0 <= gx < Wg:
                                    ch = G[n, gy, gx, cg * 32:cg * 32 + 32]
                                    gbs[(tap, cg)][i, :ch.numel()] = ch
                            i += 1
                for g_ in groups:
                    parts[g_] += pb.t() @ gbs[g_]
            for (tap, cg) in groups:
                w_ = min(32, C - cg * 32)
                dw[:, tap, cg * 32:cg * 32 + w_] += parts[(tap, cg)][:, :w_]
    return dw


@pytest.mark.parametrize("N,Cin,H,W,Cout,k,stride,pads", CONV)
def test_wgrad_plan_conv(N, Cin, H, W, Cout, k, stride, pads):
    pt, pb, pl, pr = pads
    g = torch.Generator().manual_seed(k * 11 + Cin)
    x = torch.randn(N, Cin, H, W, generator=g, dtype=torch.float64)
    xp = F.pad(x, (pl, pr, pt, pb))
    Ho, Wo = (xp.shape[2] - k) // stride + 1, (xp.shape[3] - k) // stride + 1
    gy = torch.randn(N, Cout, Ho, Wo, generator=g, dtype=torch.float64)
    ref = torch.nn.grad.conv2d_weight(xp, (Cout, Cin, k, k), gy, stride=stride)      # [Cout, Cin, k, k]
    p = wgrad_plan(N, Ho, Wo, Cout, Cin, stride, k, k, pt, pl)
    got = execute_wgrad(p, gy.permute(0, 2, 3, 1), x.permute(0, 2, 3, 1), stride, k, k, pt, pl)
    torch.testing.assert_close(got.reshape(Cout, k, k, Cin).permute(0, 3, 1, 2), ref, rtol=1e-11, atol=1e-11)


def test_wgrad_plan_deconv():
    """slim.conv2d_transpose(k=4, s=2, SAME): dW[ci, co, ky, kx] = sum_p x[p, ci] * gy[2p - 1 + k, co]."""
    N, Ci, Co, H, W = 2, 5, 6, 4, 6
    g = torch.Generator().manual_seed(4)
    x = torch.randn(N, Ci, H, W, generator=g, dtype=torch.float64, requires_grad=True)
    w = torch.randn(Ci, Co, 4, 4, generator=g, dtype=torch.float64, requires_grad=True)
    gy = torch.randn(N, Co, 2 * H, 2 * W, generator=g, dtype=torch.float64)
    F.conv_transpose2d(x, w, stride=2, padding=1).backward(gy)
    p = wgrad_plan(N, H, W, Ci, Co, 2, 4, 4, 1, 1)
    got = execute_wgrad(p, x.detach().permute(0, 2, 3, 1), gy.permute(0, 2, 3, 1), 2, 4, 4, 1, 1)
    torch.testing.assert_close(got.reshape(Ci, 4, 4, Co).permute(0, 3, 1, 2), w.grad, rtol=1e-11, atol=1e-11)


def test_wgrad_split_k_fills_the_gpu():
    """conv3_1 at the benchmark geometry: 9 taps x 2 x 4 blocks = 72 tiles -> K is split so that the grid
    has several waves of work items, each with at least 8 K blocks."""
    p = wgrad_plan(8, 48, 160, 256, 473, 1, 3, 3, 1, 1)
    items = p["n_chunks"] * p["r_blocks"] * p["c_blocks"]
    assert p["BN"] == 128 and p["r_blocks"] == 2 and p["cgroups"] == 15 and p["c_blocks"] == 34 and p["n_ptiles"] == 1920
    assert items >= 4 * 148 and p["kc"] >= 8
    # conv2 (64 input channels, 25 taps): two taps share one 128-wide block instead of half-empty MMAs
    p = wgrad_plan(8, 96, 320, 128, 64, 2, 5, 5, 1, 1)
    assert p["BN"] == 128 and p["cgroups"] == 2 and p["c_blocks"] == 13


def execute_pair_px(p, x, w_taps, N, Hout, Wout, Cout):
    """The two-parity-classes-per-tile form (csrc/tc_conv.cu, pair_px_plan): a class = an output ROW parity, a
    tile computes 2 * Cout virtual columns -- [0, Cout) the channels of px = 0 with tap widx, [Cout, 2 Cout) those
    of px = 1 with tap widx2; -1 = that class has no tap for the input offset (zero weights)."""
    _, Hin, Win, Cin = x.shape
    out = torch.full((N, Hout, Wout, Cout), float("nan"), dtype=x.dtype)
    written = torch.zeros((N, Hout, Wout), dtype=torch.int32)
    TW, TH, TN = p["TW"], p["TH"], p["TN"]
    assert p["pair_px"] == 1 and p["n_classes"] == 2 and p["n_blocks"] == 1 and p["BN"] == 128 and p["s_out"] == 2
    for cls in range(2):
        py = p["class_pxy"][cls][1]
        lo, hi = p["class_start"][cls], p["class_start"][cls + 1]
        for tn in range(p["tiles_n"]):
            for ty in range(p["tiles_y"]):
                for tx in range(p["tiles_x"]):
                    n0, iy0, ix0 = tn * TN, ty * TH, tx * TW
                    acc = torch.zeros((TN, TH, TW, 2 * Cout), dtype=x.dtype)
                    for ti in range(lo, hi):
                        dx, dy, widx = p["taps"][ti]
                        widx2 = p["widx2"][ti]
                        assert widx >= 0 or widx2 >= 0
                        box = torch.zeros((TN, TH, TW, Cin), dtype=x.dtype)
                        for a in range(TN):
                            for b in range(TH):
                                for c in range(TW):
                                    n, yy, xx = n0 + a, iy0 + b + dy, ix0 + c + dx
                                    if n < N and 0 <= yy < Hin and 0 <= xx < Win:
                                        box[a, b, c] = x[n, yy, xx]
                        if widx >= 0:
                            acc[..., :Cout] += box @ w_taps[widx].t()
                        if widx2 >= 0:
                            acc[..., Cout:] += box @ w_taps[widx2].t()
                    for a in range(TN):
                        for b in range(TH):
                            for c in range(TW):
                                n, iy, ix = n0 + a, iy0 + b, ix0 + c
                                if n < N and iy < p["Hit"] and ix < p["Wit"]:
                                    for px in range(2):
                                        oy, ox = 2 * iy + py, 2 * ix + px
                                        out[n, oy, ox] = acc[a, b, c, px * Cout:(px + 1) * Cout]
                                        written[n, oy, ox] += 1
    assert int(written.min()) == 1 and int(written.max()) == 1
    return out


@pytest.mark.parametrize("N,Cin,H,W,Cout,k,pad,out_hw,units", [(2, 5, 9, 12, 40, 4, 1, None, 12), (2, 3, 8, 12, 64, 5, 1, (16, 24), 15),
                                                              (2, 4, 8, 12, 33, 3, 0, (16, 24), 6)])
def test_two_parity_classes_per_tile_plan(N, Cin, H, W, Cout, k, pad, out_hw, units):
    """Narrow (33..64 channel) transposed layers: the paired plan covers every output exactly once, reproduces
    conv_transpose2d, and needs `units` (input offset, class pair) blocks per channel block where the plain plan has
    k * k (tap, class) blocks: k4 s2 12 instead of 16, 5x5 s2 15 instead of 25, 3x3 s2 6 instead of 9 -- each at
    N = 128, which costs the tensor core the same as the plain plan's N = 64."""
    g = torch.Generator().manual_seed(k * 5 + Cout)
    x = torch.randn(N, Cin, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(Cin, Cout, k, k, generator=g, dtype=torch.float64)
    Ho, Wo = (H - 1) * 2 - 2 * pad + k, (W - 1) * 2 - 2 * pad + k
    oph = opw = 0
    if out_hw:
        oph, opw = out_hw[0] - Ho, out_hw[1] - Wo
        Ho, Wo = out_hw
    ref = F.conv_transpose2d(x, w, stride=2, padding=pad, output_padding=(max(oph, 0), max(opw, 0)))[:, :, :Ho, :Wo]
    p = plan(N, H, W, Cin, Ho, Wo, Cout, 1 | 4, 2, k, k, pad, pad)
    assert p["pair_px"] == 1 and p["ntaps"] == units
    plain = plan(N, H, W, Cin, Ho, Wo, Cout, 1, 2, k, k, pad, pad)
    assert plain["pair_px"] == 0 and plain["ntaps"] == k * k and plain["BN"] == 64
    w_taps = w.permute(2, 3, 1, 0).reshape(k * k, Cout, Cin)
    got = execute_pair_px(p, x.permute(0, 2, 3, 1), w_taps, N, Ho, Wo, Cout)
    torch.testing.assert_close(got.permute(0, 3, 1, 2), ref, rtol=1e-12, atol=1e-12)
    # layers it is not meant for keep the plain plan
    assert plan(N, H, W, Cin, Ho, Wo, 128, 1 | 4, 2, k, k, pad, pad)["pair_px"] == 0
    assert plan(N, H, W, Cin, Ho, Wo, 16, 1 | 4, 2, k, k, pad, pad)["pair_px"] == 0
