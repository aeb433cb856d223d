"""The tensor-core launches of a FlowNetC training step at 384x1280 for per-rank batches B = 1, 2, 3, 4, 8 and 16
(N = 2B: both directions run through the trunk), planned on the CPU.  No GPU.

The reference's default [run] batch_size = 4 divided over the GPUs of gpu_list gives every rank a batch of 1 or 2;
the batch changes the plan unflow_tc_conv / unflow_tc_wgrad run, not only the tensor sizes: which layers are cut into
K slices, how many work items a launch has (and so whether it runs on the stream-K schedule alone), and the tile and
pixel boxes.  launches(B) generates every tc_conv launch (forward and input gradient) and tc_wgrad launch of the
step from the layer table below.  For every batch each launch goes through the schedule invariants of
test_tc_schedule_cpu.py (with the K slices the launcher takes); the launches of batches 1 and 3 whose box or class plan differs from batch 4
are executed tile by tile with the plan executors of test_tc_conv_plan_cpu.py against torch; and the item / K-slice /
box table of the launches that tests/test_gpu_batch_step_launches.py relies on is pinned here, so that a planner
change cannot move them out of that test's reach unnoticed."""
import pytest
import torch
import torch.nn.functional as F

from test_tc_conv_plan_cpu import execute, execute_pair_px, execute_wgrad, plan, wgrad_plan
from test_tc_schedule_cpu import check, conv_lengths, driver, wgrad_lengths  # noqa: F401  (driver: a fixture)

H, W = 384, 1280
BATCHES = (1, 2, 3, 4, 8, 16)

# name: (kind, C_in, C_out, k, stride, pad_t = pad_l, input H, input W, output into a concat slot).  conv1 runs in
# the row-window form (unflow_tc_conv_window, no input gradient); the flow heads and their up-sampling deconvs
# contract over 2 channels and run on the narrow / FMA kernels, not on these plans.
LAYERS = {
    "conv2": ("conv", 64, 128, 5, 2, 1, H // 2, W // 2, True),
    "conv3": ("conv", 128, 256, 5, 2, 1, H // 4, W // 4, False),
    "conv_redir": ("conv", 256, 32, 1, 1, 0, H // 8, W // 8, True),
    "conv3_1": ("conv", 32 + 441, 256, 3, 1, 1, H // 8, W // 8, True),
    "conv4": ("conv", 256, 512, 3, 2, 0, H // 8, W // 8, False),
    "conv4_1": ("conv", 512, 512, 3, 1, 1, H // 16, W // 16, True),
    "conv5": ("conv", 512, 512, 3, 2, 0, H // 16, W // 16, False),
    "conv5_1": ("conv", 512, 512, 3, 1, 1, H // 32, W // 32, True),
    "conv6": ("conv", 512, 1024, 3, 2, 0, H // 32, W // 32, False),
    "conv6_1": ("conv", 1024, 1024, 3, 1, 1, H // 64, W // 64, False),
    "deconv5": ("deconv", 1024, 512, 4, 2, 1, H // 64, W // 64, True),
    "deconv4": ("deconv", 512 + 512 + 2, 256, 4, 2, 1, H // 32, W // 32, True),
    "deconv3": ("deconv", 512 + 256 + 2, 128, 4, 2, 1, H // 16, W // 16, True),
    "deconv2": ("deconv", 256 + 128 + 2, 64, 4, 2, 1, H // 8, W // 8, True),
}


def launches(B):
    """{(name, "fwd" | "dX"): (unflow_tc_conv_plan arguments without kw, K slices the launcher takes),
        (name, "dW"): unflow_tc_wgrad_plan arguments without kw} of one step at batch B.
    Forwards carry bias + leaky ReLU: the launcher slices them only into a dense output; input gradients have no
    epilogue and take the plan's slices."""
    N = 2 * B
    out = {}
    for name, (kind, ci, co, k, s, pad, hi, wi, slot) in LAYERS.items():
        if kind == "conv":
            ho, wo = -(-hi // s), -(-wi // s)
            fwd = (N, hi, wi, ci, ho, wo, co, 0, s, k, pad, pad)
            dx = (N, ho, wo, co, hi, wi, ci, 1, s, k, pad, pad)
            out[(name, "dW")] = (N, ho, wo, co, ci, s, k, pad, pad)           # P = dL/dy: rows C_out
        else:
            ho, wo = 2 * hi, 2 * wi
            fwd = (N, hi, wi, ci, ho, wo, co, 1, 2, k, pad, pad)
            dx = (N, ho, wo, co, hi, wi, ci, 0, 2, k, pad, pad)
            out[(name, "dW")] = (N, hi, wi, ci, co, 2, k, pad, pad)           # P = x: rows C_in
        out[(name, "fwd")] = (fwd, 1 if slot else conv_plan(*fwd)["ksplit"])
        out[(name, "dX")] = (dx, conv_plan(*dx)["ksplit"])
    return out


def conv_plan(N, Hin, Win, Cin, Hout, Wout, Cout, mode, stride, k, pt, pl):
    p = plan(N, Hin, Win, Cin, Hout, Wout, Cout, mode, stride, k, k, pt, pl)
    p["items"] = p["n_classes"] * p["tiles_x"] * p["tiles_y"] * p["tiles_n"] * p["n_blocks"]
    return p


def wplan(N, Hp, Wp, R, C, stride, k, pt, pl):
    p = wgrad_plan(N, Hp, Wp, R, C, stride, k, k, pt, pl)
    p["items"] = p["n_chunks"] * p["r_blocks"] * p["c_blocks"]
    return p



@pytest.mark.parametrize("B", BATCHES)
def test_schedules_of_every_launch(driver, B):  # noqa: F811
    """Every tc_conv launch (with the K slices the launcher takes) and tc_wgrad launch of the step: each (item, K
    block) run once, cuts on chunk multiples, balanced ranges (test_tc_schedule_cpu.check)."""
    for key, val in sorted(launches(B).items()):
        if key[1] == "dW":
            lengths = wgrad_lengths(*val)
            assert len(lengths) == wplan(*val)["items"], key
        else:
            args, ks = val
            lengths = conv_lengths(*args, ksplit=ks)
            assert len(lengths) == conv_plan(*args)["items"] * ks, key
        check(driver, lengths)


def _box(p):
    return (p["TW"], p["TH"], p["TN"], p["n_classes"], p["pair_px"], p["class_start"], p["taps"], p["widx2"])


def _narrow(ci, co):
    """Channel counts the executor runs a launch at: the box and class plan depend on the channels only through
    pair_px (33..64 output channels, more than 4 input channels), which these keep."""
    return min(ci, 8), (co if co <= 64 else 8)


@pytest.mark.parametrize("B", [1, 3])
def test_plans_that_differ_from_batch_4_reproduce_torch(B):
    """The tc_conv launches of batches 1 and 3 whose tile box or class plan is not the one of batch 4, executed tile
    by tile (test_tc_conv_plan_cpu.execute / execute_pair_px) at fewer channels with the same box and class plan,
    against torch's conv2d / conv_transpose2d in float64."""
    ran = []
    for key, val in sorted(launches(B).items()):
        if key[1] == "dW":
            continue
        args = val[0]
        N, Hin, Win, Cin, Hout, Wout, Cout, mode, s, k, pt, pl = args
        p = conv_plan(*args)
        if _box(p) == _box(conv_plan(*launches(4)[key][0])):
            continue
        ci, co = _narrow(Cin, Cout)
        q = conv_plan(N, Hin, Win, ci, Hout, Wout, co, mode, s, k, pt, pl)
        assert _box(q) == _box(p), key
        g = torch.Generator().manual_seed(len(ran))
        x = torch.randn(N, ci, Hin, Win, generator=g, dtype=torch.float64)
        if mode == 0:
            w = torch.randn(co, ci, k, k, generator=g, dtype=torch.float64)
            pb, pr = (Hout - 1) * s + k - Hin - pt, (Wout - 1) * s + k - Win - pl
            ref = F.conv2d(F.pad(x, (pl, pr, pt, pb)), w, stride=s)
            w_taps = w.permute(2, 3, 0, 1).reshape(k * k, co, ci)
        else:
            w = torch.randn(ci, co, k, k, generator=g, dtype=torch.float64)
            full = F.conv_transpose2d(x, w, stride=s)                  # full[s*i + k] += x[i] W[k]
            ref = full[:, :, pt:pt + Hout, pl:pl + Wout]
            assert ref.shape[2:] == (Hout, Wout)
            w_taps = w.permute(2, 3, 1, 0).reshape(k * k, co, ci)
        run = execute_pair_px if q["pair_px"] else execute
        got = run(q, x.permute(0, 2, 3, 1), w_taps, N, Hout, Wout, co)
        torch.testing.assert_close(got.permute(0, 3, 1, 2), ref, rtol=1e-12, atol=1e-12)
        ran.append(key)
    # the small levels change their boxes with the batch (TN = 1 at N = 2, TN = 3 or 6 at N = 6)
    assert {("conv5", "fwd"), ("conv5_1", "dX"), ("deconv4", "dX")} <= set(ran), ran
    if B == 3:
        assert {("conv6", "fwd"), ("conv6_1", "dX"), ("deconv5", "dX")} <= set(ran), ran


@pytest.mark.parametrize("B", [1, 3])
def test_wgrad_boxes_that_differ_from_batch_4_reproduce_torch(B):
    """The tc_wgrad launches of the coarse levels (at most 24x80 pixels) whose pixel box differs from batch 4,
    executed K block by K block (test_tc_conv_plan_cpu.execute_wgrad) at fewer channels with the same box."""
    ran = []
    for key, args in sorted(launches(B).items()):
        if key[1] != "dW":
            continue
        N, Hp, Wp, R, C, s, k, pt, pl = args
        p = wgrad_plan(N, Hp, Wp, R, C, s, k, k, pt, pl)
        p4 = wgrad_plan(*launches(4)[key][:5], s, k, k, pt, pl)
        if Hp * Wp > 24 * 80 or (p["TW"], p["TH"], p["TN"]) == (p4["TW"], p4["TH"], p4["TN"]):
            continue
        r, c = min(R, 8), min(C, 8)
        q = wgrad_plan(N, Hp, Wp, r, c, s, k, k, pt, pl)
        assert (q["TW"], q["TH"], q["TN"]) == (p["TW"], p["TH"], p["TN"]), key
        g = torch.Generator().manual_seed(len(ran))
        Hg, Wg = (Hp * s, Wp * s) if LAYERS[key[0]][0] == "conv" else (Hp * 2, Wp * 2)
        P = torch.randn(N, r, Hp, Wp, generator=g, dtype=torch.float64)
        G = torch.randn(N, c, Hg, Wg, generator=g, dtype=torch.float64)
        # dw[r, c, ky, kx] = sum_p P[p, r] G[s*p + k - pad, c]
        pb, pr = (Hp - 1) * s + k - Hg - pt, (Wp - 1) * s + k - Wg - pl
        gin = F.pad(G, (pl, max(pr, 0), pt, max(pb, 0)))[:, :, :(Hp - 1) * s + k, :(Wp - 1) * s + k]
        ref = torch.nn.grad.conv2d_weight(gin, (r, c, k, k), P, stride=s)
        got = execute_wgrad(q, P.permute(0, 2, 3, 1), G.permute(0, 2, 3, 1), s, k, k, pt, pl)
        torch.testing.assert_close(got.reshape(r, k, k, c).permute(0, 3, 1, 2), ref, rtol=1e-11, atol=1e-11)
        ran.append(key[0])
    assert {"conv6", "conv6_1"} <= set(ran), ran


# The launches tests/test_gpu_batch_step_launches.py relies on: per batch B = 1, 2, 3, 4 the (work items, K slices
# of the plan, TN of the tile box).  conv5_1's forward writes a channel slice of concat5 with bias + leaky ReLU, so
# the launcher runs it unsliced whatever the plan reports.
PINNED = {
    # B:                   1             2             3             4
    ("conv5", "fwd"): ((32, 4, 1), (60, 2, 4), (96, 1, 3), (120, 1, 8)),
    ("conv6", "fwd"): ((16, 4, 2), (32, 4, 2), (48, 2, 6), (64, 2, 2)),
    ("conv6_1", "fwd"): ((16, 4, 2), (32, 4, 2), (48, 2, 6), (64, 2, 2)),
    ("conv5_1", "dX"): ((32, 4, 1), (60, 2, 4), (96, 1, 3), (120, 1, 8)),
    ("conv6_1", "dX"): ((16, 4, 2), (32, 4, 2), (48, 2, 6), (64, 2, 2)),
    ("deconv5", "dX"): ((16, 4, 2), (32, 4, 2), (48, 2, 6), (64, 2, 2)),
    ("conv6", "dX"): ((32, 1, 2), (64, 1, 2), (96, 1, 6), (128, 1, 2)),
    ("deconv4", "dX"): ((72, 1, 1), (135, 1, 4), (216, 1, 3), (270, 1, 8)),
    ("conv5_1", "fwd"): ((32, 4, 1), (60, 2, 4), (96, 1, 3), (120, 1, 8)),
}
# tc_wgrad: (TW, TH, TN, work items)
PINNED_WGRAD = {
    "conv6": ((8, 2, 2, 576), (4, 2, 4, 576), (8, 2, 2, 864), (4, 1, 8, 864)),
    "conv2": ((32, 1, 1, 780), (32, 1, 1, 793), (32, 1, 1, 793), (32, 1, 1, 793)),
}


def test_pinned_plans():
    for B in (1, 2, 3, 4):
        L = launches(B)
        for key, want in PINNED.items():
            args, ks = L[key]
            p = conv_plan(*args)
            got = (p["items"], p["ksplit"], p["TN"])
            assert got == want[B - 1], "%s at batch %d: (items, K slices, TN) %s, pinned %s" % (
                key, B, got, want[B - 1])
            assert ks == (1 if key == ("conv5_1", "fwd") else p["ksplit"])
        for name, want in PINNED_WGRAD.items():
            p = wplan(*L[(name, "dW")])
            got = (p["TW"], p["TH"], p["TN"], p["items"])
            assert got == want[B - 1], "%s dW at batch %d: (TW, TH, TN, items) %s, pinned %s" % (
                name, B, got, want[B - 1])
