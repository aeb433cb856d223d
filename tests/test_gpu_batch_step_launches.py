"""Every launch of the FlowNetC training step at per-rank batches 1, 2 and 3, checked against float64.

The reference's default [run] batch_size = 4 is divided over the GPUs of gpu_list: with 4 GPUs every rank trains on
batch 1, with 2 GPUs on batch 2, and batch_size = 12 on 4 GPUs gives batch 3.  The batch changes the plan the
tensor-core kernels run (tests/test_tc_batch_plans_cpu.py pins it): at batch 1 (N = 2, both directions) conv5, conv6
and conv6_1 and the input gradients of conv5_1, conv6_1 and deconv5 are cut into four K slices whose partial sums
meet in the output through red.add, the forwards followed by unflow_bias_lrelu; conv5_1's plan reports four slices
too but its output is a channel slice of concat5 that gets bias + leaky ReLU, so the launcher must not slice it;
every one of those launches has fewer work items than the 132 SMs and runs on the stream-K schedule alone; and the
small levels take other tile boxes (TN = 1 at N = 2, TN = 3 and 6 at N = 6).

Each case runs one eager Trainer.step in 3xTF32 (run_checked_step of test_gpu_variant_step_launches.py) with both
shadow checks installed: the Recorder of test_gpu_tc_step_launches.py on tc_conv (bound TAU) and the LibProxy with
VARIANT_CHECKERS on the library handle (TAU_SUM, TAU_LOSS, TAU_ADAM, TAU_FOLD).  Cases: FlowNetC at 384x1280 with
batch 1, 2 and 3 (the [train_kitti] loss), the CSS stack at batch 1 (each rank of a data-parallel bench.py --spec
CSS run), and the evaluation forward (eval.network_flow_fn on one 384x1280 pair, no gradient).  Each case asserts
every checked launch within its bound, no entry point without a checker, the entry points called
(native_entry_points.BATCH_STEP_CALLS), and the paths: every tc_conv launch is joined with unflow_tc_conv_plan on
its own arguments and with the launches the library counted during it (unflow_bias_lrelu runs inside
unflow_tc_conv, so it shows as a second counted launch rather than as a call of the handle), and the launches of
the pinned table must have run with the plan pinned there, the K-sliced forwards with their bias pass, conv5_1
unsliced.  A planner change that moves these regimes fails here by name.

Measured on an H100 SXM 80 GB (HBM3) at a 700 W power limit: checked launches (library + tensor-core), the worst
|err| / A per family (TAU: tensor core 1e-5, sum 4e-6, level loss 6e-5, Adam 2e-6, fold 2^-24) and over the
K-sliced tc_conv launches alone, the seconds of each case and torch.cuda.max_memory_allocated() over it.

  case     launches   tensor core  sum      level loss  Adam     fold     K-sliced (launches)   time    peak
  C-b1     114 + 61   3.8e-6       1.2e-6   9.2e-6      3.0e-7   6.0e-8   2.9e-7 (6)            3.9 s   5.54 GiB
  C-b2     114 + 61   3.3e-6       1.2e-6   1.1e-5      3.0e-7   6.0e-8   3.3e-7 (6)            2.4 s   5.94 GiB
  C-b3     114 + 61   2.7e-6       1.2e-6   6.7e-6      2.8e-7   6.0e-8   3.7e-7 (4)            2.9 s   6.33 GiB
  CSS-b1   158 + 95   5.3e-6       1.2e-6   2.8e-6      2.3e-7   -        3.1e-7 (12)           2.5 s   6.32 GiB
  eval      47 + 19   1.3e-6       1.2e-6   2.2e-6      -        -        2.8e-7 (3)            0.9 s   1.16 GiB

Copies (relayout, weight split) are bit-exact in every case.  The negative control (conv6_1 at batch 1, four K
slices): correct 1.5e-7, slice 1 left out 7.9e-2, bias added twice 0.12, each over 7000 x TAU.  The file takes
about 13 s of GPU time.
"""
import time

import pytest
import torch

import native_entry_points as EP
from test_gpu_step_launches import LibProxy, count_input_copies
from test_gpu_tc_conv import real_lib
from test_gpu_tc_step_launches import TAU, Recorder, check_run
from test_gpu_variant_step_launches import (CSS_BENCH_PARAMS, KITTI_PARAMS, VARIANT_CHECKERS, run_checked_step,
                                            worst_by_family)
from test_tc_batch_plans_cpu import PINNED, conv_plan, launches

pytestmark = pytest.mark.gpu

SMS = 132
H, W = 384, 1280

# id -> (loss parameters, per-rank batch); "eval" is the evaluation forward at batch 1
CASES = {
    "C-b1": (KITTI_PARAMS, 1),
    "C-b2": (KITTI_PARAMS, 2),
    "C-b3": (KITTI_PARAMS, 3),
    "CSS-b1": (CSS_BENCH_PARAMS, 1),
    "eval": (KITTI_PARAMS, 1),
}


# ---- the plan of each tc_conv launch ----------------------------------------------------------------------------
def track_plans(monkeypatch):
    """Wraps tc_conv.run (before the Recorder takes it): the returned list gets, per launch in call order, its
    unflow_tc_conv_plan arguments, its epilogue and the launches the library counted during the call (add_plans
    joins the plan)."""
    from unflow_b200.e2eflow.core import tc_conv
    real, rows = tc_conv.run, []

    def run(x, planes, out, *, mode, stride, kh, kw, pad_t, pad_l, bias=None, act=False, accumulate=False, slope=0.1):
        lib = real_lib()
        n0 = lib.unflow_launch_count()
        real(x, planes, out, mode=mode, stride=stride, kh=kh, kw=kw, pad_t=pad_t, pad_l=pad_l, bias=bias, act=act,
             accumulate=accumulate, slope=slope)
        launched = lib.unflow_launch_count() - n0
        N, Hin, Win, Cin, _ = tc_conv.nhwc_geometry(x)
        _, Hout, Wout, Cout, yp = tc_conv.nhwc_geometry(out)
        assert kh == kw
        rows.append(dict(args=(N, Hin, Win, Cin, Hout, Wout, Cout, mode, stride, kh, pad_t, pad_l), fma=Cin <= 4,
                         post=bias is not None and act, dense=yp == Cout and Cout % 4 == 0, acc=bool(accumulate),
                         launched=launched))
        return out
    monkeypatch.setattr(tc_conv, "run", run)
    return rows


def add_plans(rows):
    """The plan of each row, queried once the step is over (a query during it would be a call of the step)."""
    for r in rows:
        p = conv_plan(*r["args"])
        r.update(items=p["items"], ksplit=p["ksplit"], TN=p["TN"])
    return rows


def sliced(r):
    """The launcher cuts the launch into K slices (csrc/tc_conv.cu: unflow_tc_conv)."""
    return (not r["fma"] and r["ksplit"] > 1 and
            (not r["post"] or (r["dense"] and not r["acc"])))


def path_misses(B, plans, train):
    """The regimes the launches of batch B must take and did not (descriptions); empty when they took them all."""
    L = launches(B)
    by_key = {key: [r for r in plans if r["args"] == val[0]] for key, val in L.items() if key[1] != "dW"}
    need = []
    # a bias + leaky ReLU launch that is K-sliced counts a second launch (unflow_bias_lrelu), any other one
    bad = [r["args"] for r in plans if r["launched"] != (2 if sliced(r) and r["post"] else 1)]
    need.append(("one launch per call, two for a K-sliced bias + leaky ReLU launch: %s" % bad, not bad))
    for key, want in PINNED.items():
        if key[1] == "dX" and not train:
            continue
        rows = by_key[key]
        items, ks, tn = want[B - 1]
        need.append(("%s %s ran" % key, bool(rows)))
        got = sorted({(r["items"], r["ksplit"], r["TN"]) for r in rows})
        need.append(("%s %s planned as (items, K slices, TN) %s, got %s" % (key + (want[B - 1], got)),
                     got in ([], [want[B - 1]])))
    if B == 1:
        fwd = [("conv5", "fwd"), ("conv6", "fwd"), ("conv6_1", "fwd")]
        dx = [("conv5_1", "dX"), ("conv6_1", "dX"), ("deconv5", "dX")] if train else []
        for key in fwd:
            need.append(("%s %s: 4 K slices, then unflow_bias_lrelu" % key,
                         bool(by_key[key]) and all(sliced(r) and r["ksplit"] == 4 and r["post"] and r["launched"] == 2
                                                   for r in by_key[key])))
        for key in dx:
            need.append(("%s %s: 4 K slices, no epilogue" % key,
                         bool(by_key[key]) and all(sliced(r) and r["ksplit"] == 4 and not r["post"]
                                                   for r in by_key[key])))
        need.append(("every launch of the table under %d work items" % SMS,
                     all(r["items"] < SMS for key in PINNED for r in by_key[key])))
    if B in (1, 2):
        c51 = by_key[("conv5_1", "fwd")]
        need.append(("conv5_1 forward: the plan reports K slices, bias + leaky ReLU into a concat slice, unsliced",
                     bool(c51) and all(r["ksplit"] > 1 and r["post"] and not r["dense"] and not sliced(r)
                                       and r["launched"] == 1 for r in c51)))
    if B == 3:
        need.append(("a launch with TN = 3", any(r["TN"] == 3 and not r["fma"] for r in plans)))
        need.append(("a launch with TN = 6", any(r["TN"] == 6 and not r["fma"] for r in plans)))
    return [d for d, ok in need if not ok]


# ---- the cases ------------------------------------------------------------------------------------------------
def run_checked_eval(monkeypatch, B):
    """eval.network_flow_fn on one pair with both shadow checks around the call -> (proxy, rec, copies)."""
    from unflow_b200 import _native
    from unflow_b200 import synthetic as synth
    from unflow_b200.e2eflow.core import conv_ops, tc_conv
    from unflow_b200.e2eflow.core.flownet import FlowNetVariables
    from unflow_b200.eval import network_flow_fn

    prev = conv_ops.get_mode()
    conv_ops.set_mode("3xtf32")
    rec = Recorder(tc_conv, conv_ops)
    try:
        v = FlowNetVariables("C", False, seed=1234).cuda()
        fn = network_flow_fn(dict(KITTI_PARAMS), synth.KITTI_NORMALIZATION, v)
        im1, im2, _ = synth.image_pair(B, H, W, seed=1234)
        im1, im2 = im1.cuda(), im2.cuda()
        proxy = LibProxy(_native.lib(), VARIANT_CHECKERS)
        rec.install(monkeypatch)
        copies = count_input_copies(monkeypatch, conv_ops)
        monkeypatch.setattr(_native, "_lib", proxy)
        try:
            fn(im1, im2)
            torch.cuda.synchronize()
        finally:
            monkeypatch.setattr(_native, "_lib", proxy._real)
    finally:
        conv_ops.set_mode(prev)
    return proxy, rec, copies


@pytest.mark.parametrize("cid", list(CASES))
def test_every_launch_at_a_per_rank_batch(monkeypatch, cid):
    params, B = CASES[cid]
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    plans = track_plans(monkeypatch)
    if cid == "eval":
        proxy, rec, copies = run_checked_eval(monkeypatch, B)
        loss = float("nan")
    else:
        proxy, rec, copies, _, loss = run_checked_step(monkeypatch, params, False, B, H, W)
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    add_plans(plans)
    print("\n" + proxy.table())
    print(rec.table())
    print("%s: %d + %d checked launches, worst |err|/A by family: %s, loss %.6f, %.1f s, peak %.2f GiB" % (
        cid, proxy.launches, len(rec.rows), {k: "%.3e" % v for k, v in worst_by_family(proxy, rec).items()}, loss,
        time.time() - t0, peak))
    print("entry points called: %s" % sorted(proxy.calls))
    print("tc_conv plans (args: items / K slices / TN, sliced, counted launches):")
    for r in plans:
        if r["items"] < SMS and not r["fma"]:
            print("  %s: %d / %d / %d %s %d" % (r["args"], r["items"], r["ksplit"], r["TN"],
                                                "sliced" if sliced(r) else "-", r["launched"]))
    assert not proxy.unchecked, "entry points without a checker: %s" % sorted(set(proxy.unchecked))
    assert not copies, "inputs copied for the tensor-core layers: %s" % copies
    bad = [r for r in proxy.rows if not r[4] <= r[5]]
    assert not bad, "over TAU: %s" % bad
    bad_tc = [i for i, r in enumerate(rec.rows) if not r["ratio"] <= TAU]
    assert not bad_tc, "tensor-core launches over TAU = %g: %s" % (TAU, bad_tc)
    runs = [r for r in rec.rows if r["kind"] in ("conv s1", "conv s2", "transposed s1", "transposed s2")]
    assert len(runs) == len(plans)
    missing = path_misses(B, plans, train=cid != "eval")
    assert not missing, "%s did not take: %s" % (cid, missing)
    pinned = EP.BATCH_STEP_CALLS[cid]
    assert proxy.calls == pinned, "entry points called changed: +%s -%s" % (
        sorted(proxy.calls - pinned), sorted(pinned - proxy.calls))


# ---- negative control ---------------------------------------------------------------------------------------------
def test_the_bound_catches_a_lost_k_slice_and_a_doubled_bias():
    """conv6_1's forward at batch 1 (N = 2, 6x20, 1024 -> 1024, bias + leaky ReLU, four K slices and the bias pass)
    checked by the Recorder's check_run against the right reference and two wrong ones: one whose weights leave out
    the K range of slice 1 (K blocks 72..143 of the 288: taps 2..4, part of the channels of each end tap), one that
    adds the bias twice.  Measured on an H100: correct 1.5e-7, slice left out 7.9e-2, bias twice 0.12."""
    from unflow_b200.e2eflow.core import tc_conv
    N, C, Hh, Ww, k = 2, 1024, 6, 20, 3
    g = torch.Generator().manual_seed(61)
    x = tc_conv.empty_nhwc(N, C, Hh, Ww, "cuda")
    x.copy_(torch.randn(N, C, Hh, Ww, generator=g) * 0.25)
    w = (torch.randn(C, k, k, C, generator=g) * (2.0 / (9 * C)) ** 0.5).cuda().permute(0, 3, 1, 2)
    b = (torch.randn(C, generator=g) * 0.5).cuda()
    planes = tc_conv.split_weights(w)
    out = tc_conv.empty_nhwc(N, C, Hh, Ww, "cuda")
    kw = dict(mode=0, stride=1, kh=k, kw=k, pad_t=1, pad_l=1)
    p = conv_plan(N, Hh, Ww, C, Hh, Ww, C, 0, 1, k, 1, 1)
    assert p["ksplit"] == 4 and p["items"] == 16
    n0 = real_lib().unflow_launch_count()
    tc_conv.run(x, planes, out, bias=b, act=True, **kw)
    torch.cuda.synchronize()
    assert real_lib().unflow_launch_count() - n0 == 2            # the sliced kernel and unflow_bias_lrelu

    kblocks = p["kblocks"]
    per = -(-p["ntaps"] * kblocks // 4)
    hi, lo = planes.hi.clone(), planes.lo.clone()
    for it in range(per, 2 * per):                               # K block it = tap * kblocks + channel block
        t, cb = divmod(it, kblocks)
        hi[t, :, 32 * cb:32 * cb + 32] = 0
        lo[t, :, 32 * cb:32 * cb + 32] = 0
    lost = tc_conv.WeightPlanes(hi, lo, planes.taps, planes.rows, planes.cols)
    good = check_run(x, planes, None, out, bias=b, act=True, **kw)
    no_slice = check_run(x, lost, None, out, bias=b, act=True, **kw)
    twice = check_run(x, planes, None, out, bias=2 * b, act=True, **kw)
    print("\ncorrect %.3e, slice 1 left out %.3e, bias twice %.3e (TAU %.0e)" % (good, no_slice, twice, TAU))
    assert good <= TAU
    assert min(no_slice, twice) >= 100 * TAU
