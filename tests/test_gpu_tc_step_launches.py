"""Every tensor-core launch of one FlowNetC training step, checked against float64 at the step's own shapes.

One eager step as bench.py runs it (batch 4 at 384x1280, 3xTF32, default options) with tc_conv.run / wgrad /
run_window / wgrad_window wrapped: each call snapshots the destination (input gradients accumulate into shared
gradient slots, weight gradients into w.grad, and the Siamese conv1..conv3 weights get two calls), runs, and is
compared with a float64 evaluation of the formulas in include/unflow.h on the same operands.  The weights are
taken as hi + lo of the planes the kernel read, which is exactly the fp32 variable.

The bound is elementwise and cannot be hidden by cancellation:  |got - ref| <= TAU * A, where A is the same
float64 operation applied to |operands| (plus |bias| and |old destination|).  Error model: the 3xTF32 split drops
lo * lo' and truncates lo to TF32 (~2^-21 of a product); each wgmma instruction truncates the accumulator once,
12 instructions per K block, 96 per chunk of 8 K blocks; the fp32 sums of chunks, of K slices and of the
weight-gradient split-K atomics round to nearest.  A 1xTF32 kernel is off by ~2^-11 of A and fails by far.
Measured on an H100 SXM 80 GB (400 W power limit): 61 launches, worst ratio 3.3e-6 (the weight gradient of
deconv5, 1024 x 512 channels over 8 x 6 x 20 pixels); input-gradient and forward launches stay under 1.4e-6.
TAU = 1e-5 leaves a margin of 3x.  The whole file takes about 2 s of GPU time.
"""
import sys
import time

import pytest
import torch
import torch.nn.functional as F

from test_gpu_tc_conv import launch_plan, real_lib

pytestmark = pytest.mark.gpu

TAU = 1e-5


# ---- float64 references (include/unflow.h) --------------------------------------------------------------------
def _window(t, dim, start, length):
    """Elements [start, start + length) of t along dim, zero outside t."""
    n = t.shape[dim]
    before, after = max(0, -start), max(0, start + length - n)
    if before or after:
        t = F.pad(t, [0, 0] * (t.dim() - 1 - dim) + [before, after])
    return t.narrow(dim, start + before, length)


def _crop(t, hw_start, hw_len):
    return _window(_window(t, 2, hw_start[0], hw_len[0]), 3, hw_start[1], hw_len[1])


def ref_conv(x, wt, mode, stride, kh, kw, pad_t, pad_l, Hout, Wout):
    """x [N, Cin, Hin, Win], wt [kh*kw, Cout, Cin] (float64).
    mode 0: y[oy, ox] = sum_t x[stride*oy - pad_t + ky, stride*ox - pad_l + kx] W[t]
    mode 1: y[stride*iy - pad_t + ky, stride*ix - pad_l + kx] += x[iy, ix] W[t]"""
    Cout, Cin = wt.shape[1], wt.shape[2]
    w = wt.reshape(kh, kw, Cout, Cin)
    if mode == 0:
        xin = _crop(x, (-pad_t, -pad_l), (stride * (Hout - 1) + kh, stride * (Wout - 1) + kw))
        return F.conv2d(xin, w.permute(2, 3, 0, 1), stride=stride)
    full = F.conv_transpose2d(x, w.permute(3, 2, 0, 1), stride=stride)       # full[stride*i + k] += x[i] W[k]
    return _crop(full, (pad_t, pad_l), (Hout, Wout))


def ref_wgrad(P, G, stride, kh, kw, pad_t, pad_l):
    """dw[r, c, ky, kx] = sum_p P[p, r] G[stride*p + k - pad, c]"""
    Hp, Wp = P.shape[2:]
    gin = _crop(G, (-pad_t, -pad_l), (stride * (Hp - 1) + kh, stride * (Wp - 1) + kw))
    return torch.nn.grad.conv2d_weight(gin, (P.shape[1], G.shape[1], kh, kw), P, stride=stride)


def _rows(xp, stride, kh, pad_t, Hout, Wout):
    """The row-window input [N, H, Wp, Cp] as a one-channel image whose rows are Wp*Cp floats, cut to what
    output rows [0, Hout) and the 8-pixel windows of output columns [0, Wout) read."""
    N, H, Wp, Cp = xp.shape
    X = xp.reshape(N, 1, H, Wp * Cp)
    return _crop(X, (-pad_t, 0), (stride * (Hout - 1) + kh, stride * Cp * (Wout - 1) + 8 * Cp))


def ref_conv_window(xp, wt, stride, kh, pad_t, Hout, Wout):
    """y[n, co, oy, ox] = sum_{ky, j} xp[n, stride*oy + ky - pad_t, j-th float of output column ox's window]
    W[ky, co, j]; the window of column ox starts at pixel stride*ox."""
    Cp = xp.shape[3]
    X = _rows(xp, stride, kh, pad_t, Hout, Wout)
    return F.conv2d(X, wt.permute(1, 0, 2).unsqueeze(1), stride=(stride, stride * Cp))


def ref_wgrad_window(P, xp, stride, kh, pad_t):
    """dw [R, 8*Cp, kh, 1]: the weight gradient of ref_conv_window."""
    Cp = xp.shape[3]
    Ho, Wo = P.shape[2:]
    X = _rows(xp, stride, kh, pad_t, Ho, Wo)
    dw = torch.nn.grad.conv2d_weight(X, (P.shape[1], 1, kh, 8 * Cp), P, stride=(stride, stride * Cp))
    return dw.permute(0, 3, 2, 1)


def planes_f64(planes):
    """[taps, rows, cols] float64: hi + lo, exactly the fp32 weights."""
    return (planes.hi.double() + planes.lo.double())[:, :, :planes.cols]


def worst_ratio(got, ref, A):
    """max |got - ref| / A; an error where A == 0 counts as infinite."""
    err = (got.double() - ref).abs()
    return float((err / A.clamp_min(1e-300)).max()) if err.numel() else 0.0


def check_run(x, planes, old, out, *, mode, stride, kh, kw, pad_t, pad_l, bias=None, act=False, slope=0.1):
    """Worst |got - ref| / A of one tc_conv.run call: `old` = the destination before the call when it
    accumulated (float64), else None; `out` = the destination after it."""
    Hout, Wout = out.shape[2:]
    x64, wt = x.double(), planes_f64(planes)
    ref = ref_conv(x64, wt, mode, stride, kh, kw, pad_t, pad_l, Hout, Wout)
    A = ref_conv(x64.abs(), wt.abs(), mode, stride, kh, kw, pad_t, pad_l, Hout, Wout)
    if bias is not None:
        ref = ref + bias.double().view(1, -1, 1, 1)
        A = A + bias.double().abs().view(1, -1, 1, 1)
    if act:
        ref = F.leaky_relu(ref, slope)
    if old is not None:
        ref, A = ref + old, A + old.abs()
    return worst_ratio(out, ref, A)


# ---- the shadow check -----------------------------------------------------------------------------------------
def _caller(conv_ops):
    """The autograd function of conv_ops that made the call, e.g. '_ConvTC.backward'."""
    f = sys._getframe(2)
    while f is not None and not (f.f_globals.get("__name__") == conv_ops.__name__ and "." in f.f_code.co_qualname):
        f = f.f_back
    return f.f_code.co_qualname.split(".<locals>")[0] if f is not None else "?"


def _wgrad_plan(N, Hp, Wp, R, C, stride, kh, kw, pad_t, pad_l):
    """BN, K blocks per work item and work items along K of a tc_wgrad launch (unflow_tc_wgrad_plan)."""
    import ctypes
    v = (ctypes.c_int * 15)()
    assert real_lib().unflow_tc_wgrad_plan(N, Hp, Wp, R, C, stride, kh, kw, pad_t, pad_l, v) == 15
    return "BN%d kc%d x%d" % (v[11], v[7], v[8])


def _geom(t):
    from unflow_b200.e2eflow.core import tc_conv
    return tc_conv.nhwc_geometry(t)


class Recorder:
    def __init__(self, tc_conv, conv_ops):
        self.tc, self.ops = tc_conv, conv_ops
        self.real = {k: getattr(tc_conv, k) for k in ("run", "wgrad", "run_window", "wgrad_window")}
        self.rows = []

    def install(self, monkeypatch):
        for k in self.real:
            monkeypatch.setattr(self.tc, k, getattr(self, k))

    def run(self, x, planes, out, *, mode, stride, kh, kw, pad_t, pad_l, bias=None, act=False, accumulate=False,
            slope=0.1):
        caller = _caller(self.ops)
        old = out.double() if accumulate else None
        self.real["run"](x, planes, out, mode=mode, stride=stride, kh=kh, kw=kw, pad_t=pad_t, pad_l=pad_l, bias=bias,
                         act=act, accumulate=accumulate, slope=slope)
        torch.cuda.synchronize()
        N, Hin, Win, Cin, xp = _geom(x)
        _, Hout, Wout, Cout, yp = _geom(out)
        p = launch_plan(N, Hin, Win, Cin, Hout, Wout, Cout, mode, stride, kh, kw, pad_t, pad_l)
        sliceable = (bias is None and not act) or (bias is not None and act and not accumulate and yp == Cout
                                                   and Cout % 4 == 0)
        ks = p["ksplit"] if sliceable else 1
        ratio = check_run(x, planes, old, out, mode=mode, stride=stride, kh=kh, kw=kw, pad_t=pad_t, pad_l=pad_l,
                          bias=bias, act=act, slope=slope)
        kind = ("conv s%d" % stride) if mode == 0 else ("transposed s%d" % stride)
        self.rows.append(dict(caller=caller, kind=kind, mode=mode, stride=stride, k=kh, nhw=(N, Hin, Win),
                              ch="%d->%d" % (Cin, Cout), pitch="%d/%d" % (xp, yp), acc=bool(accumulate),
                              ba="%s/%s" % ("b" if bias is not None else "-", "a" if act else "-"),
                              plan="BN%d cls%d%s%s" % (p["BN"], p["n_classes"], " pair" if p["pair_px"] else "",
                                                       " ks%d" % ks if ks > 1 else ""),
                              classes=p["n_classes"], pair=bool(p["pair_px"]), ksplit=ks, ratio=ratio))
        return out

    def wgrad(self, P, G, dw, *, stride, kh, kw, pad_t, pad_l):
        caller = _caller(self.ops)
        old = dw.double()
        self.real["wgrad"](P, G, dw, stride=stride, kh=kh, kw=kw, pad_t=pad_t, pad_l=pad_l)
        torch.cuda.synchronize()
        P64, G64 = P.double(), G.double()
        ref = old + ref_wgrad(P64, G64, stride, kh, kw, pad_t, pad_l)
        A = old.abs() + ref_wgrad(P64.abs(), G64.abs(), stride, kh, kw, pad_t, pad_l)
        N, Hp, Wp, R, pp = _geom(P)
        _, Hg, Wg, C, gp = _geom(G)
        kind = "deconv wgrad" if caller.startswith("_DeconvTC") else "conv wgrad"
        plan = _wgrad_plan(N, Hp, Wp, R, C, stride, kh, kw, pad_t, pad_l)
        self.rows.append(dict(caller=caller, kind=kind, mode="-", stride=stride, k=kh, nhw=(N, Hp, Wp),
                              ch="%dx%d" % (R, C), pitch="%d/%d" % (pp, gp), acc=True, ba="-/-", plan=plan,
                              classes=0, pair=False, ksplit=1, ratio=worst_ratio(dw, ref, A)))
        return dw

    def run_window(self, xp, planes, out, *, kh, stride, pad_t, bias=None, act=False, slope=0.1):
        caller = _caller(self.ops)
        self.real["run_window"](xp, planes, out, kh=kh, stride=stride, pad_t=pad_t, bias=bias, act=act, slope=slope)
        torch.cuda.synchronize()
        Hout, Wout = out.shape[2:]
        x64, wt = xp.double(), planes_f64(planes)
        ref = ref_conv_window(x64, wt, stride, kh, pad_t, Hout, Wout)
        A = ref_conv_window(x64.abs(), wt.abs(), stride, kh, pad_t, Hout, Wout)
        if bias is not None:
            ref = ref + bias.double().view(1, -1, 1, 1)
            A = A + bias.double().abs().view(1, -1, 1, 1)
        if act:
            ref = F.leaky_relu(ref, slope)
        N, H, Wp, Cp = xp.shape
        self.rows.append(dict(caller=caller, kind="window fwd", mode=0, stride=stride, k=kh, nhw=(N, H, Wp),
                              ch="%d->%d" % (8 * Cp, out.shape[1]), pitch="%d/%d" % (Cp, _geom(out)[4]), acc=False,
                              ba="%s/%s" % ("b" if bias is not None else "-", "a" if act else "-"), plan="",
                              classes=1, pair=False, ksplit=1, ratio=worst_ratio(out, ref, A)))
        return out

    def wgrad_window(self, P, xp, dw, *, kh, stride, pad_t):
        caller = _caller(self.ops)
        old = dw.double()
        self.real["wgrad_window"](P, xp, dw, kh=kh, stride=stride, pad_t=pad_t)
        torch.cuda.synchronize()
        P64, x64 = P.double(), xp.double()
        ref = old + ref_wgrad_window(P64, x64, stride, kh, pad_t)
        A = old.abs() + ref_wgrad_window(P64.abs(), x64.abs(), stride, kh, pad_t)
        N, Ho, Wo, R, pp = _geom(P)
        plan = _wgrad_plan(N, Ho, Wo, R, 8 * xp.shape[3], stride, kh, 1, pad_t, 0)
        self.rows.append(dict(caller=caller, kind="window wgrad", mode="-", stride=stride, k=kh, nhw=(N, Ho, Wo),
                              ch="%dx%d" % (R, 8 * xp.shape[3]), pitch="%d/%d" % (pp, xp.shape[3]), acc=True,
                              ba="-/-", plan=plan, classes=0, pair=False, ksplit=1, ratio=worst_ratio(dw, ref, A)))
        return dw

    def table(self):
        head = "%3s %-22s %-14s %2s %2s %-15s %-10s %-9s %-3s %-4s %-22s %s" % (
            "#", "caller", "kind", "s", "k", "N x H x W", "channels", "pitches", "acc", "b/a", "plan",
            "worst |err|/A")
        lines = [head]
        for i, r in enumerate(self.rows):
            lines.append("%3d %-22s %-14s %2s %2s %-15s %-10s %-9s %-3s %-4s %-22s %.3e" % (
                i, r["caller"], r["kind"], r["stride"], r["k"], "x".join(map(str, r["nhw"])), r["ch"], r["pitch"],
                "y" if r["acc"] else "", r["ba"], r["plan"], r["ratio"]))
        return "\n".join(lines)


def test_every_tensor_core_launch_of_a_training_step(monkeypatch):
    from unflow_b200 import synthetic as synth
    from unflow_b200.e2eflow.core import conv_ops, tc_conv
    from unflow_b200.e2eflow.core.train import Trainer

    t0 = time.time()
    dev = torch.device("cuda", 0)
    prev = conv_ops.get_mode()
    conv_ops.set_mode("3xtf32")
    rec = Recorder(tc_conv, conv_ops)
    try:
        trainer = Trainer(dict(synth.KITTI_PARAMS, flownet="C"), synth.KITTI_NORMALIZATION, dev, seed=1234)
        im1, im2, _ = synth.image_pair(4, 384, 1280, seed=1234)
        rec.install(monkeypatch)
        loss = trainer.step(im1.to(dev), im2.to(dev))
        torch.cuda.synchronize()
    finally:
        conv_ops.set_mode(prev)
    print("\n" + rec.table())
    worst = max(rec.rows, key=lambda r: r["ratio"])
    print("%d launches, worst |err|/A %.3e (launch %d), loss %.6f, %.1f s" % (
        len(rec.rows), worst["ratio"], rec.rows.index(worst), float(loss), time.time() - t0))

    bad = [i for i, r in enumerate(rec.rows) if not r["ratio"] <= TAU]
    assert not bad, "launches over TAU = %g: %s" % (TAU, bad)
    kinds = {
        "conv s1": lambda r: r["kind"] == "conv s1",
        "conv s2": lambda r: r["kind"] == "conv s2",
        "transposed, 4 classes": lambda r: r["mode"] == 1 and r["classes"] == 4,
        "pair_px": lambda r: r["pair"],
        "K-sliced": lambda r: r["ksplit"] > 1,
        "accumulate": lambda r: r["kind"] in ("conv s1", "conv s2", "transposed s1", "transposed s2") and r["acc"],
        "window fwd": lambda r: r["kind"] == "window fwd",
        "window wgrad": lambda r: r["kind"] == "window wgrad",
        "conv wgrad": lambda r: r["kind"] == "conv wgrad",
        "deconv wgrad": lambda r: r["kind"] == "deconv wgrad",
    }
    missing = [name for name, pred in kinds.items() if not any(pred(r) for r in rec.rows)]
    assert not missing, missing


def test_the_bound_catches_a_dropped_lo_plane():
    """Negative control: the checker of the step test on a launch whose weight lo plane is zeroed (1xTF32-class
    weights).  w = 1 + 2^-12 everywhere, so hi = 1 and lo = 2^-12: with U(0, 1) activations every output loses
    2^-12 / (1 + 2^-12) of A, far over TAU."""
    from unflow_b200.e2eflow.core import tc_conv
    g = torch.Generator().manual_seed(3)
    N, Cin, Cout, H, W = 2, 64, 64, 12, 20
    x = tc_conv.empty_nhwc(N, Cin, H, W, "cuda")
    x.copy_(torch.rand(N, Cin, H, W, generator=g))
    w = torch.full((Cout, 3, 3, Cin), 1.0 + 2.0 ** -12, device="cuda").permute(0, 3, 1, 2)
    planes = tc_conv.split_weights(w)
    assert bool((planes.lo[:, :, :Cin] == 2.0 ** -12).all())
    out = tc_conv.empty_nhwc(N, Cout, H, W, "cuda")
    kw = dict(mode=0, stride=1, kh=3, kw=3, pad_t=1, pad_l=1)
    tc_conv.run(x, planes, out, **kw)
    assert check_run(x, planes, None, out, **kw) <= TAU
    no_lo = tc_conv.WeightPlanes(planes.hi, torch.zeros_like(planes.lo), planes.taps, planes.rows, planes.cols)
    tc_conv.run(x, no_lo, out, **kw)
    ratio = check_run(x, planes, None, out, **kw)
    print("lo plane zeroed: worst |err|/A %.3e" % ratio)
    assert ratio > 5 * TAU, ratio
