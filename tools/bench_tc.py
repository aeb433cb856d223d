#!/usr/bin/env python
"""Time every launch of one tensor-core conv kernel in one FlowNetC training step on one H100, one by one.

    python tools/bench_tc.py --kernel {conv,wgrad} [--reps R] [--replays K] [--compare-lib PATH] [--json FILE]

--kernel conv: tc_conv_kernel (unflow_tc_conv / unflow_tc_conv_window: forward and input gradients);
--kernel wgrad: tc_wgrad_kernel (unflow_tc_wgrad / unflow_tc_wgrad_window: weight gradients).

One eager step as bench.py runs it (batch 4 at 384x1280, 3xTF32, default options).  During the step a proxy
stands in for the library handle; each call of the chosen kernel is run as the step makes it, and then, with its
operands still alive, replayed alone with the same pointers and shapes:

  * plan: BN, tiles and work items from unflow_tc_conv_plan / unflow_tc_wgrad_plan.  For conv the K slices are
    those the launcher uses for this call's epilogue; for wgrad the K blocks per item and the chunks along K.
    Schedule (csrc/tc_schedule.h): items / 132 SMs (waves), the items run whole in round robin (DP), the items
    of the stream-K tail (SK) and the segments the tail is cut into over the grid (SK 0: plain round robin).
  * time: R launches captured in a CUDA graph, replayed K times between CUDA events; the median replay / R.
    TF32 share as bench.py counts it: 3 MMA passes x nominal flops (2 x multiply-adds of the fp32 product)
    over the data-sheet TF32 rate (989 / 2 TFLOP/s, H100 SXM, a 700 W card).
  * role timers of CTA 0 (unflow_tc_conv_debug) from one more launch: the stages of the ring, the fraction of
    its cycles the producer waits for a free stage (raw slot), and the consumers wait for a loaded one (and,
    for wgrad, for a free split slot).
  * path (conv): wgmma, or fma for the contractions over at most 4 channels that unflow_tc_conv runs on the FMA
    pipes (csrc/conv_fma.cu).  Those rows have no plan, schedule or role timers; they show the bytes the launch
    must move (the input once, the output written, and read too when the launch accumulates), the achieved
    GB/s and that amount's time at the data-sheet HBM3 bandwidth (3.35 TB/s, H100 SXM), with one total line.
  * wgrad: one more line with the launches of R = 2 rows (the weight gradients of the flow up-sampling deconvs).
  * --compare-lib PATH: the destination of this launch computed with this library twice and with the library
    at PATH twice, from the same start and on the same operands: whether the two libraries agree bit for bit,
    and the largest difference between them against the largest between two runs of the other library
    (launches cut along K add their partial sums with atomics, in a varying order).  The start is the
    destination as the step left it for conv (accumulating launches add to it) and zero for wgrad.

The destination (conv: y, wgrad: dW) is snapshotted before the replays and restored afterwards, because
accumulating launches add to it; the step itself goes on unchanged.  The card, its power limit and the median
SM clock sampled during the step are printed with the table.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

from float64_refs import view  # noqa: E402
from unflow_b200 import synthetic as synth  # noqa: E402

TF32_TFLOPS = 989.0 / 2          # H100 SXM data sheet, dense: bf16 / 2
HBM_GBS = 3350.0                 # H100 SXM data sheet, HBM3
FMA_MAX_CIN = 4                  # csrc/tc_conv.cu: unflow_tc_conv runs contractions over <= 4 channels in conv_fma.cu
GRID = 132                       # CTAs of a tc launch (one per SM)
CHUNK = 8                        # K blocks per accumulation chunk (tc_chunk default): the stream-K cut unit


ENTRY_POINTS = {"conv": ("unflow_tc_conv", "unflow_tc_conv_window"),
                "wgrad": ("unflow_tc_wgrad", "unflow_tc_wgrad_window")}
PLANS = ("unflow_tc_conv_plan", "unflow_tc_wgrad_plan", "unflow_tc_conv_debug")
SPLIT_COST = 1                   # csrc/tc_schedule.h: kSkSplitCost, chunks per segment of a split item


def schedule(lengths, grid=GRID, chunk=CHUNK):
    """(DP items, SK items, SK segments) of make_sk_schedule (csrc/tc_schedule.h) for items of these K lengths;
    (items, 0, 0) where the launch stays round robin."""
    T = len(lengths)
    rr = [0] * grid
    for i, L in enumerate(lengths):
        rr[i % grid] += L
    waves = T // grid
    dp = (waves - 1 if T % grid and waves else waves) * grid
    sk = lengths[dp:]
    if not sk:
        return T, 0, 0
    load = [0] * grid
    for i in range(dp):
        load[i % grid] += lengths[i]
    total = sum(sk)
    lo, hi = 0, max(load) + total
    while lo < hi:
        mid = (lo + hi) // 2
        if sum(max(0, mid - d) for d in load) >= total:
            hi = mid
        else:
            lo = mid + 1
    room_all = sum(max(0, lo - d) for d in load)
    bounds, j, off, room = [], 0, 0, 0
    for g in range(grid + 1):
        if g:
            room += max(0, lo - load[g - 1])
        target = total if g == grid else total * room // room_all
        while j < len(sk) and off + sk[j] <= target:
            off += sk[j]
            j += 1
        if j == len(sk):
            bounds.append((len(sk), 0))
            continue
        k = -(-(target - off) // chunk) * chunk
        bounds.append((j, k) if k < sk[j] else (j + 1, 0))
    segs, span = 0, 0
    for g, ((j0, k0), (je, ke)) in enumerate(zip(bounds, bounds[1:])):
        cta = load[g]
        for jj in range(j0, min(je, len(sk) - 1) + 1):
            a, b = (k0 if jj == j0 else 0), (ke if jj == je else sk[jj])
            if b <= a:
                continue
            segs += 1
            cta += b - a + (SPLIT_COST * chunk if a > 0 or b < sk[jj] else 0)
        span = max(span, cta)
    if span + chunk > max(rr):
        return T, 0, 0
    return dp, len(sk), segs


def conv_plan(lib, plan_args):
    """(BN, tiles, n_classes, n_blocks, K slices when the epilogue allows slicing, K blocks per class) of
    unflow_tc_conv_plan."""
    buf = (ctypes.c_int * 1024)()
    n = lib.unflow_tc_conv_plan(*plan_args, buf, 1024)
    assert n > 0, n
    cs = list(buf[15:16 + buf[0]])
    return buf[12], buf[8] * buf[9] * buf[10], buf[0], buf[11], buf[n - 1], [(b - a) * buf[13] for a, b in zip(cs, cs[1:])]


def conv_lengths(tiles, ncls, nblk, ks, class_k):
    """K blocks of each work item in the kernel's order (csrc/tc_conv.cu: decode_work)."""
    out = []
    for w in range(tiles * ncls * nblk * ks):
        tile, s = divmod(w, ks)
        total = class_k[(tile // nblk) % ncls]
        per = -(-total // ks)
        out.append(max(0, min(per, total - s * per)))
    return out


def geometry(lib, name, a):
    """What one call does, from its ctypes arguments: the destination (pointer, floats), nominal flops, the
    plan columns of the table and whether the launch cuts K into parts that meet through atomics."""
    if name == "unflow_tc_conv":
        (_, N, Hin, Win, Cin, _, _, _, y, Hout, Wout, Cout, y_pitch, bias, _, act, accumulate, mode, stride, kh, kw,
         pad_t, pad_l, _) = a
        BN, tiles, ncls, nblk, ks, class_k = conv_plan(lib, (N, Hin, Win, Cin, Hout, Wout, Cout, mode | 4, stride, kh,
                                                             kw, pad_t, pad_l))
        # the launcher's rule (csrc/tc_conv.cu, unflow_tc_conv): slice only where the epilogue allows it
        if not ((not bias and not act) or (bias and act and not accumulate and y_pitch == Cout and Cout % 4 == 0)):
            ks = 1
        pix = N * (Hin * Win if mode == 1 else Hout * Wout)
        row = dict(kind="deconv" if mode == 1 else "conv", acc=bool(accumulate), taps="%d/%d" % (kh * kw, stride),
                   shape="%dx%dx%dx%d>%dx%dx%d" % (N, Hin, Win, Cin, Hout, Wout, Cout),
                   BN=BN, ksplit=ks, items=tiles * ncls * nblk * ks, path="wgmma")
        if Cin <= FMA_MAX_CIN:
            row.update(path="fma", bytes=4 * (N * Hin * Win * Cin + N * Hout * Wout * Cout * (2 if accumulate else 1)))
            return y, (N * Hout * Wout - 1) * y_pitch + Cout, 2 * pix * Cout * Cin * kh * kw, row, False
        row["dp"], row["sk"], row["sk_segments"] = schedule(conv_lengths(tiles, ncls, nblk, ks, class_k))
        return y, (N * Hout * Wout - 1) * y_pitch + Cout, 2 * pix * Cout * Cin * kh * kw, row, ks > 1
    if name == "unflow_tc_conv_window":
        _, N, H, _, Cp, _, _, y, Hout, Wout, Cout, y_pitch, _, _, _, kh, stride, pad_t, _ = a
        BN, tiles, ncls, nblk, _, class_k = conv_plan(lib, (N, H, Wout, 8 * Cp, Hout, Wout, Cout, 0, stride, kh, 1,
                                                            pad_t, 0))
        row = dict(kind="window", acc=False, taps="%d/%d" % (kh, stride),
                   shape="%dx%dx%dx%d>%dx%dx%d" % (N, H, Wout, 8 * Cp, Hout, Wout, Cout),
                   BN=BN, ksplit=1, items=tiles * ncls * nblk, path="wgmma")
        row["dp"], row["sk"], row["sk_segments"] = schedule(conv_lengths(tiles, ncls, nblk, 1, class_k))
        return y, (N * Hout * Wout - 1) * y_pitch + Cout, 2 * N * Hout * Wout * Cout * 8 * Cp * kh, row, False
    if name == "unflow_tc_wgrad":
        _, N, Hp, Wp, R, _, _, _, _, C, _, dw, pitch_r, _, stride, kh, kw, pad_t, pad_l, _ = a
        plan = (N, Hp, Wp, R, C, stride, kh, kw, pad_t, pad_l)
        n_dw, flops, kind, taps = R * pitch_r, 2 * N * Hp * Wp * R * C * kh * kw, "conv", kh * kw
    else:
        _, N, Ho, Wo, R, _, _, _, _, Cp, dw, kh, stride, pad_t, _ = a
        plan = (N, Ho, Wo, R, 8 * Cp, stride, kh, 1, pad_t, 0)
        n_dw, flops, kind, taps = R * kh * 8 * Cp, 2 * N * Ho * Wo * R * 8 * Cp * kh, "window", kh
    v = (ctypes.c_int * 15)()
    assert lib.unflow_tc_wgrad_plan(*plan, v) == 15
    row = dict(kind=kind, taps="%d/%d" % (taps, stride), shape="%dx%dx%d, %dx%d" % (plan[:5]), R=R,
               BN=v[11], kc=v[7], n_chunks=v[8], items=v[8] * v[9] * v[10])
    row["dp"], row["sk"], row["sk_segments"] = schedule(
        [min(v[7], v[6] - c * v[7]) for c in range(v[8]) for _ in range(v[9] * v[10])])
    return dw, n_dw, flops, row, v[8] > 1


def with_stream(a, stream):
    return a[:-1] + (stream,)


def bind(lib, kernel):
    from unflow_b200 import _native
    for name in ENTRY_POINTS[kernel] + PLANS:
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = _native.SIGNATURES[name]
    return lib


class Bench:
    """Stands in for the ctypes library handle during the step."""

    def __init__(self, real, args, other):
        self._real, self.args, self.other = real, args, other
        self.rows = []

    def __getattr__(self, name):
        fn = getattr(self._real, name)
        if name not in ENTRY_POINTS[self.args.kernel]:
            return fn

        def wrapped(*a):
            rc = fn(*a)
            if rc == 0:
                torch.cuda.synchronize()
                self.measure(name, a)
            return rc
        return wrapped

    def launch(self, lib, name, a, stream=None):
        rc = getattr(lib, name)(*(a if stream is None else with_stream(a, stream)))
        assert rc == 0, lib.unflow_last_error()

    def measure(self, name, a):
        ptr, n_dst, flops, row, sliced = geometry(self._real, name, a)
        dst = view(ptr, (n_dst,))
        keep = dst.clone()

        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            s = side.cuda_stream
            for _ in range(3):
                self.launch(self._real, name, a, s)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=side):
                for _ in range(self.args.reps):
                    self.launch(self._real, name, a, torch.cuda.current_stream().cuda_stream)
            g.replay()
            times = []
            for _ in range(self.args.replays):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                g.replay()
                e1.record()
                e1.synchronize()
                times.append(e0.elapsed_time(e1) * 1e3 / self.args.reps)
            del g
            dbg = torch.zeros(16, dtype=torch.int64, device="cuda")
            if row.get("path") != "fma":           # the FMA kernel has no role timers
                self._real.unflow_tc_conv_debug(dbg.data_ptr())
                try:
                    self.launch(self._real, name, a, s)
                finally:
                    self._real.unflow_tc_conv_debug(None)
            torch.cuda.synchronize()
            t = dbg.tolist()
            cmp = None
            if self.other is not None:
                cmp = self.compare(name, a, dst, keep if self.args.kernel == "conv" else None, s)
            dst.copy_(keep)
        torch.cuda.synchronize()

        us = statistics.median(times)
        wgrad = self.args.kernel == "wgrad"
        row.update(stages=([t[5], t[6]] if wgrad else [t[5]]) if t[5] else None, us=us,
                   tf32_share=3 * flops / (us * 1e-6) / 1e12 / TF32_TFLOPS,
                   cons_full_wait=t[2] / max(t[3], 1), prod_empty_wait=t[0] / max(t[1], 1),
                   cons_split_wait=(t[4] / max(t[3], 1)) if wgrad and t[5] else None, sliced=sliced, compare=cmp)
        if row.get("path") == "fma":
            row.update(gbs=row["bytes"] / (us * 1e-6) / 1e9, floor_us=row["bytes"] / (HBM_GBS * 1e9) * 1e6)
        self.rows.append(row)
        print(fmt(self.args.kernel, len(self.rows) - 1, row), flush=True)

    def compare(self, name, a, dst, start, s):
        """The destination from `start` (None: zero): this library twice, the other one twice."""
        def run(lib):
            if start is None:
                dst.zero_()
            else:
                dst.copy_(start)
            self.launch(lib, name, a, s)
            torch.cuda.synchronize()
            return dst.clone()
        new1, new2, old1, old2 = run(self._real), run(self._real), run(self.other), run(self.other)
        return dict(bit_identical=bool(torch.equal(new1, old1)), new_vs_old=float((new1 - old1).abs().max()),
                    old_vs_old=float((old1 - old2).abs().max()), new_vs_new=float((new1 - new2).abs().max()),
                    scale=float(old1.abs().max()))


HEAD = {
    "conv": "%3s %-5s %-6s %-3s %-26s %-6s %4s %3s %5s %6s %5s %5s %5s %6s %8s %6s %6s %6s" % (
        "#", "path", "kind", "acc", "N x Hin x Win x Cin>out", "taps/s", "BN", "ks", "items", "waves", "DP", "SK",
        "segs", "stages", "us", "tf32", "c.full", "p.empt"),
    "wgrad": "%3s %-6s %-22s %-7s %4s %3s %3s %5s %6s %5s %5s %5s %6s %8s %6s %6s %6s %6s" % (
        "#", "kind", "N x Hp x Wp, R x C", "taps/s", "BN", "kc", "ch", "items", "waves", "DP", "SK", "segs",
        "stages", "us", "tf32", "c.full", "p.empt", "c.splt"),
}


def fmt(kernel, i, r):
    st = "+".join("%d" % x for x in r["stages"]) if r["stages"] else "-"
    if kernel == "conv" and r["path"] == "fma":
        # no plan, schedule or role timers: the bytes the launch must move, the rate it moved them at, their time
        # at the data-sheet HBM bandwidth
        line = "%3d %-5s %-6s %-3s %-26s %-6s %46s %8.1f  %.1f MB, %.0f GB/s, HBM floor %.1f us" % (
            i, "fma", r["kind"], "+=" if r["acc"] else "", r["shape"], r["taps"], "", r["us"], r["bytes"] / 1e6,
            r["gbs"], r["floor_us"])
    elif kernel == "conv":
        line = "%3d %-5s %-6s %-3s %-26s %-6s %4d %3d %5d %6.2f %5d %5d %5d %6s %8.1f %5.1f%% %5.1f%% %5.1f%%" % (
            i, r["path"], r["kind"], "+=" if r["acc"] else "", r["shape"], r["taps"], r["BN"], r["ksplit"], r["items"],
            r["items"] / GRID, r["dp"], r["sk"], r["sk_segments"], st, r["us"], 100 * r["tf32_share"], 100 * r["cons_full_wait"], 100 * r["prod_empty_wait"])
    else:
        line = "%3d %-6s %-22s %-7s %4d %3d %3d %5d %6.2f %5d %5d %5d %6s %8.1f %5.1f%% %5.1f%% %5.1f%% %6s" % (
            i, r["kind"], r["shape"], r["taps"], r["BN"], r["kc"], r["n_chunks"], r["items"], r["items"] / GRID,
            r["dp"], r["sk"], r["sk_segments"], st, r["us"],
            100 * r["tf32_share"], 100 * r["cons_full_wait"], 100 * r["prod_empty_wait"],
            "-" if r["cons_split_wait"] is None else "%.1f%%" % (100 * r["cons_split_wait"]))
    c = r["compare"]
    if c:
        line += "  | bit-identical %s, max|new-old| %.2e, max|old-old| %.2e, max|new-new| %.2e (max|out| %.2e)" % (
            c["bit_identical"], c["new_vs_old"], c["old_vs_old"], c["new_vs_new"], c["scale"])
    return line


def card():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kernel", choices=sorted(ENTRY_POINTS), required=True,
                    help="conv: tc_conv_kernel (forward, input gradients); wgrad: tc_wgrad_kernel")
    ap.add_argument("--reps", type=int, default=20, help="launches per CUDA graph")
    ap.add_argument("--replays", type=int, default=5, help="timed replays of the graph")
    ap.add_argument("--compare-lib", default=None, metavar="PATH",
                    help="another build of libunflow.so to compare the destination with, launch by launch")
    ap.add_argument("--json", default=None, metavar="FILE", help="also write the rows as JSON")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tc.py needs a CUDA device")

    import bench
    from unflow_b200 import _native
    from unflow_b200.e2eflow.core import conv_ops
    from unflow_b200.e2eflow.core.train import Trainer
    real = _native.lib()
    other = bind(ctypes.CDLL(os.path.abspath(args.compare_lib)), args.kernel) if args.compare_lib else None
    conv_ops.set_mode("3xtf32")
    dev = torch.device("cuda", 0)
    trainer = Trainer(dict(synth.KITTI_PARAMS, learning_rate=1.0e-5, flownet="C"), synth.KITTI_NORMALIZATION, dev,
                      seed=1234)
    im1, im2, _ = synth.image_pair(4, 384, 1280, seed=1234)
    im1, im2 = im1.to(dev), im2.to(dev)
    trainer.step(im1, im2)
    torch.cuda.synchronize()

    sampler = bench.ClockSampler(0)
    sampler.start()
    proxy = Bench(real, args, other)
    print(HEAD[args.kernel])
    t0 = time.time()
    _native._lib = proxy
    try:
        trainer.step(im1, im2)
        torch.cuda.synchronize()
    finally:
        _native._lib = real
    clocks = sampler.window(t0, time.time())
    sampler.close()

    info = card()
    total = sum(r["us"] for r in proxy.rows)
    print("%d launches, %.3f ms in all | %s, power limit %s, SM clock median %s MHz (max %s), %d samples, "
          "throttle reasons %s" % (len(proxy.rows), total / 1e3, info.get("name"), info.get("power.limit"),
                                   clocks["sm_mhz"], info.get("clocks.max.sm"), clocks["samples"],
                                   clocks["reasons"]))
    fma = [r for r in proxy.rows if r.get("path") == "fma"]
    if fma:
        print("fma: %d launches, %.1f us in all, %.1f MB at %.0f GB/s (HBM floor %.1f us)" % (
            len(fma), sum(r["us"] for r in fma), sum(r["bytes"] for r in fma) / 1e6,
            sum(r["bytes"] for r in fma) / (sum(r["us"] for r in fma) * 1e-6) / 1e9, sum(r["floor_us"] for r in fma)))
    r2 = [(i, r) for i, r in enumerate(proxy.rows) if r.get("R") == 2]
    if r2:
        print("R = 2: %d launches, %.1f us in all (%s)" % (
            len(r2), sum(r["us"] for _, r in r2), ", ".join("#%d %.1f us" % (i, r["us"]) for i, r in r2)))
    if other is not None:
        single = [r for r in proxy.rows if not r["sliced"]]
        print("compare: %d/%d launches with one part along K bit-identical; worst max|new-old| / max|old-old| on "
              "the others %s" % (sum(r["compare"]["bit_identical"] for r in single), len(single),
                                 max((r["compare"]["new_vs_old"] / max(r["compare"]["old_vs_old"], 1e-30)
                                      for r in proxy.rows if r["sliced"]), default=None)))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(dict(kernel=args.kernel, card=info, clocks=clocks, rows=proxy.rows), fh, indent=1)


if __name__ == "__main__":
    main()
