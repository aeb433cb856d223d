"""The work-item schedule of the wgmma conv kernels (csrc/tc_schedule.h), compiled on its own with the host compiler
and run over the launches of the bench step (FlowNetC, 2 x batch 4 at 384x1280) and the plan-test shapes: the item
counts come from unflow_tc_conv_plan / unflow_tc_wgrad_plan.  For every launch: each (item, K block) is run by
exactly one CTA, cuts fall on chunk multiples from the item's start, the DP items are the round robin of a plain
persistent grid, and the K blocks per CTA differ by at most two chunks (one chunk of rounding at each end of a range;
a range's ends are cut on chunk boundaries).  No GPU."""
import ctypes
import os
import shutil
import subprocess

import pytest

from unflow_b200 import _native, build

GRID = 132
CHUNK = 8

DRIVER = r"""
#include <cstdio>
#include <vector>
#include "tc_schedule.h"
int main() {
  int items, grid, chunk;
  while (std::scanf("%d %d %d", &items, &grid, &chunk) == 3) {
    std::vector<int> len(items);
    for (int &l : len)
      if (std::scanf("%d", &l) != 1) return 1;
    static unflow::tc::SkSchedule s;
    const long long span = unflow::tc::make_sk_schedule(s, items, grid, chunk, [&](int i) { return len[i]; });
    std::printf("%lld %d %d", span, s.grid, s.dp_items);
    for (int g = 0; g <= grid; ++g) std::printf(" %d %d", s.sk_item[g], s.sk_k[g]);
    std::printf("\n");
  }
  return 0;
}
"""
SPLIT_COST = 1     # tc_schedule.h: kSkSplitCost


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    cxx = shutil.which("g++") or shutil.which("c++")
    if not cxx:
        pytest.skip("no host C++ compiler")
    d = tmp_path_factory.mktemp("sched")
    (d / "driver.cpp").write_text(DRIVER)
    subprocess.run([cxx, "-std=c++17", "-O1", "-Wall", "-Werror", "-I", build.CSRC, str(d / "driver.cpp"), "-o",
                    str(d / "driver")], check=True)

    def run(lengths, grid=GRID, chunk=CHUNK):
        text = "%d %d %d %s\n" % (len(lengths), grid, chunk, " ".join(map(str, lengths)))
        out = subprocess.run([str(d / "driver")], input=text, capture_output=True, text=True, check=True).stdout
        v = list(map(int, out.split()))
        return v[0], v[1], v[2], [(v[3 + 2 * g], v[4 + 2 * g]) for g in range(grid + 1)]
    return run


def segments(lengths, grid, dp_items, bounds):
    """Per CTA: its (item, k0, k1) list, walked as the kernels walk it (tc_common.cuh: segment_walk / segment_at)."""
    per = []
    for g in range(grid):
        segs = [(i, 0, lengths[i]) for i in range(g, dp_items, grid)]
        (j0, k0), (je, ke) = bounds[g], bounds[g + 1]
        n_sk = (1 if ke > k0 else 0) if j0 == je else je - j0 + (1 if ke > 0 else 0)
        for q in range(n_sk):
            j = j0 + q
            segs.append((dp_items + j, k0 if q == 0 else 0, ke if j == je else lengths[dp_items + j]))
        per.append(segs)
    return per


def check(run, lengths, grid=GRID, chunk=CHUNK):
    """Checks one schedule; returns (stream-K used, DP items, segments per CTA)."""
    T = len(lengths)
    span, launch_grid, dp_items, bounds = run(lengths, grid, chunk)
    rr = [sum(lengths[g::grid]) for g in range(grid)]
    if dp_items == T:                                      # plain round robin
        assert launch_grid == min(T, grid) and span == max(rr)
        assert all(b == (0, 0) for b in bounds)
        return False, T, segments(lengths, grid, T, [(0, 0)] * (grid + 1))
    assert launch_grid == grid
    waves = T // grid
    assert dp_items == (waves - 1 if T % grid and waves else waves) * grid
    assert grid <= T - dp_items < 2 * grid or T < grid
    first = next((j for j in range(T - dp_items) if lengths[dp_items + j]), T - dp_items)   # empty items: skipped
    assert bounds[0] == (first, 0) and bounds[grid] == (T - dp_items, 0)
    assert all(bounds[g] <= bounds[g + 1] for g in range(grid))
    per = segments(lengths, grid, dp_items, bounds)
    covered = {}
    for g, segs in enumerate(per):
        for (i, k0, k1) in segs:
            assert 0 <= k0 <= k1 <= lengths[i]
            if i < dp_items:
                assert i % grid == g and (k0, k1) == (0, lengths[i])          # round robin, whole items
            assert k0 % chunk == 0 and (k1 == lengths[i] or k1 % chunk == 0)   # cuts on chunk multiples
            for k in range(k0, k1):
                assert (i, k) not in covered, "K block %d of item %d twice" % (k, i)
                covered[(i, k)] = g
    assert len(covered) == sum(lengths), "K blocks left out"
    # balance: every CTA that got stream-K work ends within two chunks of the others, DP load included (a CTA
    # whose DP items alone reach past that level gets none)
    load = [sum(k1 - k0 for (_, k0, k1) in segs) for segs in per]
    busy = [load[g] for g in range(grid) if any(i >= dp_items for (i, _, _) in per[g])]
    assert max(busy) - min(busy) <= 2 * chunk - 1, (max(busy), min(busy))
    assert all(load[g] >= min(busy) - chunk for g in range(grid))
    # the model: the chosen schedule, split costs included, ends at least a chunk before round robin
    split = [sum(1 for (i, k0, k1) in segs if i >= dp_items and (k0 > 0 or k1 < lengths[i])) for segs in per]
    assert span == max(l + SPLIT_COST * chunk * s for l, s in zip(load, split))
    assert span + chunk <= max(rr)
    return True, dp_items, per


def conv_lengths(N, Hin, Win, Cin, Hout, Wout, Cout, mode, stride, k, pt, pl, ksplit=1):
    buf = (ctypes.c_int * 1024)()
    n = _native.lib().unflow_tc_conv_plan(N, Hin, Win, Cin, Hout, Wout, Cout, mode, stride, k, k, pt, pl, buf, 1024)
    assert n > 0
    ncls, nblk, kblocks = buf[0], buf[11], buf[13]
    cs = list(buf[15:20])
    tiles = buf[8] * buf[9] * buf[10]
    out = []
    for w in range(ncls * tiles * nblk * ksplit):           # tc_conv.cu: decode_work / work_len
        tile, ks = divmod(w, ksplit)
        cls = (tile // nblk) % ncls
        total = (cs[cls + 1] - cs[cls]) * kblocks
        per = -(-total // ksplit)
        out.append(max(0, min(per, total - ks * per)))
    return out


def wgrad_lengths(N, Hp, Wp, R, C, stride, k, pt, pl):
    v = (ctypes.c_int * 15)()
    assert _native.lib().unflow_tc_wgrad_plan(N, Hp, Wp, R, C, stride, k, k, pt, pl, v) == 15
    n_ptiles, kc, n_chunks, tiles = v[6], v[7], v[8], v[9] * v[10]
    return [min(kc, n_ptiles - c * kc) for c in range(n_chunks) for _ in range(tiles)]


# the bench step's tc_conv launches (N = 8: both directions, batch 4) with the item counts of the issue's table
CONV_BENCH = {
    "conv3": ((8, 96, 320, 128, 48, 160, 256, 0, 2, 5, 1, 1), 960),
    "conv3_1": ((8, 48, 160, 256, 48, 160, 256, 0, 1, 3, 1, 1), 960),
    "conv4": ((8, 48, 160, 256, 24, 80, 512, 0, 2, 3, 0, 0), 480),
    "conv5": ((8, 24, 80, 512, 12, 40, 512, 0, 2, 3, 0, 0), 120),
    "deconv4": ((8, 12, 40, 1026, 24, 80, 256, 1, 2, 4, 1, 1), 240),
    "conv2": ((8, 192, 640, 64, 96, 320, 128, 0, 2, 5, 1, 1), 1920),
    "dX_conv3_5x5_s2": ((8, 48, 160, 256, 96, 320, 128, 1, 2, 5, 2, 2), None),     # 4 classes: 9 / 6 / 6 / 4 taps
    "deconv2_pair_px": ((8, 48, 160, 386, 96, 320, 64, 1, 2, 4, 1, 1), 960),
}


@pytest.mark.parametrize("name", sorted(CONV_BENCH))
def test_conv_bench_launches(driver, name):
    args, items = CONV_BENCH[name]
    lengths = conv_lengths(*args)
    if items is not None:
        assert len(lengths) == items
    check(driver, lengths)


def test_unequal_classes_and_k_slices(driver):
    lengths = conv_lengths(8, 48, 160, 256, 96, 320, 128, 1, 2, 5, 2, 2)
    assert sorted(set(lengths)) == [32, 48, 72]
    check(driver, lengths)
    check(driver, conv_lengths(8, 12, 40, 512, 6, 20, 1024, 0, 2, 3, 0, 0, ksplit=4))   # conv6 cut in 4 K slices
    check(driver, conv_lengths(2, 6, 10, 1024, 6, 10, 1024, 0, 1, 3, 1, 1, ksplit=3))


@pytest.mark.parametrize("shape", [(8, 96, 320, 64, 128, 2, 5, 2, 2), (8, 48, 160, 128, 256, 2, 5, 2, 2),
                                   (8, 48, 160, 256, 256, 1, 3, 1, 1), (8, 24, 80, 256, 512, 2, 3, 0, 0),
                                   (8, 6, 20, 1024, 1024, 1, 3, 1, 1), (2, 16, 24, 128, 64, 1, 3, 1, 1)])
def test_wgrad_launches(driver, shape):
    # dW of conv2, conv3, conv3_1, conv4, conv6_1 (P = dL/dy: rows = C_out) and a small test shape
    N, Ho, Wo, Ci, Co, s, k, pt, pl = shape
    check(driver, wgrad_lengths(N, Ho, Wo, Co, Ci, s, k, pt, pl))


@pytest.mark.parametrize("lengths", [[5], [1] * 7, [72] * 120, [72] * 132, [72] * 133, [18] * 300, [3] * 500,
                                     [0, 8, 0, 16] * 50, [9, 6, 6, 4] * 70, [17] * 263, [8] * 264])
def test_synthetic(driver, lengths):
    check(driver, lengths)


def test_small_grid(driver):
    for grid in (1, 2, 7):
        check(driver, [20, 3, 8, 9, 30], grid=grid)
        check(driver, [11] * 23, grid=grid, chunk=3)


def test_balance_on_the_bench_tail(driver):
    # conv3: 960 items of 100 K blocks (25 taps x 4 channel blocks); 6 DP waves (792 items) and 168 items over
    # 132 CTAs: 7.27 item-times in all instead of the 8 of a plain round robin
    lengths = conv_lengths(*CONV_BENCH["conv3"][0])
    assert set(lengths) == {100}
    used, dp_items, per = check(driver, lengths)
    assert used and dp_items == 6 * GRID
    load = [sum(k1 - k0 for (_, k0, k1) in segs) for segs in per]
    assert max(load) <= 6 * 100 + -(-168 * 100 // GRID) + CHUNK - 1


def test_which_launches_take_a_stream_k_tail(driver):
    # long K loops and a part-filled last wave: stream-K (conv3 7.27 waves, conv4_1 3.64, dX of conv5 -> 1026 ch)
    assert check(driver, conv_lengths(*CONV_BENCH["conv3"][0]))[0]
    assert check(driver, conv_lengths(8, 24, 80, 512, 24, 80, 512, 0, 1, 3, 1, 1))[0]
    assert check(driver, conv_lengths(8, 24, 80, 256, 12, 40, 1026, 0, 2, 4, 1, 1))[0]
    # unequal classes (9 / 6 / 6 / 4 taps): the ranges make up for the unequal DP loads
    assert check(driver, conv_lengths(*CONV_BENCH["dX_conv3_5x5_s2"][0]))[0]
    # round robin: K loops no longer than a chunk (nothing to cut), short K loops of the 2-channel contractions,
    # a last wave that is nearly full (conv5: 120 items), long DP waves beside a short tail (conv2: 14.55 waves)
    assert not check(driver, [7] * 7680)[0]
    assert not check(driver, conv_lengths(8, 96, 320, 2, 48, 160, 2, 0, 2, 4, 1, 1))[0]
    assert not check(driver, conv_lengths(*CONV_BENCH["conv5"][0]))[0]
    assert not check(driver, conv_lengths(*CONV_BENCH["conv2"][0]))[0]
    # unequal classes with 4 / 2 / 2 / 1 taps x 16 channel blocks (dX of conv4, +=): round robin hands every CTA
    # one item of each class over the 4 waves (144 K blocks); two DP waves load the CTAs with 48 to 96 of them,
    # and the 59 per CTA of the tail on top of the heaviest would end later than round robin
    assert not check(driver, conv_lengths(8, 12, 40, 512, 24, 80, 512, 1, 2, 3, 1, 1))[0]
