"""Index model of the A fragments and the G split of csrc/tc_wgrad.cu, executed on the CPU.

The weight-gradient kernel takes its A operand (rows of P) from registers: each consumer thread loads its tf32
fragment straight from the raw P box, which TMA writes in the 128-byte swizzle.  Its B operand (G) is split
into hi / lo planes written transposed into shared memory.  Inside each 8-pixel K step the pixels are
permuted (positions 0-3 = pixels 0, 2, 4, 6, positions 4-7 = pixels 1, 3, 5, 7) so that the fragment loads are
free of bank conflicts.  The result is only right if the fragments and the G planes agree on that order, and
fast only if the loads really are conflict-free; no GPU is needed to check either.  The index expressions are
taken from the source and evaluated here, so the model cannot drift from the kernel silently."""
import os
import re

import pytest

CSRC = os.path.join(os.path.dirname(__file__), "..", "unflow_b200", "csrc")
SRC = open(os.path.join(CSRC, "tc_wgrad.cu")).read()
COMMON = open(os.path.join(CSRC, "tc_common.cuh")).read()


def grab(pattern, text=SRC):
    m = re.search(pattern, text, re.S)
    assert m, pattern
    return m.groups() if len(m.groups()) > 1 else m.group(1)


def const(name, text):
    return int(grab(r"constexpr int %s = ([0-9]+);" % name, text))


def c_expr(expr):
    """A C integer expression over non-negative ints as Python (integer division)."""
    return compile(expr.replace("/", "//"), expr, "eval")


KP, NTHREADS = const("KP", SRC), const("NTHREADS", SRC)
BM = const("BM", COMMON)
SW128 = c_expr(grab(r"unsigned sw128_offset\(int r, int k\) \{\s*return \(unsigned\)\((.+?)\);\s*\}", COMMON))

# consumer: accumulator / A rows of a thread, its P box, the channel in that box, the fragment load
CONSUMER = SRC[SRC.index("consumers: G split"):]
ROW0 = c_expr(grab(r"const int row0 = (.+?);", CONSUMER))
A_BOX = c_expr(grab(r"const float \*a = split\(\) \+ (.+?);", CONSUMER))
A_CH = c_expr(grab(r"const int ch = (.+?);", CONSUMER))
A_PX, A_C = (c_expr(e) for e in grab(r"a\[sw128_offset\((.+?), (.+?)\) / 4\]", CONSUMER))

# split_transpose: loop, row / K group of an item, source offsets, destination column
SPLIT = SRC[SRC.index("split_transpose(const float *raw"):]
SPLIT = SPLIT[:SPLIT.index("\n}\n")]
S_J = c_expr(grab(r"for \(int j = 0; j < (.+?); \+\+j\)", SPLIT))
S_I = c_expr(grab(r"const int i = (.+?);", SPLIT))
S_R, S_C = (c_expr(e) for e in grab(r"const int r = (.+?), c = (.+?);", SPLIT))
S_SRC = c_expr(grab(r"const float \*src = raw \+ (.+?);", SPLIT))
S_OFFS = [int(x) for x in grab(r"make_float4\(src\[(\d+)\], src\[(\d+)\], src\[(\d+)\], src\[(\d+)\]\)", SPLIT)]
S_DST = c_expr(grab(r"sw128_offset\(r, (.+?)\)", SPLIT))

BNS = (32, 64, 128)


def sw128(r, k):
    return eval(SW128, {}, dict(r=r, k=k))


def tma_swizzled_box():
    """float offset in a 1024-byte aligned box of 32 px x 32 ch written with CU_TENSOR_MAP_SWIZZLE_128B ->
    (pixel, channel): 16-byte chunk j of the 128-byte row px lands at chunk j ^ (px % 8)."""
    return {px * 32 + 4 * ((c // 4) ^ (px % 8)) + c % 4: (px, c) for px in range(32) for c in range(32)}


def fragment_loads():
    """Every A fragment load of both consumer warpgroups: (cw, warp, lane, k, e) -> float offset in the raw slot.
    The hardware fixes what the register holds: A[row + 8 (e & 1)][K position 8k + lane % 4 + 4 (e >> 1)]."""
    out = {}
    for cw in range(2):
        for ct in range(128):
            lane = ct % 32
            row0 = eval(ROW0, {}, dict(cw=cw, ct=ct, lane=lane))
            box = eval(A_BOX, {}, dict(row0=row0))
            ch = eval(A_CH, {}, dict(row0=row0))
            for k in range(KP // 8):
                for e in range(4):
                    v = dict(k=k, lane=lane, e=e, ch=ch)
                    off = sw128(eval(A_PX, {}, v), eval(A_C, {}, v))
                    assert off % 4 == 0
                    out[cw, ct // 32, lane, k, e] = (box + off // 4, row0 + 8 * (e & 1), 8 * k + lane % 4 + 4 * (e >> 1))
    return out


def g_planes(BN):
    """The G split of both warpgroups: (G row n, K position) -> pixel, and the float offsets its lanes read."""
    ROWS = BN // 2
    kpos_px, reads = {}, {}
    for cw in range(2):
        row0 = cw * ROWS
        for ct in range(128):
            for j in range(eval(S_J, {}, dict(ROWS=ROWS))):
                i = eval(S_I, {}, dict(ct=ct, j=j))
                r = eval(S_R, {}, dict(row0=row0, i=i, ROWS=ROWS))
                c = eval(S_C, {}, dict(i=i, ROWS=ROWS))
                src = eval(S_SRC, {}, dict(r=r, c=c))
                dst = sw128(r, eval(S_DST, {}, dict(c=c)))
                assert dst % 16 == 0
                for comp, o in enumerate(S_OFFS):
                    f = src + o                                    # raw G: [group][32 px][32 ch], unswizzled
                    grp, px, ch = f // 1024, f % 1024 // 32, f % 32
                    assert 32 * grp + ch == r, (BN, cw, ct, j)
                    # element comp of the float4 at dst: row r, K position of that byte offset
                    off = dst + 4 * comp
                    row, kp = off // 128, None
                    for kk in range(KP):
                        if sw128(row, kk) == off:
                            kp = kk
                    assert row == r and kp is not None
                    assert (r, kp) not in kpos_px, "K position written twice"
                    kpos_px[r, kp] = px
                    reads[cw, ct // 32, j, comp, ct % 32] = f
    return kpos_px, reads


def test_consumer_layout_matches_the_launch():
    assert NTHREADS == 384 and BM == 128 and KP == 32
    assert "split_transpose<BN / 2>(raw + C::G_RAW / 4, sp + C::B_HI, sp + C::B_LO, cw * (BN / 2), ct)" in SRC


@pytest.mark.parametrize("BN", BNS)
def test_fragments_read_what_the_g_split_puts_at_their_k_position(BN):
    kpos_px, _ = g_planes(BN)
    assert len(kpos_px) == BN * KP
    perm = [kpos_px[0, kp] for kp in range(KP)]
    assert sorted(perm) == list(range(KP))
    for n in range(BN):
        assert [kpos_px[n, kp] for kp in range(KP)] == perm, "every G row in the same K order"
    # the permutation stays inside each 8-pixel K step
    assert all(perm[kp] // 8 == kp // 8 for kp in range(KP))
    box = tma_swizzled_box()
    seen = set()
    for (cw, w, lane, k, e), (off, row, kp) in fragment_loads().items():
        pbox, (px, ch) = off // 1024, box[off % 1024]
        assert 32 * pbox + ch == row, "fragment row"
        assert px == perm[kp], "fragment pixel (cw %d warp %d lane %d k %d e %d)" % (cw, w, lane, k, e)
        seen.add((row, kp))
    assert seen == {(r, kp) for r in range(BM) for kp in range(KP)}


def test_fragment_loads_are_bank_conflict_free():
    loads = fragment_loads()
    for cw in range(2):
        for w in range(4):
            for k in range(KP // 8):
                for e in range(4):
                    banks = {loads[cw, w, lane, k, e][0] % 32 for lane in range(32)}
                    assert len(banks) == 32, (cw, w, k, e)


@pytest.mark.parametrize("BN", BNS)
def test_g_split_reads_are_bank_conflict_free(BN):
    # a warp reads 32 consecutive G rows (channels) of one pixel; at BN = 32 a warpgroup splits only 16 rows,
    # so a warp reads 16 rows of two pixels 32 floats apart: two lanes per bank, in any K order
    want = 32 if BN // 2 >= 32 else 16
    _, reads = g_planes(BN)
    keys = {key[:4] for key in reads}
    for key in keys:
        banks = {reads[key + (lane,)] % 32 for lane in range(32)}
        assert len(banks) == want, (BN, key)
