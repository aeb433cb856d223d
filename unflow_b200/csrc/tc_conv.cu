// tc_conv.cu -- the conv / deconv stacks of FlowNet on the Hopper tensor cores: a wgmma implicit GEMM with
// the 3xTF32 operand split done inside the kernel (activations: in registers, per K step; weights: hi / lo
// planes made once per step).
//
// Replaces the library convolutions behind slim.conv2d / slim.conv2d_transpose
// (reference src/e2eflow/core/flownet.py:166-233, _flownet_upconv :89-155) for the forward pass
// and the input gradient.  One kernel serves every case because the host describes a layer as a
// list of TAPS over an iteration space of output positions:
//
//     out[n, s_out*iy + py, s_out*ix + px, co] (+)= act( bias[co] +
//         sum_{t in taps(class)} sum_ci  in[n, s_in*iy + dy_t, s_in*ix + dx_t, ci] * W[t.widx][co][ci] )
//
//   * convolution, stride 1 or 2 (TF SAME padding = the tap offsets): one class, s_out = 1;
//   * transposed convolution with stride 2 (deconvN forward, input gradient of a stride-2 conv):
//     four output-parity classes, each a stride-1 gather over its own subset of the taps;
//   * input gradient of a stride-1 convolution: one class, mirrored tap offsets.
//
// GEMM view per tile: M = 128 output positions (a TW x TH x TN box of one class), N = BN output
// channels, K = taps x Cin walked in blocks of 32 channels (one 128-byte swizzle row of fp32).
//
// Pipeline (one CTA per SM, persistent over work items, warp-specialised, 3 warpgroups):
//   warp 0           TMA producer: per K block one 4-D box of the ACTIVATIONS as they lie in HBM (fp32,
//                    NHWC, any channel pitch -- e.g. a channel slice of a concat buffer; image borders,
//                    the TF SAME padding and the channel tail are TMA zero fill, stride 2 is the tensor
//                    map's element stride) plus the hi and lo planes of the weights, into a ring of stages
//                    sized from the opt-in shared-memory limit.
//   warpgroups 1, 2  consumers, 64 tile rows each: per K step of 8 channels each thread loads its tf32 A
//                    fragment (4 floats) straight from the swizzled fp32 tile and splits it in registers
//                    (hi = tf32(x), lo = x - hi), then the warpgroup issues wgmma m64nBNk8 kind tf32 with A
//                    from registers, three per K step: lo*hi' + hi*lo' + hi*hi', fp32 accumulators in
//                    registers.  One wgmma group per K step; two fragment sets alternate, so a K step's MMAs
//                    run while the next one's fragment is loaded.  The stage is released once the next K
//                    block's first group has been issued and every group of this one has completed.
//                    The K loop is cut into CHUNKS of 8 K blocks (tc_common.cuh: CHUNK): every chunk starts a
//                    fresh wgmma accumulator that is then added to a second fp32 register accumulator with
//                    round to nearest (see "Accuracy"); after the last chunk: bias + leaky ReLU (or += for
//                    gradient accumulation) -> stores straight into the destination (which may be a channel
//                    slice of a concat buffer, with stride 2 for the transposed classes).
// The activations are read from HBM once, as fp32; no [hi,hi,lo] operand copies exist, no layout
// conversion, no separate bias / activation pass.
//
// Schedule (tc_schedule.h): whole work items round robin for all but the last one or two waves; the K blocks of
// the rest are spread over the grid so that every CTA ends at the same time (where that shortens the launch), and
// a tile run by several CTAs is finished by the warp that completes it last (sk_fixup).
//
// Accuracy: hi carries 11 significant bits, lo the next 11; the dropped lo*lo' term and the
// truncation of lo are ~2^-22 relative.  What limits a long tensor-core accumulation is not the
// split but the accumulator itself: the MMA adds with truncation, a bias of a fraction of an ulp
// per instruction that grows LINEARLY with K.  Summing chunks of 256 K elements in fp32 registers
// (round to nearest) bounds it.
#include <algorithm>

#include "tc_conv_plan.cuh"

namespace unflow {
namespace tc {

constexpr int NTHREADS = 384;    // warpgroup 0: TMA producer (warp 0); warpgroups 1-2: consumers

// Stage: [A raw fp32] [B hi] [B lo].  Each 1024-byte aligned (128-byte swizzle atoms).  The ring fills the opt-in
// limit: BN = 128: 4 x 48 KB, BN = 64: 7 x 32 KB, BN = 32: 8 x 24 KB (capped at 8).
template <int BN>
struct Cfg {
  static constexpr int B_BYTES = BN * BK * 4;
  static constexpr int STAGE_BYTES = A_BYTES + 2 * B_BYTES;
  static constexpr int B_OFF = A_BYTES;
  static constexpr int FIXED = 1024 /*alignment slack*/ + 256 /*barriers*/;
  static constexpr int STAGES = (SMEM_LIMIT - FIXED) / STAGE_BYTES < 8 ? (SMEM_LIMIT - FIXED) / STAGE_BYTES : 8;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + FIXED;
  static_assert(STAGES >= 2, "at least two stages");
  static_assert(SMEM_BYTES <= SMEM_LIMIT, "over the shared memory of a block");
};
// Fragment sets of the consumer (hi + lo tf32 A fragments of one K step each): K step k of a K block uses set
// k % FRAG_SETS and is one wgmma group, so a set is rewritten once wait_group FRAG_SETS - 1 has retired the group
// that read it.  Two sets divide the 4 K steps of a block, keep the set index a compile-time constant and leave
// the MMAs of one K step in flight while the next one's fragment is loaded and split.  Four sets compile as
// cleanly but were not faster (DESIGN.md §3.8).  After the wait of K step FRAG_SETS - 1, only groups of the
// current K block can still run: that is where the previous block's stage is released.
constexpr int FRAG_SETS = 2;
static_assert((BK / 8) % FRAG_SETS == 0 && FRAG_SETS <= BK / 8, "fragment sets per K block");

struct TileCoord {
  int cls, n0, iy0, ix0, nb;
};
// Tile order, fastest first: column block, output-parity class, M tile.  The classes of a transposed layer all
// read the same input box: next to each other in the schedule they run at the same time on neighbouring SMs and
// share it in L2 (with the class outermost every class would sweep the whole input again).
__device__ __forceinline__ TileCoord decode_tile(const ConvParams &p, int tile) {
  TileCoord t;
  t.nb = tile % p.n_blocks; tile /= p.n_blocks;
  t.cls = tile % p.n_classes; tile /= p.n_classes;
  t.ix0 = (tile % p.tiles_x) * p.TW; tile /= p.tiles_x;
  t.iy0 = (tile % p.tiles_y) * p.TH; tile /= p.tiles_y;
  t.n0 = tile * p.TN;
  return t;
}

// Work item = (tile, K slice).  Layers with few tiles and long K loops (conv6 / conv6_1) cut the K loop of a tile
// into p.ksplit slices that run at the same time on different CTAs (adjacent in the schedule: the slice index is
// the fastest).
struct Work {
  TileCoord t;
  int it0, iters;       // first K block (tap * kblocks + channel block) and count of this item
};
__device__ __host__ __forceinline__ void work_range(const ConvParams &p, int cls, int ks, int &it0, int &iters) {
  const int total = (p.class_start[cls + 1] - p.class_start[cls]) * p.kblocks;
  const int per = (total + p.ksplit - 1) / p.ksplit;
  it0 = ks * per;
  iters = total - it0 < per ? total - it0 : per;
  if (iters < 0) iters = 0;
}
__device__ __forceinline__ Work decode_work(const ConvParams &p, int w) {
  Work k;
  const int tile = w / p.ksplit, ks = w - tile * p.ksplit;
  k.t = decode_tile(p, tile);
  work_range(p, k.t.cls, ks, k.it0, k.iters);
  return k;
}
// K blocks of work item w (the schedule's item length)
__device__ __host__ __forceinline__ int work_len(const ConvParams &p, int w) {
  const int tile = w / p.ksplit, ks = w - tile * p.ksplit;
  int it0, iters;
  work_range(p, (tile / p.n_blocks) % p.n_classes, ks, it0, iters);
  return iters;
}

// Stream-K fixup of a tile that several CTAs run one K range each (tc_schedule.h).  Bias, leaky ReLU and += are
// not linear in the partial sums, so one of them has to see the whole sum.  Per consumer warp (a warp owns 16 rows
// of the tile and nothing else): every segment stores its partial to its slot -- 2g for the first segment of CTA g,
// 2g + 1 for its last -- then, after a warp barrier, one lane counts the warp on the item's counter with an
// acq_rel atomic (release: the warp's stores are visible before the count; acquire: the last arriver sees every
// other partial).  The warp that completes the count adds all partials in segment order (a fixed order: the result
// does not depend on who arrives last), resets the counter for the next launch and runs the epilogue.  No CTA waits
// for another.
__device__ __forceinline__ unsigned atom_add_acq_rel(unsigned *addr, unsigned v) {
  unsigned old;
  asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], %2;" : "=r"(old) : "l"(addr), "r"(v) : "memory");
  return old;
}
template <int R>
__device__ __forceinline__ bool sk_fixup(const ConvParams &p, const Segment &sg, int len, int cwarp, int lane,
                                         float (&sum)[R]) {
  const SkSchedule &s = p.sk;
  const int g = blockIdx.x, j = sg.sk;
  auto slot_of = [&](int c) { return 2 * c + (s.sk_item[c] == j ? 0 : 1); };
  auto part = [&](int slot) { return p.sk_part + ((long long)(slot * 8 + cwarp) * R) * 32 + lane; };
  {
    float *dst = part(slot_of(g));
#pragma unroll
    for (int c = 0; c < R; ++c) __stcg(dst + 32 * c, sum[c]);
  }
  __syncwarp();
  // the CTAs whose ranges meet item j: ga holds its first K block, gb its last; empty ranges in between run nothing
  int ga = g, gb = g;
  while (ga > 0 && (s.sk_item[ga] > j || (s.sk_item[ga] == j && s.sk_k[ga] > 0))) --ga;
  while (s.sk_item[gb + 1] < j || (s.sk_item[gb + 1] == j && s.sk_k[gb + 1] < len)) ++gb;
  auto empty = [&](int c) { return s.sk_item[c] == s.sk_item[c + 1] && s.sk_k[c] == s.sk_k[c + 1]; };
  unsigned n = 0;
  for (int c = ga; c <= gb; ++c) n += empty(c) ? 0u : 1u;
  unsigned *cnt = p.sk_count + 8 * j + cwarp;
  unsigned old = 0;
  if (lane == 0) old = atom_add_acq_rel(cnt, 1u);
  old = __shfl_sync(0xffffffffu, old, 0);
  if (old != n - 1) return false;
  __syncwarp();                                 // lane 0's acquire before every lane's loads
  if (lane == 0) *cnt = 0u;
#pragma unroll
  for (int c = 0; c < R; ++c) sum[c] = 0.f;
  for (int c = ga; c <= gb; ++c) {
    if (empty(c)) continue;
    const float *src = part(slot_of(c));
#pragma unroll
    for (int e = 0; e < R; ++e) sum[e] += __ldcg(src + 32 * e);
  }
  return true;
}

// ------------------------------------------------------------------------------------------
// The kernel
// ------------------------------------------------------------------------------------------
template <int BN>
__global__ void __launch_bounds__(NTHREADS, 1)
tc_conv_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapBhi,
               const __grid_constant__ CUtensorMap mapBlo, const __grid_constant__ ConvParams p) {
  using C = Cfg<BN>;
  constexpr int R = BN / 2;              // accumulator registers per thread (64 x BN per warpgroup)
  extern __shared__ unsigned char smem_raw[];
  const unsigned base = (s32(smem_raw) + 1023u) & ~1023u;          // 128B swizzle atoms need 1024 B alignment
  unsigned char *gbase = smem_raw + (base - s32(smem_raw));
  const unsigned bars = base + C::STAGES * C::STAGE_BYTES;
  auto full = [&](int s) { return bars + 8u * s; };                   // stage s landed (TMA)
  auto empty = [&](int s) { return bars + 8u * (C::STAGES + s); };    // stage s consumed (MMAs of both consumers done)

  // warp index made warp-uniform for ptxas: with a plain threadIdx.x >> 5 it cannot prove the role branch is uniform
  // across a warpgroup, treats the wgmma code as divergent and waits for every MMA before issuing the next (C7518)
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < C::STAGES; ++s) {
      mbar_init(full(s), 1);
      mbar_init(empty(s), 8);          // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapBhi) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapBlo) : "memory");
  }
  __syncthreads();

  // registers: 40 for warpgroup 0, 232 for the consumers (40 * 128 + 232 * 256 <= 64K).  Each setmaxnreg sits
  // inside its role's branch: ptxas ignores one in code shared by both roles (C7507).
  if (warp < 4) setmaxnreg_dec<40>();
  if (warp == 0) {
    // ===================== TMA producer (whole warp converged, one elected lane issues) =====================
    int s = 0;
    unsigned ph = 0;
    long long t_wait = 0, t_all = clock64();          // role timers: cycles blocked on the barrier / in total
    const unsigned a_box_bytes = (unsigned)(p.TW * p.TH * p.TN) * BK * 4u;
    const SegmentWalk walk = segment_walk(p.sk);
    for (int q = 0; q < walk.n_seg; ++q) {
      const Segment sg = segment_at(p.sk, walk, q);
      const Work wk = decode_work(p, sg.item);
      const TileCoord t = wk.t;
      const int x0 = p.s_in_x * t.ix0, y0 = p.s_in_y * t.iy0;
      int ti = p.class_start[t.cls] + (wk.it0 + sg.k0) / p.kblocks, kc = (wk.it0 + sg.k0) % p.kblocks;
      const int k1 = sg.k1 < 0 ? wk.iters : sg.k1;
      for (int it = sg.k0; it < k1; ++it) {
        const Tap tap = p.taps[ti];
        { const long long t0 = clock64(); mbar_wait(empty(s), ph ^ 1u); t_wait += clock64() - t0; }
        const unsigned st = base + s * C::STAGE_BYTES;
        if (elect_one()) {
          mbar_expect_tx(full(s), a_box_bytes + 2u * C::B_BYTES);
          tma_4d(st, &mapA, full(s), kc * BK, x0 + tap.dx, y0 + tap.dy, t.n0);
          if (p.pair_px) {      // rows [0, BN/2): the weights of class px = 0, [BN/2, BN): px = 1; no tap: zero fill
            const int w0 = tap.widx < 0 ? (1 << 20) : tap.widx, w1 = tap.widx2 < 0 ? (1 << 20) : tap.widx2;
            tma_3d(st + C::B_OFF, &mapBhi, full(s), kc * BK, 0, w0);
            tma_3d(st + C::B_OFF + C::B_BYTES / 2, &mapBhi, full(s), kc * BK, 0, w1);
            tma_3d(st + C::B_OFF + C::B_BYTES, &mapBlo, full(s), kc * BK, 0, w0);
            tma_3d(st + C::B_OFF + C::B_BYTES + C::B_BYTES / 2, &mapBlo, full(s), kc * BK, 0, w1);
          } else {
            tma_3d(st + C::B_OFF, &mapBhi, full(s), kc * BK, t.nb * BN, tap.widx);
            tma_3d(st + C::B_OFF + C::B_BYTES, &mapBlo, full(s), kc * BK, t.nb * BN, tap.widx);
          }
        }
        __syncwarp();
        if (++s == C::STAGES) { s = 0; ph ^= 1u; }
        if (++kc == p.kblocks) { kc = 0; ++ti; }
      }
    }
    if (p.dbg && blockIdx.x == 0 && lane == 0) { p.dbg[0] = t_wait; p.dbg[1] = clock64() - t_all; }
  } else if (warp >= 4) {
    // ===================== consumers: A fragments, split, wgmma, epilogue =====================
    setmaxnreg_inc<232>();
    const int cw = (warp >> 2) - 1;                  // consumer warpgroup: tile rows [64 cw, 64 cw + 64)
    const int ct = threadIdx.x - 128 * (cw + 1);     // thread within the warpgroup
    const int row0 = 64 * cw + 16 * (ct >> 5) + (lane >> 2);     // this thread's accumulator / A rows: row0, row0 + 8
    const int col0 = 2 * (lane & 3);
    const int per_img = p.TW * p.TH;
    int s = 0;
    unsigned ph = 0;
    long long t_wait = 0, t_all = clock64();
    float sum[R], acc[R];
    unsigned a_hi[FRAG_SETS][4], a_lo[FRAG_SETS][4];
    const SegmentWalk walk = segment_walk(p.sk);
    for (int q = 0; q < walk.n_seg; ++q) {
      // a segment starts on a chunk boundary of its item: its chunks are the item's chunks
      const Segment sg = segment_at(p.sk, walk, q);
      const Work wk = decode_work(p, sg.item);
      const TileCoord t = wk.t;
      const int k1 = sg.k1 < 0 ? wk.iters : sg.k1, iters = k1 - sg.k0;
#pragma unroll
      for (int c = 0; c < R; ++c) sum[c] = 0.f;
      // Outer loop over chunks, inner loop over the K blocks of a chunk.  Inside a chunk the only waits are
      // wait_group FRAG_SETS - 1 before a fragment set is rewritten, so the MMAs run while the next K step's
      // fragment is loaded and split; the accumulator is read only after the inner loop, behind wait_group 0.
      // A read of acc inside the inner loop would make ptxas wait for every MMA group (C7517).
      for (int c0 = 0; c0 < iters; c0 += p.chunk) {
        const int c1 = c0 + p.chunk < iters ? c0 + p.chunk : iters;
        int pending = -1;                            // stage whose MMAs may still be running
        for (int it = c0; it < c1; ++it) {
          { const long long t0 = clock64(); mbar_wait(full(s), ph); t_wait += clock64() - t0; }
          const float *a = reinterpret_cast<const float *>(gbase + s * C::STAGE_BYTES);
          const unsigned st = base + s * C::STAGE_BYTES;
          const unsigned long long b_hi = wgmma_desc_k128(st + C::B_OFF), b_lo = wgmma_desc_k128(st + C::B_OFF + C::B_BYTES);
#pragma unroll
          for (int k = 0; k < BK / 8; ++k) {         // K step = 8 tf32 = 32 bytes: +2 in 16-byte units
            unsigned (&hi)[4] = a_hi[k % FRAG_SETS], (&lo)[4] = a_lo[k % FRAG_SETS];
            wgmma_wait<FRAG_SETS - 1>();             // the group that last read this set has completed
            fence_regs(acc);
            if (k == FRAG_SETS - 1) {
              // every group of the previous K block has completed: free its stage
              __syncwarp();
              if (pending >= 0 && lane == 0) mbar_arrive(empty(pending));
            }
            // this thread's tf32 A fragment of the K step, straight from the swizzled fp32 tile (the 8 rows of a
            // quarter-warp lie in 8 different 16-byte chunks: no bank conflicts), split in registers
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float x = a[sw128_offset(row0 + 8 * (e & 1), 8 * k + (lane & 3) + 4 * (e >> 1)) / 4];
              const float h = tf32_rna_fast(x);
              hi[e] = __float_as_uint(h);
              lo[e] = __float_as_uint(x - h);
            }
            wgmma_fence();
            const unsigned long long adv = (unsigned long long)(2 * k);
            Wgmma<BN>::mma_rs(acc, lo, b_hi + adv, (it - c0 | k) != 0);
            Wgmma<BN>::mma_rs(acc, hi, b_lo + adv, 1);
            Wgmma<BN>::mma_rs(acc, hi, b_hi + adv, 1);
            wgmma_commit();
          }
          pending = s;
          if (++s == C::STAGES) { s = 0; ph ^= 1u; }
        }
        // chunk end: all MMAs have completed; free the last stage and add the chunk to the fp32 sum
        wgmma_wait<0>();
        fence_regs(acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(empty(pending));
#pragma unroll
        for (int c = 0; c < R; ++c) sum[c] += acc[c];
      }
      // a tile split over CTAs: only the last warp to finish its part goes on, with the whole sum (K slices add
      // their parts with red.add anyway)
      if (p.ksplit == 1 && sg.sk >= 0 && (sg.k0 > 0 || k1 < wk.iters) &&
          !sk_fixup(p, sg, wk.iters, warp - 4, lane, sum))
        continue;
      // ---- epilogue: rows row0 and row0 + 8, columns 8j + col0 (+1) ----
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = row0 + 8 * h;
        const int tn = row / per_img, rem = row - tn * per_img;
        const int ty = rem / p.TW, tx = rem - ty * p.TW;
        const int n = t.n0 + tn, iy = t.iy0 + ty, ix = t.ix0 + tx;
        if (!(tn < p.TN && n < p.N && iy < p.Hit && ix < p.Wit)) continue;
        const int oy = p.s_out * iy + p.class_py[t.cls];
        float *const orow = p.out + ((long long)n * p.Hout + oy) * p.Wout * p.out_pitch;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int col = 8 * j + col0;
          // pair_px: the two column halves of the tile are the two px classes of the same (<= 64) output channels
          const int half = p.pair_px && col >= BN / 2 ? 1 : 0;
          const int c = p.pair_px ? col - half * (BN / 2) : t.nb * BN + col;
          const int ox = p.s_out * ix + (p.pair_px ? half : p.class_px[t.cls]);
          if (c >= p.Cout) continue;
          float *dst = orow + (long long)ox * p.out_pitch + c;
          float v0 = sum[4 * j + 2 * h], v1 = sum[4 * j + 2 * h + 1];
          const bool two = c + 1 < p.Cout;
          if (p.ksplit > 1) {        // K slice: add the raw partial sums (the launcher zeroed the output unless it accumulates anyway)
            if (iters > 0) {
              red_add_f32(dst, v0);
              if (two) red_add_f32(dst + 1, v1);
            }
            continue;
          }
          if (p.bias) {              // scalar loads: a bias is a view into the flat variable buffer at any 4-byte offset
            v0 += __ldg(p.bias + c);
            if (two) v1 += __ldg(p.bias + c + 1);
          }
          if (p.act) {
            v0 = v0 > 0.f ? v0 : p.slope * v0;
            v1 = v1 > 0.f ? v1 : p.slope * v1;
          }
          if (two) {                 // c is even and the pitch a multiple of 4: 8-byte aligned
            float2 *o = reinterpret_cast<float2 *>(dst);
            if (p.accumulate) { const float2 old = *o; v0 += old.x; v1 += old.y; }
            *o = make_float2(v0, v1);
          } else {                   // channel tail
            *dst = p.accumulate ? *dst + v0 : v0;
          }
        }
      }
    }
    if (p.dbg && blockIdx.x == 0 && threadIdx.x == 128) {
      p.dbg[2] = t_wait; p.dbg[3] = clock64() - t_all; p.dbg[5] = C::STAGES;
      p.dbg[8] = (long long)p.sk_count; p.dbg[9] = 8 * 2 * kSkMaxGrid;    // the fixup counters (tests)
    }
  }
}

// ------------------------------------------------------------------------------------------
// Weight planes: w -> hi = tf32(w), lo = w - hi, in the K-major layout [tap][R][Cp] the kernel's
// B operand wants (R = output channels of the GEMM, C = contraction channels, Cp = C rounded up to
// 4 so every TMA stride is a multiple of 16 bytes; the tail is zero).  The source is read through
// strides, so the same kernel serves [Cout][kh][kw][Cin] and [Cin][kh][kw][Cout] variables and
// their transposes (forward / input-gradient operands).  Runs once per optimiser step per layer.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
wsplit_kernel(const float *__restrict__ w, float *__restrict__ hi, float *__restrict__ lo, int taps, int R,
              int C, int Cp, long long s_t, long long s_r, long long s_c, int r_fast) {
  __shared__ float tile[32][33];
  const int t = blockIdx.z;
  const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;      // 32 x 8
  for (int k = ty; k < 32; k += 8) {
    // r_fast: consecutive threads walk r (the source is contiguous in r), else they walk c
    const int r = r0 + (r_fast ? tx : k), c = c0 + (r_fast ? k : tx);
    float v = 0.f;
    if (r < R && c < C) v = w[t * s_t + r * s_r + c * s_c];
    if (r_fast) tile[tx][k] = v; else tile[k][tx] = v;          // tile[r][c]
  }
  __syncthreads();
  for (int k = ty; k < 32; k += 8) {
    const int r = r0 + k, c = c0 + tx;
    if (r < R && c < Cp) {
      const float v = tile[k][tx];
      const float h = tf32_rna(v);
      const long long o = ((long long)t * R + r) * Cp + c;
      hi[o] = h;
      lo[o] = v - h;
    }
  }
}

// ------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------
static int floordiv(int a, int b) { return (a >= 0) ? a / b : -((-a + b - 1) / b); }

int g_chunk = CHUNK;     // unflow_set_int_option("tc_chunk"): K blocks per wgmma accumulation
long long *g_dbg = nullptr;   // unflow_tc_conv_debug: device buffer of 16 long longs for the role timers of CTA 0

// Stream-K fixup storage, per device, allocated on first use and kept: 2 partial-sum slots per CTA (its first and
// its last segment; a range holds at most two pieces of split tiles) of 128 x BN floats at BN = 128, and one
// counter per SK item (fewer than 2 x grid) and consumer warp, which the last arriver resets to zero.  A launch
// uses them from start to end, so tc_conv launches on one device must run one at a time: on one stream (as every
// caller in this project does), never side by side on two.
static int sk_storage(float **part, unsigned **count) {
  static float *parts[64] = {};
  static unsigned *counts[64] = {};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess && (dev < 0 || dev >= 64)) { set_error("tc_conv: device %d out of range", dev); return UNFLOW_ECUDA; }
  if (e == cudaSuccess && !parts[dev]) {
    // may be first reached inside a graph capture: allocate and zero outside it, on a stream of our own
    cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
    cudaThreadExchangeStreamCaptureMode(&mode);
    float *pp = nullptr;
    unsigned *cc = nullptr;
    cudaStream_t s = nullptr;
    const size_t n_count = 8 * 2 * kSkMaxGrid;
    e = cudaMalloc(&pp, sizeof(float) * 2 * kSkMaxGrid * BM * 128);
    if (e == cudaSuccess) e = cudaMalloc(&cc, sizeof(unsigned) * n_count);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaMemsetAsync(cc, 0, sizeof(unsigned) * n_count, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (s) cudaStreamDestroy(s);
    cudaThreadExchangeStreamCaptureMode(&mode);
    if (e == cudaSuccess) { parts[dev] = pp; counts[dev] = cc; }
    else { cudaFree(pp); cudaFree(cc); }
  }
  if (e != cudaSuccess) { set_error("tc_conv: stream-K storage: %s", cudaGetErrorString(e)); return UNFLOW_ECUDA; }
  *part = parts[dev];
  *count = counts[dev];
  return UNFLOW_OK;
}

template <int BN>
static int launch(const CUtensorMap &mA, const CUtensorMap &mBh, const CUtensorMap &mBl, ConvParams &p,
                  cudaStream_t stream) {
  using C = Cfg<BN>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(tc_conv_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
    if (e != cudaSuccess) { set_error("tc_conv: cannot opt in to %d bytes of shared memory: %s", C::SMEM_BYTES, cudaGetErrorString(e)); return UNFLOW_ECUDA; }
    attr_set = true;
  }
  // one CTA per SM: DP waves of whole items, then the last items' K blocks spread over the grid where that pays
  const int total = p.n_classes * p.tiles_n * p.tiles_y * p.tiles_x * p.n_blocks * p.ksplit;
  make_sk_schedule(p.sk, total, kNumSMs, p.chunk, [&](int w) { return work_len(p, w); });
  if (int rc = sk_storage(&p.sk_part, &p.sk_count)) return rc;
  tc_conv_kernel<BN><<<p.sk.grid, NTHREADS, C::SMEM_BYTES, stream>>>(mA, mBh, mBl, p);
  count_launch();
  return check_launch("tc_conv_kernel");
}

// K slices for a layer with few tiles and long K loops (work items <= half of the SMs): how many
inline int choose_ksplit(const ConvParams &p) {
  const long long items = (long long)p.n_classes * p.tiles_n * p.tiles_y * p.tiles_x * p.n_blocks;
  if (2 * items > kNumSMs) return 1;
  int min_iters = 1 << 30;
  for (int c = 0; c < p.n_classes; ++c) min_iters = std::min(min_iters, (p.class_start[c + 1] - p.class_start[c]) * p.kblocks);
  const long long ks = std::min<long long>(std::min<long long>(kNumSMs / items, 4), std::max(1, min_iters / (4 * p.chunk)));
  return ks < 1 ? 1 : (int)ks;
}

// tile -> kernel: encodes the two weight-plane maps (box = BN rows, or BN / 2 for pair_px) and launches
static int launch_bn(int BN, const CUtensorMap &mA, const float *w_hi, const float *w_lo, const cuuint64_t *wdims,
                     const cuuint64_t *wstrides, ConvParams &p, cudaStream_t stream) {
  CUtensorMap mBh, mBl;
  cuuint32_t box[3] = {(cuuint32_t)BK, (cuuint32_t)(p.pair_px ? BN / 2 : BN), 1};
  cuuint32_t estr[3] = {1, 1, 1};
  int rc = encode(&mBh, w_hi, 3, wdims, wstrides, box, estr);
  if (rc) return rc;
  rc = encode(&mBl, w_lo, 3, wdims, wstrides, box, estr);
  if (rc) return rc;
  if (BN == 128) return launch<128>(mA, mBh, mBl, p, stream);
  if (BN == 64) return launch<64>(mA, mBh, mBl, p, stream);
  return launch<32>(mA, mBh, mBl, p, stream);
}

}  // namespace tc
int set_tc_chunk(int v) { if (v < 1 || v > 64) return 0; tc::g_chunk = v; return 1; }
}  // namespace unflow

using namespace unflow;

extern "C" int unflow_bias_lrelu(float *y, const float *bias, long long pixels, int C, float slope, void *stream);   // bias_act.cu

extern "C" int unflow_tc_wsplit(const float *w, float *w_hi, float *w_lo, int taps, int R, int C, long long s_t,
                                long long s_r, long long s_c, void *stream) {
  UNFLOW_REQUIRE(w && w_hi && w_lo && taps > 0 && R > 0 && C > 0, "tc_wsplit: bad arguments");
  UNFLOW_REQUIRE(taps <= 65535 && (R + 31) / 32 <= 65535, "tc_wsplit: too many taps / rows");
  const int Cp = (C + 3) / 4 * 4;
  dim3 grid((Cp + 31) / 32, (R + 31) / 32, taps);
  tc::wsplit_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(w, w_hi, w_lo, taps, R, C, Cp, s_t, s_r, s_c,
                                                           (s_r == 1 && s_c != 1) ? 1 : 0);
  count_launch();
  return check_launch("tc_wsplit_kernel");
}

// Build the tap / class / tile description of one layer (host only; shared by the launcher and by
// unflow_tc_conv_plan, which lets the CPU tests execute the same plan with plain loops).
static int make_plan(tc::ConvParams &p, int &BN, int N, int Hin, int Win, int Cin, int Hout, int Wout, int Cout,
                     int mode, int stride, int kh, int kw, int pad_t, int pad_l) {
  UNFLOW_REQUIRE(N > 0 && Hin > 0 && Win > 0 && Cin > 0 && Hout > 0 && Wout > 0 && Cout > 0, "tc_conv: bad extents");
  UNFLOW_REQUIRE(mode == 0 || mode == 1, "tc_conv: mode must be 0 (conv) or 1 (transposed)");
  UNFLOW_REQUIRE(stride == 1 || stride == 2, "tc_conv: stride must be 1 or 2");
  UNFLOW_REQUIRE(kh > 0 && kw > 0 && kh * kw <= tc::MAX_TAPS, "tc_conv: at most %d taps", tc::MAX_TAPS);
  p.N = N; p.Cin = Cin; p.Cout = Cout; p.kblocks = (Cin + tc::BK - 1) / tc::BK; p.chunk = tc::g_chunk; p.dbg = tc::g_dbg; p.ksplit = 1;
  p.Hout = Hout; p.Wout = Wout;
  int nt = 0;
  if (mode == 0) {
    p.n_classes = 1; p.s_in_x = p.s_in_y = stride; p.s_out = 1; p.Hit = Hout; p.Wit = Wout;
    p.class_px[0] = p.class_py[0] = 0;
    p.class_start[0] = 0;
    for (int ky = 0; ky < kh; ++ky)
      for (int kx = 0; kx < kw; ++kx) p.taps[nt++] = tc::Tap{(short)(kx - pad_l), (short)(ky - pad_t), ky * kw + kx};
    p.class_start[1] = nt;
  } else {
    UNFLOW_REQUIRE(Hout % stride == 0 && Wout % stride == 0, "tc_conv: transposed output extents must be multiples of the stride");
    p.n_classes = stride * stride; p.s_in_x = p.s_in_y = 1; p.s_out = stride; p.Hit = Hout / stride; p.Wit = Wout / stride;
    int c = 0;
    for (int py = 0; py < stride; ++py)
      for (int px = 0; px < stride; ++px, ++c) {
        p.class_px[c] = (short)px; p.class_py[c] = (short)py;
        p.class_start[c] = nt;
        for (int ky = 0; ky < kh; ++ky) {
          if (((py + pad_t - ky) % stride + stride) % stride) continue;
          for (int kx = 0; kx < kw; ++kx) {
            if (((px + pad_l - kx) % stride + stride) % stride) continue;
            UNFLOW_REQUIRE(nt < tc::MAX_TAPS, "tc_conv: too many taps");
            p.taps[nt++] = tc::Tap{(short)tc::floordiv(px + pad_l - kx, stride),
                                   (short)tc::floordiv(py + pad_t - ky, stride), ky * kw + kx};
          }
        }
      }
    p.class_start[p.n_classes] = nt;
    for (int c2 = 0; c2 < p.n_classes; ++c2)
      UNFLOW_REQUIRE(p.class_start[c2 + 1] > p.class_start[c2], "tc_conv: an output parity class has no taps");
  }
  // tile box: fewest tiles over (TW, TH, TN) with TW*TH*TN <= 128 (ties: the widest rows)
  long long best = -1;
  for (int TW = 1; TW <= p.Wit && TW <= 128; ++TW)
    for (int TH = 1; TH <= p.Hit && TW * TH <= 128; ++TH) {
      int TN = 128 / (TW * TH);
      if (TN > N) TN = N;
      const long long tiles = (long long)((p.Wit + TW - 1) / TW) * ((p.Hit + TH - 1) / TH) * ((N + TN - 1) / TN);
      if (best < 0 || tiles < best || (tiles == best && TW > p.TW)) {
        best = tiles; p.TW = TW; p.TH = TH; p.TN = TN;
      }
    }
  p.tiles_x = (p.Wit + p.TW - 1) / p.TW; p.tiles_y = (p.Hit + p.TH - 1) / p.TH; p.tiles_n = (N + p.TN - 1) / p.TN;
  BN = Cout > 64 ? 128 : (Cout > 32 ? 64 : 32);     // channel tail: TMA zero rows, masked stores
  p.n_blocks = (Cout + BN - 1) / BN;
  const long long total = (long long)p.n_classes * p.tiles_n * p.tiles_y * p.tiles_x * p.n_blocks;
  UNFLOW_REQUIRE(total < (1ll << 30), "tc_conv: too many tiles");
  return UNFLOW_OK;
}

// Narrow transposed layers (33..64 output channels: deconv2, the input gradient of conv2): the two output-parity
// classes px = 0 / 1 of a row class py read overlapping input offsets (k4 s2: dx {0,-1} and {+1,0}; 5x5 s2: {0,-1}
// and {+1,0,-1}): ONE 128-wide tile computes both -- columns [0,64) = the channels of px = 0, [64,128) = those of
// px = 1 -- over the union of the offsets; where only one class has a tap for an offset that half of the weight
// tile is TMA zero fill.  Each activation box is loaded and split once for both classes, and a channel block
// walks fewer K blocks over all classes: k4 s2 12 instead of 16, 5x5 s2 15 instead of 25.
static bool pair_px_plan(tc::ConvParams &p, int &BN, int mode, int stride, int Cout) {
  if (mode != 1 || stride != 2 || p.n_classes != 4) return false;
  if (Cout <= 32 || Cout > 64 || (long long)p.tiles_n * p.tiles_y * p.tiles_x < 2) return false;
  tc::Tap taps[tc::MAX_TAPS];
  int start[3], nt = 0;
  for (int py = 0; py < 2; ++py) {
    start[py] = nt;
    for (int px = 0; px < 2; ++px) {
      const int c = py * 2 + px;                        // make_plan's class order: py outer, px inner
      if (p.class_py[c] != py || p.class_px[c] != px) return false;
      for (int ti = p.class_start[c]; ti < p.class_start[c + 1]; ++ti) {
        const tc::Tap &a = p.taps[ti];
        int e = -1;
        for (int k = start[py]; k < nt; ++k)
          if (taps[k].dx == a.dx && taps[k].dy == a.dy) e = k;
        if (e < 0) {
          if (nt >= tc::MAX_TAPS) return false;
          e = nt++;
          taps[e] = tc::Tap{a.dx, a.dy, -1, -1};
        }
        if (px == 0) taps[e].widx = a.widx; else taps[e].widx2 = a.widx;
      }
    }
  }
  start[2] = nt;
  for (int k = 0; k < nt; ++k) p.taps[k] = taps[k];
  p.n_classes = 2;
  for (int c = 0; c < 3; ++c) p.class_start[c] = start[c];
  p.class_py[0] = 0; p.class_py[1] = 1; p.class_px[0] = p.class_px[1] = 0;
  p.pair_px = 1; p.n_blocks = 1;
  BN = 128;
  return true;
}

// Debug hook: role timers.  `buf` = device memory for 16 long longs (or nullptr to switch off); every following
// tc_conv launch makes CTA 0 write, in clocks: [0] TMA producer blocked on a free stage, [1] its total; [2] the
// first consumer thread blocked on the TMA data, [3] its total, [5] the stages of the ring.
extern "C" int unflow_tc_conv_debug(long long *buf) { tc::g_dbg = buf; return UNFLOW_OK; }

// Debug / test hook: the plan unflow_tc_conv launches, as integers --
// [n_classes, s_in, s_out, Hit, Wit, TW, TH, TN, tiles_x, tiles_y, tiles_n, n_blocks, BN, kblocks, ntaps,
//  class_start[5], (class_px, class_py)[4], (dx, dy, widx)[ntaps], pair_px, widx2[ntaps], ksplit]; returns the
// count written.  pair_px = 1: a narrow transposed layer computes two parity classes per tile (pair_px_plan), and
// widx2 holds the px = 1 class's tap per input offset.  ksplit: the K slices the launcher cuts each tile into when
// the epilogue allows slicing (no bias and no activation, or both on a dense output that is not accumulated into).
extern "C" int unflow_tc_conv_plan(int N, int Hin, int Win, int Cin, int Hout, int Wout, int Cout, int mode,
                                   int stride, int kh, int kw, int pad_t, int pad_l, int *out, int cap) {
  // bits above the first two are ignored, as they always were: callers written when bit 2 asked for the
  // two-parity-classes rewrite get the plan they asked for, which is now the only one
  mode &= 3;
  tc::ConvParams p{};
  int BN = 0;
  if (make_plan(p, BN, N, Hin, Win, Cin, Hout, Wout, Cout, mode, stride, kh, kw, pad_t, pad_l)) return -1;
  if (Cin > 4) pair_px_plan(p, BN, mode, stride, Cout);   // unflow_tc_conv hands Cin <= 4 to conv_fma first
  const int nt = p.class_start[p.n_classes];
  const int need = 15 + 5 + 8 + 3 * nt + 1 + nt + 1;
  if (!out || cap < need) return -need;
  int i = 0;
  const int head[15] = {p.n_classes, p.s_in_y, p.s_out, p.Hit, p.Wit, p.TW, p.TH, p.TN, p.tiles_x, p.tiles_y,
                        p.tiles_n, p.n_blocks, BN, p.kblocks, nt};
  for (int k = 0; k < 15; ++k) out[i++] = head[k];
  for (int k = 0; k < 5; ++k) out[i++] = p.class_start[k];
  for (int k = 0; k < 4; ++k) { out[i++] = p.class_px[k]; out[i++] = p.class_py[k]; }
  for (int k = 0; k < nt; ++k) { out[i++] = p.taps[k].dx; out[i++] = p.taps[k].dy; out[i++] = p.taps[k].widx; }
  out[i++] = p.pair_px;
  for (int k = 0; k < nt; ++k) out[i++] = p.taps[k].widx2;
  out[i++] = tc::choose_ksplit(p);
  return i;
}

// mode 0: y = conv(x, W; stride, TF-SAME offsets pad_t / pad_l)          taps (ky,kx) -> offset (ky-pad_t, kx-pad_l)
// mode 1: y = conv_transpose(x, W; stride, padding pad_t / pad_l)        o = stride*i - pad + k
// The weight planes are [kh*kw][Cout][Cin_p] (see unflow_tc_wsplit); tap index = ky*kw + kx.
extern "C" int unflow_tc_conv(const float *x, int N, int Hin, int Win, int Cin, long long x_pitch,
                              const float *w_hi, const float *w_lo, float *y, int Hout, int Wout, int Cout,
                              long long y_pitch, const float *bias, float slope, int act, int accumulate,
                              int mode, int stride, int kh, int kw, int pad_t, int pad_l, void *stream) {
  UNFLOW_REQUIRE(x && w_hi && w_lo && y, "tc_conv: null pointer");
  UNFLOW_REQUIRE(x_pitch % 4 == 0 && y_pitch % 4 == 0 && x_pitch >= Cin && y_pitch >= Cout,
                 "tc_conv: channel pitches must be multiples of 4 floats");
  UNFLOW_REQUIRE(((uintptr_t)x & 15) == 0 && ((uintptr_t)y & 15) == 0 && ((uintptr_t)w_hi & 15) == 0 &&
                 ((uintptr_t)w_lo & 15) == 0, "tc_conv: x, y and the weight planes must be 16-byte aligned");
  tc::ConvParams p{};
  int BN = 0;
  int rc0 = make_plan(p, BN, N, Hin, Win, Cin, Hout, Wout, Cout, mode, stride, kh, kw, pad_t, pad_l);
  if (rc0) return rc0;
  p.out = y; p.out_pitch = y_pitch;
  p.bias = bias; p.slope = slope; p.act = act; p.accumulate = accumulate;
  // A contraction over at most 4 channels fills one 32-channel K block per tap with 28 zero channels: with 3 MMA
  // passes its useful rate is at most 495 / 3 * 4 / 32 ~ 21 TFLOP/s, below the FMA pipes' 67, and both paths write
  // the same bytes.  Such layers (the flow heads' input gradients, the flow up-sampling deconvs) run in conv_fma.cu.
  if (Cin <= 4) return tc::conv_fma(p, x, Hin, Win, x_pitch, w_hi, w_lo, (cudaStream_t)stream);
  pair_px_plan(p, BN, mode, stride, Cout);
  // K slices (few tiles, long K): partial sums are added into the output, which is zeroed first unless the call
  // accumulates anyway; bias + leaky ReLU then run as unflow_bias_lrelu over the (dense) result.  That pass sees
  // only the sum in y, so a call that accumulates into y and needs it (y += act(bias + conv)) is not sliced.
  const bool post = bias && act;
  if ((!bias && !act) || (post && !accumulate && y_pitch == Cout && Cout % 4 == 0)) p.ksplit = tc::choose_ksplit(p);
  if (p.ksplit > 1 && !accumulate) {
    cudaError_t e = cudaMemset2DAsync(y, (size_t)y_pitch * 4, 0, (size_t)Cout * 4, (size_t)N * Hout * Wout, (cudaStream_t)stream);
    if (e != cudaSuccess) { set_error("tc_conv: memset of the output: %s", cudaGetErrorString(e)); return UNFLOW_ECUDA; }
  }

  CUtensorMap mA;
  {
    cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)Win, (cuuint64_t)Hin, (cuuint64_t)N};
    cuuint64_t strides[3] = {(cuuint64_t)x_pitch * 4, (cuuint64_t)x_pitch * 4 * Win, (cuuint64_t)x_pitch * 4 * Win * Hin};
    cuuint32_t box[4] = {(cuuint32_t)tc::BK, (cuuint32_t)(p.TW * p.s_in_x), (cuuint32_t)(p.TH * p.s_in_y), (cuuint32_t)p.TN};
    cuuint32_t estr[4] = {1, (cuuint32_t)p.s_in_x, (cuuint32_t)p.s_in_y, 1};
    int rc = tc::encode(&mA, x, 4, dims, strides, box, estr);
    if (rc) return rc;
  }
  const int Cp = (Cin + 3) / 4 * 4;
  cuuint64_t wdims[3] = {(cuuint64_t)Cin, (cuuint64_t)Cout, (cuuint64_t)(kh * kw)};
  cuuint64_t wstrides[2] = {(cuuint64_t)Cp * 4, (cuuint64_t)Cp * 4 * Cout};
  const int rc = tc::launch_bn(BN, mA, w_hi, w_lo, wdims, wstrides, p, (cudaStream_t)stream);
  if (rc || p.ksplit == 1 || !post) return rc;
  return unflow_bias_lrelu(y, bias, (long long)N * Hout * Wout, Cout, slope, stream);
}

// First layers (7x7, stride 2, 3 / 6 / 14 input channels): with so few channels a K block of 32
// channels per filter tap would be 90 % zeros.  In a channel-padded image (Cp = 4 / 8 / 16 floats per
// pixel) the kw taps of one filter ROW are contiguous in memory -- 8 pixels x Cp floats -- so the layer
// is run as a convolution with kh "taps" (the filter rows) whose contraction dimension is that
// 8*Cp-float window: the tensor map's x axis counts OUTPUT columns with a stride of `stride` pixels
// (overlapping windows), y keeps the element stride.  The image must be physically zero-padded in x
// (pad_l pixels on the left, enough on the right for the last window) -- out-of-image ROWS are TMA
// zero fill.  Weight planes: [kh][Cout][8*Cp] with column kx*Cp + c (zero for kx >= kw, c >= Cin).
extern "C" int unflow_tc_conv_window(const float *xp, int N, int H, int Wp, int Cp, const float *w_hi,
                                     const float *w_lo, float *y, int Hout, int Wout, int Cout, long long y_pitch,
                                     const float *bias, float slope, int act, int kh, int stride, int pad_t,
                                     void *stream) {
  UNFLOW_REQUIRE(xp && w_hi && w_lo && y, "tc_conv_window: null pointer");
  UNFLOW_REQUIRE(Cp == 4 || Cp == 8 || Cp == 16, "tc_conv_window: padded channel count must be 4, 8 or 16");
  UNFLOW_REQUIRE(y_pitch % 4 == 0 && y_pitch >= Cout, "tc_conv_window: bad output pitch");
  UNFLOW_REQUIRE(((uintptr_t)xp & 15) == 0 && ((uintptr_t)y & 15) == 0 && ((uintptr_t)w_hi & 15) == 0 &&
                 ((uintptr_t)w_lo & 15) == 0, "tc_conv_window: pointers must be 16-byte aligned");
  const int win = 8 * Cp;                              // floats per window = contraction length per filter row
  UNFLOW_REQUIRE(N > 0 && H > 0 && Hout > 0 && Wout > 0 && Wp >= stride * (Wout - 1) + 8,
                 "tc_conv_window: the padded row must hold the last 8-pixel window");
  tc::ConvParams p{};
  int BN = 0;
  int rc0 = make_plan(p, BN, N, H, Wout, win, Hout, Wout, Cout, 0, stride, kh, 1, pad_t, 0);
  if (rc0) return rc0;
  p.s_in_x = 1;                                        // the x stride lives in the tensor map
  p.out = y; p.out_pitch = y_pitch;
  p.bias = bias; p.slope = slope; p.act = act; p.accumulate = 0;
  CUtensorMap mA;
  {
    cuuint64_t dims[4] = {(cuuint64_t)win, (cuuint64_t)Wout, (cuuint64_t)H, (cuuint64_t)N};
    cuuint64_t strides[3] = {(cuuint64_t)stride * Cp * 4, (cuuint64_t)Wp * Cp * 4, (cuuint64_t)Wp * Cp * 4 * H};
    cuuint32_t box[4] = {(cuuint32_t)tc::BK, (cuuint32_t)p.TW, (cuuint32_t)(p.TH * stride), (cuuint32_t)p.TN};
    cuuint32_t estr[4] = {1, 1, (cuuint32_t)stride, 1};
    int rc = tc::encode(&mA, xp, 4, dims, strides, box, estr);
    if (rc) return rc;
  }
  cuuint64_t wdims[3] = {(cuuint64_t)win, (cuuint64_t)Cout, (cuuint64_t)kh};
  cuuint64_t wstrides[2] = {(cuuint64_t)win * 4, (cuuint64_t)win * 4 * Cout};
  return tc::launch_bn(BN, mA, w_hi, w_lo, wdims, wstrides, p, (cudaStream_t)stream);
}
