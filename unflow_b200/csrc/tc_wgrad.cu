// tc_wgrad.cu -- weight gradients of the conv / deconv stacks on the Hopper tensor cores (wgmma, 3xTF32: P split
// in registers, G split in shared memory; fp32 register accumulation, split-K).
//
// Replaces the library weight-gradient kernels behind tf.gradients of slim.conv2d /
// slim.conv2d_transpose (reference src/e2eflow/core/flownet.py:166-233, :89-155; train.py:151-152)
// and the two 3x-wide operand copies each of them needed.
//
//   dW[r][t][c] += sum over pixels p of  P[p][r] * G[stride * p + d_t][c]          (zero outside G)
//
//   convolution   y = conv(x, W):     P = dL/dy (rows r = C_out), G = x   (cols c = C_in),  d_t = k - pad
//   transposed    y = deconv(x, W):   P = x     (rows r = C_in),  G = dL/dy (cols c = C_out), stride 2
//
// GEMM view per work item: M = 128 rows of P's channels, N = BN channels of G, K = pixels.  NHWC
// memory has the channels contiguous and the contraction index (pixels) across rows.  TMA brings boxes of 32
// pixels x 32 channels as they lie in memory: P's in the 128-byte swizzle, G's unswizzled.  The A operand (P)
// comes from registers, so it needs no transpose: each thread loads its tf32 A fragment straight from the raw
// P box and splits it there.  The B operand (G) is read by wgmma from shared memory, K-major only: the
// consumers split it into hi / lo planes written TRANSPOSED (row = channel, 32 pixels per 128-byte row,
// 128-byte swizzle).  No transposed copy of any activation exists in global memory.
//
// K order.  A sum over pixels does not depend on their order, and the fragment row of a lane is fixed by the
// hardware.  With the natural order the 32 lanes of a fragment load hit only 16 banks of the swizzled box, so
// inside each 8-pixel K step k the K positions 0-3 hold the pixels 8k + 0, 2, 4, 6 and positions 4-7 the pixels
// 8k + 1, 3, 5, 7: fragment columns t and t + 4 (t = lane % 4) read pixels 8k + 2t and 8k + 2t + 1, and every
// fragment load is conflict-free.  The G planes are written in the same order
// (tests/test_tc_wgrad_fragment_model_cpu.py checks both).
//
// Work item = (pixel chunk, 128-row block, BN-column block); the BN columns are BN/32 consecutive
// (tap, 32-channel group) pairs, so a layer with few input channels fills the tile with several taps at
// once (conv2: 64 channels -> two taps per block).  A chunk is a run of 32-pixel K blocks sized so that the
// grid has a few waves of items; items of one chunk are adjacent in the schedule, so the chunk's
// activations are read from HBM once and re-read from L2.  The last items are cut into K ranges spread evenly
// over the grid (tc_schedule.h); each range ends in the same red.add epilogue.
//   warp 0           TMA into the raw ring: per K block 4 boxes of P (32 px x 32 ch each) and BN/32 boxes of G
//                    (element stride = the conv stride, tap offset in the start coordinate, zero fill outside)
//   warpgroups 1, 2  each splits + transposes half of the G tile from a raw slot into a split slot; then (after
//                    a barrier over both, since both read all of G), per 8-pixel K step, each thread loads its
//                    A fragment of P (rows r, r + 8 of the warpgroup's 64) from the raw slot and splits it in
//                    registers, and the warpgroup issues wgmma m64nBNk8 with A from registers:
//                    lo*hi + hi*lo + hi*hi, one commit group per K step, two fragment sets alternating (as in
//                    tc_conv.cu).  A warp frees the raw slot once it has loaded its last fragment from it, and
//                    the split slot once every MMA group on it has completed.  Every 8 K blocks the wgmma
//                    accumulator is added to fp32 registers (see tc_conv.cu, "Accuracy"); at the end of the
//                    item: red.global.add into dW.  A warpgroup whose 64 rows all lie at or past R only splits
//                    its half of G: no fragments, no wgmma, no epilogue.
// dW is accumulated with fp32 atomics (split-K partial sums from several CTAs): the caller zeroes
// it; the order of the additions, hence the last bits, vary from run to run.
#include "tc_common.cuh"

namespace unflow {
namespace tcw {

using namespace unflow::tc;

constexpr int NTHREADS = 384;       // warpgroup 0: TMA (warp 0); warpgroups 1-2: split + MMA + epilogue
constexpr int KP = 32;              // pixels per K block

struct WgradParams {
  int N, Hp, Wp;                    // pixel grid of the plain operand P
  int TW, TH, TN;                   // pixel box of one K block, TW*TH*TN == 32
  int tiles_x, tiles_y, tiles_n;    // boxes covering the grid
  int n_ptiles, kc, n_chunks;       // K blocks in total / per chunk, chunks
  int R, C;                         // rows (channels of P) / columns (channels of G) of dW
  int cgroups, vgroups;             // 32-channel groups of G per tap; (tap, group) pairs = "virtual" column groups
  int r_blocks, c_blocks, taps, kw;  // c_blocks: blocks of BN/32 consecutive virtual groups
  int chunk;                        // K blocks per wgmma accumulation (tc::g_chunk)
  long long *dbg;                   // role timers of CTA 0 (unflow_tc_conv_debug), or nullptr
  int stride, stride_x, pad_t, pad_l;   // stride_x = 1 in the row-window form (x stride inside the tensor map)
  float *dw;
  long long pitch_r, pitch_t;       // dW[r * pitch_r + t * pitch_t + c]
  SkSchedule sk;                    // the segments of each CTA (tc_schedule.h): every one ends in red.add
};

// Two rings.  Raw slot (TMA): [P raw] [G raw], per 32-channel group [32 px][32 ch]; the P boxes in the 128-byte
// swizzle (the A fragments are loaded from them), the G boxes unswizzled (the transposing split reads them with
// conflict-free scalar loads).  Split slot (consumers -> wgmma): [G hi] [G lo] (K-major, 128-byte swizzle).  A raw
// slot is free once both warpgroups have split its G and loaded their last A fragment from it; a split slot only
// when the MMAs of both warpgroups on it are done.  Two split slots let split(k + 1) run while MMA(k) reads the
// other one; the rest of shared memory holds raw slots, so TMA runs several K blocks ahead of the consumers.
// Every part is a multiple of 4 KB.
//   BN = 128: 2 x 32 KB split + 5 x 32 KB raw;  BN = 64: 2 x 16 KB + 8 x 24 KB;  BN = 32: 2 x 8 KB + 8 x 20 KB
template <int BN>
struct Cfg {
  static constexpr int G_BYTES = BN * KP * 4;
  static constexpr int B_HI = 0;
  static constexpr int B_LO = B_HI + G_BYTES;
  static constexpr int SPLIT_BYTES = B_LO + G_BYTES;
  static constexpr int SPLIT_STAGES = 2;
  static constexpr int G_RAW = A_BYTES;                     // within a raw slot
  static constexpr int RAW_BYTES = A_BYTES + G_BYTES;
  static constexpr int RAW0 = SPLIT_STAGES * SPLIT_BYTES;   // first raw slot
  static constexpr int FIXED = RAW0 + 1024 /*alignment slack*/ + 256 /*barriers*/;
  static constexpr int RAW_STAGES = (SMEM_LIMIT - FIXED) / RAW_BYTES < 8 ? (SMEM_LIMIT - FIXED) / RAW_BYTES : 8;
  static constexpr int SMEM_BYTES = FIXED + RAW_STAGES * RAW_BYTES;
  static_assert(RAW_STAGES >= 3, "TMA at least two K blocks ahead of the split");
  static_assert(SMEM_BYTES <= SMEM_LIMIT, "over the shared memory of a block");
  static_assert(8 * (2 * RAW_STAGES + SPLIT_STAGES) <= 256, "barriers");
};

struct Item {
  int chunk, rb, cb;
};
__device__ __forceinline__ Item decode_item(const WgradParams &p, int it) {
  Item w;
  w.cb = it % p.c_blocks; it /= p.c_blocks;
  w.rb = it % p.r_blocks; it /= p.r_blocks;
  w.chunk = it;
  return w;
}
__device__ __host__ __forceinline__ int chunk_len(const WgradParams &p, int chunk) {
  const int k0 = chunk * p.kc;
  return (k0 + p.kc <= p.n_ptiles) ? p.kc : p.n_ptiles - k0;
}
// K blocks of work item `it` (the schedule's item length)
__device__ __host__ __forceinline__ int item_len(const WgradParams &p, int it) {
  return chunk_len(p, it / (p.r_blocks * p.c_blocks));
}

// Fragment sets of the consumer, as in tc_conv.cu: K step k of a K block uses set k % FRAG_SETS and is one wgmma
// group; a set is rewritten once wait_group FRAG_SETS - 1 has retired the group that read it, and after the wait
// of K step FRAG_SETS - 1 only groups of the current K block can still run.
constexpr int FRAG_SETS = 2;
static_assert((KP / 8) % FRAG_SETS == 0 && FRAG_SETS <= KP / 8, "fragment sets per K block");

// raw [group][32 px][32 ch] tile -> rows [row0, row0 + rows) of the transposed hi / lo tiles, one float4 of
// 4 K positions per item.  K positions 4c .. 4c + 3 hold the pixels 8 (c / 2) + c % 2 + {0, 2, 4, 6} (the K
// order of the header).  Consecutive threads take consecutive rows (conflict-free reads and swizzled writes).
template <int ROWS>
__device__ __forceinline__ void split_transpose(const float *raw, unsigned char *hi, unsigned char *lo, int row0, int ct) {
#pragma unroll
  for (int j = 0; j < ROWS * 8 / 128; ++j) {
    const int i = ct + 128 * j;
    const int r = row0 + i % ROWS, c = i / ROWS;
    const float *src = raw + (r >> 5) * 1024 + (8 * (c >> 1) + (c & 1)) * 32 + (r & 31);
    const float4 v = make_float4(src[0], src[64], src[128], src[192]), h = tf32_hi4(v);
    const unsigned o = sw128_offset(r, 4 * c);
    *reinterpret_cast<float4 *>(hi + o) = h;
    *reinterpret_cast<float4 *>(lo + o) = sub4(v, h);
  }
}

template <int BN>
__global__ void __launch_bounds__(NTHREADS, 1)
tc_wgrad_kernel(const __grid_constant__ CUtensorMap mapP, const __grid_constant__ CUtensorMap mapG,
                const __grid_constant__ WgradParams p) {
  using C = Cfg<BN>;
  constexpr int R = BN / 2;
  constexpr int GROUPS = BN / 32;
  extern __shared__ unsigned char smem_raw[];
  const unsigned base = (s32(smem_raw) + 1023u) & ~1023u;
  unsigned char *gbase = smem_raw + (base - s32(smem_raw));
  const unsigned bars = base + C::RAW0 + C::RAW_STAGES * C::RAW_BYTES;
  auto raw_full = [&](int s) { return bars + 8u * s; };                           // raw slot s loaded
  auto raw_empty = [&](int s) { return bars + 8u * (C::RAW_STAGES + s); };        // raw slot s split by both
  auto split_empty = [&](int s) { return bars + 8u * (2 * C::RAW_STAGES + s); };  // MMAs of both on split slot s done

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp-uniform: see tc_conv.cu

  if (threadIdx.x == 0) {
    for (int s = 0; s < C::RAW_STAGES; ++s) {
      mbar_init(raw_full(s), 1);
      mbar_init(raw_empty(s), 8);      // one arrive per consumer warp
    }
    for (int s = 0; s < C::SPLIT_STAGES; ++s) mbar_init(split_empty(s), 8);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapP) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapG) : "memory");
  }
  __syncthreads();

  // registers: 40 for warpgroup 0, 232 for the consumers, inside the role branches (see tc_conv.cu)
  if (warp < 4) setmaxnreg_dec<40>();
  if (warp == 0) {
    // ===================== TMA producer (whole warp converged, one elected lane issues) =====================
    int s = 0;
    unsigned ph = 0;
    long long t_wait = 0, t_all = clock64();
    const SegmentWalk walk = segment_walk(p.sk);
    for (int q = 0; q < walk.n_seg; ++q) {
      const Segment sg = segment_at(p.sk, walk, q);
      const Item w = decode_item(p, sg.item);
      int gch[GROUPS], gdx[GROUPS], gdy[GROUPS];           // per column group: channel, tap offset
#pragma unroll
      for (int j = 0; j < GROUPS; ++j) {
        const int v = w.cb * GROUPS + j;
        if (v < p.vgroups) {
          const int tap = v / p.cgroups, ky = tap / p.kw;
          gch[j] = (v - tap * p.cgroups) * 32; gdy[j] = ky - p.pad_t; gdx[j] = tap - ky * p.kw - p.pad_l;
        } else {
          gch[j] = p.cgroups * 32; gdx[j] = gdy[j] = 0;    // past the last group: channels >= C, TMA zero fill
        }
      }
      const int k0 = w.chunk * p.kc, k1 = sg.k1 < 0 ? chunk_len(p, w.chunk) : sg.k1;
      for (int kb = k0 + sg.k0; kb < k0 + k1; ++kb) {
        int q = kb;
        const int px = (q % p.tiles_x) * p.TW; q /= p.tiles_x;
        const int py = (q % p.tiles_y) * p.TH; q /= p.tiles_y;
        const int pn = q * p.TN;
        { const long long t0 = clock64(); mbar_wait(raw_empty(s), ph ^ 1u); t_wait += clock64() - t0; }
        const unsigned st = base + C::RAW0 + s * C::RAW_BYTES;
        if (elect_one()) {
          mbar_expect_tx(raw_full(s), (unsigned)C::RAW_BYTES);
#pragma unroll
          for (int j = 0; j < BM / 32; ++j)       // channels past R are TMA zero fill
            tma_4d(st + j * 4096, &mapP, raw_full(s), w.rb * BM + 32 * j, px, py, pn);
#pragma unroll
          for (int j = 0; j < GROUPS; ++j)
            tma_4d(st + C::G_RAW + j * 4096, &mapG, raw_full(s), gch[j], p.stride_x * px + gdx[j],
                   p.stride * py + gdy[j], pn);
        }
        __syncwarp();
        if (++s == C::RAW_STAGES) { s = 0; ph ^= 1u; }
      }
    }
    if (p.dbg && blockIdx.x == 0 && lane == 0) { p.dbg[0] = t_wait; p.dbg[1] = clock64() - t_all; }
  } else if (warp >= 4) {
    // ===================== consumers: G split, A fragments, wgmma, red.add into dW =====================
    setmaxnreg_inc<232>();
    const int cw = (warp >> 2) - 1;                  // rows [64 cw, 64 cw + 64) of the 128-row block
    const int ct = threadIdx.x - 128 * (cw + 1);
    const int row0 = 64 * cw + 16 * (ct >> 5) + (lane >> 2);     // this thread's accumulator / A rows: row0, row0 + 8
    const int col0 = 2 * (lane & 3);
    // K blocks consumed so far: K block n uses raw slot n % RAW_STAGES and split slot n % SPLIT_STAGES
    unsigned n = 0;
    long long t_wait = 0, t_split = 0, t_all = clock64();   // role timers: blocked on a loaded raw / free split slot
    // G of K block n from its raw slot into its split slot (this warpgroup's half); the split slot is complete
    // (both halves, fenced for wgmma) after the barrier.  The raw slot stays in use: the caller frees it.
    auto split = [&]() {
      const unsigned rs = n % C::RAW_STAGES, rph = (n / C::RAW_STAGES) & 1u;
      const unsigned ss = n % C::SPLIT_STAGES, sph = (n / C::SPLIT_STAGES) & 1u;
      { const long long t0 = clock64(); mbar_wait(raw_full(rs), rph); t_wait += clock64() - t0; }
      { const long long t0 = clock64(); mbar_wait(split_empty(ss), sph ^ 1u); t_split += clock64() - t0; }
      const float *raw = reinterpret_cast<const float *>(gbase + C::RAW0 + rs * C::RAW_BYTES);
      unsigned char *sp = gbase + ss * C::SPLIT_BYTES;
      split_transpose<BN / 2>(raw + C::G_RAW / 4, sp + C::B_HI, sp + C::B_LO, cw * (BN / 2), ct);
      fence_proxy_async();
      named_bar_sync(1, 256);                        // both halves of G are split
      return raw;
    };
    float sum[R], acc[R];
    unsigned a_hi[FRAG_SETS][4], a_lo[FRAG_SETS][4];
    const SegmentWalk walk = segment_walk(p.sk);
    for (int q = 0; q < walk.n_seg; ++q) {
      // a segment starts on a chunk boundary of its item: its chunks are the item's chunks
      const Segment sg = segment_at(p.sk, walk, q);
      const Item w = decode_item(p, sg.item);
      const int iters = (sg.k1 < 0 ? chunk_len(p, w.chunk) : sg.k1) - sg.k0;
      if (w.rb * BM + 64 * cw >= p.R) {
        // all 64 rows of this warpgroup are past R: its half of G only (the other warpgroup reads it)
        for (int it = 0; it < iters; ++it) {
          split();
          __syncwarp();
          if (lane == 0) {
            mbar_arrive(raw_empty(n % C::RAW_STAGES));
            mbar_arrive(split_empty(n % C::SPLIT_STAGES));
          }
          ++n;
        }
        continue;
      }
#pragma unroll
      for (int c = 0; c < R; ++c) sum[c] = 0.f;
      // chunks and their K blocks as in tc_conv.cu: inside a chunk the only waits are wait_group FRAG_SETS - 1
      // before a fragment set is rewritten; acc is read only at the chunk's end, behind wait_group 0
      for (int c0 = 0; c0 < iters; c0 += p.chunk) {
        const int c1 = c0 + p.chunk < iters ? c0 + p.chunk : iters;
        int pending = -1;                            // split slot whose MMAs may still be running
        for (int it = c0; it < c1; ++it) {
          // this thread's A rows row0, row0 + 8 lie in P box row0 / 32, as channels row0 % 32 and row0 % 32 + 8
          const float *a = split() + (row0 >> 5) * 1024;
          const int ch = row0 & 31;
          const unsigned rs = n % C::RAW_STAGES, ss = n % C::SPLIT_STAGES;
          const unsigned st = base + ss * C::SPLIT_BYTES;
          const unsigned long long b_hi = wgmma_desc_k128(st + C::B_HI), b_lo = wgmma_desc_k128(st + C::B_LO);
#pragma unroll
          for (int k = 0; k < KP / 8; ++k) {         // K step = 8 pixels = 32 bytes: +2 in 16-byte units
            unsigned (&hi)[4] = a_hi[k % FRAG_SETS], (&lo)[4] = a_lo[k % FRAG_SETS];
            wgmma_wait<FRAG_SETS - 1>();             // the group that last read this set has completed
            fence_regs(acc);
            if (k == FRAG_SETS - 1) {
              // every group of the previous K block has completed: free its split slot
              __syncwarp();
              if (pending >= 0 && lane == 0) mbar_arrive(split_empty(pending));
            }
            // the tf32 A fragment of the K step: a[e] = P[row0 + 8 (e & 1)][pixel 8k + 2 (lane % 4) + (e >> 1)]
            // (the K order of the header), from the swizzled raw box, split in registers
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float x = a[sw128_offset(8 * k + 2 * (lane & 3) + (e >> 1), ch + 8 * (e & 1)) / 4];
              const float h = tf32_rna_fast(x);
              hi[e] = __float_as_uint(h);
              lo[e] = __float_as_uint(x - h);
            }
            if (k == KP / 8 - 1) {
              // the last fragment of this K block is loaded: the raw slot is free as far as this warp goes
              __syncwarp();
              if (lane == 0) mbar_arrive(raw_empty(rs));
            }
            wgmma_fence();
            const unsigned long long adv = (unsigned long long)(2 * k);
            Wgmma<BN>::mma_rs(acc, lo, b_hi + adv, (it - c0 | k) != 0);
            Wgmma<BN>::mma_rs(acc, hi, b_lo + adv, 1);
            Wgmma<BN>::mma_rs(acc, hi, b_hi + adv, 1);
            wgmma_commit();
          }
          pending = ss;
          ++n;
        }
        // chunk end: all MMAs have completed; free the last split slot and add the chunk to the fp32 sum
        wgmma_wait<0>();
        fence_regs(acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(split_empty(pending));
#pragma unroll
        for (int c = 0; c < R; ++c) sum[c] += acc[c];
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = w.rb * BM + row0 + 8 * h;
        if (r >= p.R) continue;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int col = 8 * j + col0;              // column within the BN block; col, col + 1 share a group
          const int v = w.cb * GROUPS + col / 32;
          if (v >= p.vgroups) continue;
          const int tap = v / p.cgroups, c = (v - tap * p.cgroups) * 32 + (col & 31);
          float *dst = p.dw + (long long)r * p.pitch_r + (long long)tap * p.pitch_t + c;
          if (c < p.C) red_add_f32(dst, sum[4 * j + 2 * h]);
          if (c + 1 < p.C) red_add_f32(dst + 1, sum[4 * j + 2 * h + 1]);
        }
      }
    }
    if (p.dbg && blockIdx.x == 0 && threadIdx.x == 128) {
      p.dbg[2] = t_wait; p.dbg[3] = clock64() - t_all; p.dbg[4] = t_split;
      p.dbg[5] = C::RAW_STAGES; p.dbg[6] = C::SPLIT_STAGES;
    }
  }
}

template <int BN>
static int launch(const CUtensorMap &mP, const CUtensorMap &mG, WgradParams &p, cudaStream_t stream) {
  using C = Cfg<BN>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(tc_wgrad_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
    if (e != cudaSuccess) { set_error("tc_wgrad: cannot opt in to %d bytes of shared memory: %s", C::SMEM_BYTES, cudaGetErrorString(e)); return UNFLOW_ECUDA; }
    attr_set = true;
  }
  // one CTA per SM: DP waves of whole items, then the last items' K blocks spread over the grid where that pays
  make_sk_schedule(p.sk, p.n_chunks * p.r_blocks * p.c_blocks, kNumSMs, p.chunk,
                   [&](int it) { return item_len(p, it); });
  tc_wgrad_kernel<BN><<<p.sk.grid, NTHREADS, C::SMEM_BYTES, stream>>>(mP, mG, p);
  count_launch();
  return check_launch("tc_wgrad_kernel");
}

static int launch_bn(int BN, const CUtensorMap &mP, const CUtensorMap &mG, WgradParams &p, cudaStream_t stream) {
  if (BN == 128) return launch<128>(mP, mG, p, stream);
  if (BN == 64) return launch<64>(mP, mG, p, stream);
  return launch<32>(mP, mG, p, stream);
}

// the K-block pixel box: TW*TH*TN == 32 exactly (rows past the tensor are TMA zero fill), fewest boxes
static void choose_box(WgradParams &p) {
  long long best = -1;
  for (int TW = 1; TW <= 32; TW *= 2)
    for (int TH = 1; TW * TH <= 32; TH *= 2) {
      const int TN = 32 / (TW * TH);
      const long long tiles = (long long)((p.Wp + TW - 1) / TW) * ((p.Hp + TH - 1) / TH) * ((p.N + TN - 1) / TN);
      if (best < 0 || tiles < best || (tiles == best && TW > p.TW)) {
        best = tiles; p.TW = TW; p.TH = TH; p.TN = TN;
      }
    }
  p.tiles_x = (p.Wp + p.TW - 1) / p.TW; p.tiles_y = (p.Hp + p.TH - 1) / p.TH; p.tiles_n = (p.N + p.TN - 1) / p.TN;
  p.n_ptiles = p.tiles_x * p.tiles_y * p.tiles_n;
}

static int make_plan(WgradParams &p, int &BN, int N, int Hp, int Wp, int R, int C, int stride, int kh, int kw,
                     int pad_t, int pad_l) {
  UNFLOW_REQUIRE(N > 0 && Hp > 0 && Wp > 0 && R > 0 && C > 0, "tc_wgrad: bad extents");
  UNFLOW_REQUIRE(stride == 1 || stride == 2, "tc_wgrad: stride must be 1 or 2");
  UNFLOW_REQUIRE(kh > 0 && kw > 0 && kh * kw <= 64, "tc_wgrad: at most 64 taps");
  p.N = N; p.Hp = Hp; p.Wp = Wp; p.R = R; p.C = C; p.chunk = g_chunk; p.dbg = g_dbg;
  p.taps = kh * kw; p.kw = kw; p.stride = p.stride_x = stride; p.pad_t = pad_t; p.pad_l = pad_l;
  choose_box(p);
  p.cgroups = (C + 31) / 32; p.vgroups = p.taps * p.cgroups;
  BN = p.vgroups >= 4 ? 128 : (p.vgroups >= 2 ? 64 : 32);
  p.r_blocks = (R + BM - 1) / BM; p.c_blocks = (p.vgroups + BN / 32 - 1) / (BN / 32);
  // split K so that the grid has ~6 waves of items; at least 8 K blocks per item
  const long long tiles = (long long)p.r_blocks * p.c_blocks;
  long long want = (6ll * kNumSMs + tiles - 1) / tiles;
  if (want < 1) want = 1;
  int kc = (int)((p.n_ptiles + want - 1) / want);
  if (kc < 8) kc = p.n_ptiles < 8 ? p.n_ptiles : 8;
  p.kc = kc; p.n_chunks = (p.n_ptiles + kc - 1) / kc;
  UNFLOW_REQUIRE(tiles * p.n_chunks < (1ll << 30), "tc_wgrad: too many work items");
  return UNFLOW_OK;
}

}  // namespace tcw
}  // namespace unflow

using namespace unflow;

// Debug / test hook (host only): [TW, TH, TN, tiles_x, tiles_y, tiles_n, n_ptiles, kc, n_chunks, r_blocks,
// c_blocks, BN, taps, cgroups, vgroups]; returns 15 or -1.
extern "C" int unflow_tc_wgrad_plan(int N, int Hp, int Wp, int R, int C, int stride, int kh, int kw, int pad_t,
                                    int pad_l, int *out) {
  tcw::WgradParams p{};
  int BN = 0;
  if (tcw::make_plan(p, BN, N, Hp, Wp, R, C, stride, kh, kw, pad_t, pad_l) || !out) return -1;
  const int v[15] = {p.TW, p.TH, p.TN, p.tiles_x, p.tiles_y, p.tiles_n, p.n_ptiles, p.kc, p.n_chunks, p.r_blocks,
                     p.c_blocks, BN, p.taps, p.cgroups, p.vgroups};
  for (int i = 0; i < 15; ++i) out[i] = v[i];
  return 15;
}

extern "C" int unflow_tc_wgrad(const float *P, int N, int Hp, int Wp, int R, long long p_pitch, const float *G,
                               int Hg, int Wg, int C, long long g_pitch, float *dw, long long pitch_r,
                               long long pitch_t, int stride, int kh, int kw, int pad_t, int pad_l, void *stream) {
  UNFLOW_REQUIRE(P && G && dw, "tc_wgrad: null pointer");
  UNFLOW_REQUIRE(Hg > 0 && Wg > 0, "tc_wgrad: bad extents");
  UNFLOW_REQUIRE(p_pitch % 4 == 0 && g_pitch % 4 == 0 && p_pitch >= R && g_pitch >= C,
                 "tc_wgrad: channel pitches must be multiples of 4 floats");
  UNFLOW_REQUIRE(((uintptr_t)P & 15) == 0 && ((uintptr_t)G & 15) == 0, "tc_wgrad: P and G must be 16-byte aligned");
  tcw::WgradParams p{};
  int BN = 0;
  int rc = tcw::make_plan(p, BN, N, Hp, Wp, R, C, stride, kh, kw, pad_t, pad_l);
  if (rc) return rc;
  p.dw = dw; p.pitch_r = pitch_r; p.pitch_t = pitch_t;
  CUtensorMap mP, mG;
  {
    cuuint64_t dims[4] = {(cuuint64_t)R, (cuuint64_t)Wp, (cuuint64_t)Hp, (cuuint64_t)N};
    cuuint64_t strides[3] = {(cuuint64_t)p_pitch * 4, (cuuint64_t)p_pitch * 4 * Wp, (cuuint64_t)p_pitch * 4 * Wp * Hp};
    cuuint32_t box[4] = {32, (cuuint32_t)p.TW, (cuuint32_t)p.TH, (cuuint32_t)p.TN};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    rc = tc::encode(&mP, P, 4, dims, strides, box, estr);   // 128-byte swizzle: conflict-free A fragment loads
    if (rc) return rc;
  }
  {
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)Wg, (cuuint64_t)Hg, (cuuint64_t)N};
    cuuint64_t strides[3] = {(cuuint64_t)g_pitch * 4, (cuuint64_t)g_pitch * 4 * Wg, (cuuint64_t)g_pitch * 4 * Wg * Hg};
    cuuint32_t box[4] = {32, (cuuint32_t)(p.TW * stride), (cuuint32_t)(p.TH * stride), (cuuint32_t)p.TN};
    cuuint32_t estr[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
    rc = tc::encode(&mG, G, 4, dims, strides, box, estr, CU_TENSOR_MAP_SWIZZLE_NONE);
    if (rc) return rc;
  }
  return tcw::launch_bn(BN, mP, mG, p, (cudaStream_t)stream);
}

// Weight gradient of the row-window form of the first layers (see unflow_tc_conv_window):
//     dw[co][ky][kx*Cp + c] += sum_p gpre[p][co] * xp[n, stride*y + ky - pad_t, window of output column x][kx*Cp + c]
extern "C" int unflow_tc_wgrad_window(const float *P, int N, int Ho, int Wo, int R, long long p_pitch,
                                      const float *xp, int H, int Wp, int Cp, float *dw, int kh, int stride,
                                      int pad_t, void *stream) {
  UNFLOW_REQUIRE(P && xp && dw, "tc_wgrad_window: null pointer");
  UNFLOW_REQUIRE(Cp == 4 || Cp == 8 || Cp == 16, "tc_wgrad_window: padded channel count must be 4, 8 or 16");
  UNFLOW_REQUIRE(p_pitch % 4 == 0 && p_pitch >= R, "tc_wgrad_window: bad pitch");
  UNFLOW_REQUIRE(((uintptr_t)P & 15) == 0 && ((uintptr_t)xp & 15) == 0, "tc_wgrad_window: pointers must be 16-byte aligned");
  UNFLOW_REQUIRE(H > 0 && Wp >= stride * (Wo - 1) + 8, "tc_wgrad_window: the padded row must hold the last 8-pixel window");
  const int win = 8 * Cp;
  tcw::WgradParams p{};
  int BN = 0;
  int rc = tcw::make_plan(p, BN, N, Ho, Wo, R, win, stride, kh, 1, pad_t, 0);
  if (rc) return rc;
  p.stride_x = 1;
  p.dw = dw; p.pitch_r = (long long)kh * win; p.pitch_t = win;
  CUtensorMap mP, mG;
  {
    cuuint64_t dims[4] = {(cuuint64_t)R, (cuuint64_t)Wo, (cuuint64_t)Ho, (cuuint64_t)N};
    cuuint64_t strides[3] = {(cuuint64_t)p_pitch * 4, (cuuint64_t)p_pitch * 4 * Wo, (cuuint64_t)p_pitch * 4 * Wo * Ho};
    cuuint32_t box[4] = {32, (cuuint32_t)p.TW, (cuuint32_t)p.TH, (cuuint32_t)p.TN};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    rc = tc::encode(&mP, P, 4, dims, strides, box, estr);   // 128-byte swizzle: conflict-free A fragment loads
    if (rc) return rc;
  }
  {
    cuuint64_t dims[4] = {(cuuint64_t)win, (cuuint64_t)Wo, (cuuint64_t)H, (cuuint64_t)N};
    cuuint64_t strides[3] = {(cuuint64_t)stride * Cp * 4, (cuuint64_t)Wp * Cp * 4, (cuuint64_t)Wp * Cp * 4 * H};
    cuuint32_t box[4] = {32, (cuuint32_t)p.TW, (cuuint32_t)(p.TH * stride), (cuuint32_t)p.TN};
    cuuint32_t estr[4] = {1, 1, (cuuint32_t)stride, 1};
    rc = tc::encode(&mG, xp, 4, dims, strides, box, estr, CU_TENSOR_MAP_SWIZZLE_NONE);
    if (rc) return rc;
  }
  return tcw::launch_bn(BN, mP, mG, p, (cudaStream_t)stream);
}
