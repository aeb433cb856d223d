// tc_wgrad.cu -- weight gradients of the conv / deconv stacks on the Hopper tensor cores (wgmma, 3xTF32
// split of BOTH operands in shared memory, fp32 register accumulation, split-K).
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
// memory has the channels contiguous and the contraction index (pixels) across rows, while wgmma reads tf32
// operands K-major only: TMA brings boxes of 32 pixels x 32 channels as they lie in memory, and the split into
// hi / lo writes them TRANSPOSED (row = channel, 32 pixels per 128-byte row, 128-byte swizzle).  No transposed
// copy of any activation exists in global memory.
//
// Work item = (pixel chunk, 128-row block, BN-column block); the BN columns are BN/32 consecutive
// (tap, 32-channel group) pairs, so a layer with few input channels fills the tile with several taps at
// once (conv2: 64 channels -> two taps per block).  A chunk is a run of 32-pixel K blocks sized so that the
// grid has a few waves of items; items of one chunk are adjacent in the schedule, so the chunk's
// activations are read from HBM once and re-read from L2.
//   warp 0           TMA: per K block 4 boxes of P (32 px x 32 ch each) and BN/32 boxes of G (element
//                    stride = the conv stride, tap offset in the start coordinate, zero fill outside)
//   warpgroups 1, 2  each splits + transposes its 64 rows of P and half of the G tile, then (after a barrier
//                    over both, since both read all of G) issues wgmma m64nBNk8 for its 64 rows:
//                    lo*hi + hi*lo + hi*hi per 8-pixel K step; every 8 K blocks the wgmma accumulator is
//                    added to fp32 registers (see tc_conv.cu, "Accuracy"); at the end of the item:
//                    red.global.add into dW
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
};

// Stage: [P raw] [G raw] (TMA, unswizzled: per 32-channel group [32 px][32 ch]) and the split, transposed
// operands [P hi] [P lo] [G hi] [G lo] (K-major, 128-byte swizzle).  Every part is a multiple of 4 KB.
template <int BN>
struct Cfg {
  static constexpr int G_BYTES = BN * KP * 4;
  static constexpr int G_RAW = A_BYTES;
  static constexpr int A_HI = G_RAW + G_BYTES;
  static constexpr int A_LO = A_HI + A_BYTES;
  static constexpr int B_HI = A_LO + A_BYTES;
  static constexpr int B_LO = B_HI + G_BYTES;
  static constexpr int STAGE_BYTES = B_LO + G_BYTES;
  static constexpr int STAGES = (200 * 1024 / STAGE_BYTES) < 8 ? (200 * 1024 / STAGE_BYTES) : 8;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 256;
  static_assert(STAGES >= 2, "at least two stages");
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
__device__ __forceinline__ int chunk_len(const WgradParams &p, int chunk) {
  const int k0 = chunk * p.kc;
  return (k0 + p.kc <= p.n_ptiles) ? p.kc : p.n_ptiles - k0;
}

// raw [group][32 px][32 ch] tile -> rows [row0, row0 + rows) of the transposed hi / lo tiles, one float4 of
// 4 pixels per item; consecutive threads take consecutive rows (conflict-free reads and swizzled writes)
template <int ROWS>
__device__ __forceinline__ void split_transpose(const float *raw, unsigned char *hi, unsigned char *lo, int row0, int ct) {
#pragma unroll
  for (int j = 0; j < ROWS * 8 / 128; ++j) {
    const int i = ct + 128 * j;
    const int r = row0 + i % ROWS, c = i / ROWS;
    const float *src = raw + (r >> 5) * 1024 + (4 * c) * 32 + (r & 31);
    const float4 v = make_float4(src[0], src[32], src[64], src[96]), h = tf32_hi4(v);
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
  const unsigned bars = base + C::STAGES * C::STAGE_BYTES;
  auto full = [&](int s) { return bars + 8u * s; };
  auto empty = [&](int s) { return bars + 8u * (C::STAGES + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int total_items = p.n_chunks * p.r_blocks * p.c_blocks;

  if (threadIdx.x == 0) {
    for (int s = 0; s < C::STAGES; ++s) {
      mbar_init(full(s), 1);
      mbar_init(empty(s), 8);          // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapP) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapG) : "memory");
  }
  __syncthreads();

  if (warp == 0) {
    // ===================== TMA producer (whole warp converged, one elected lane issues) =====================
    int s = 0;
    unsigned ph = 0;
    long long t_wait = 0, t_all = clock64();
    for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
      const Item w = decode_item(p, item);
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
      const int k0 = w.chunk * p.kc, klen = chunk_len(p, w.chunk);
      for (int kb = k0; kb < k0 + klen; ++kb) {
        int q = kb;
        const int px = (q % p.tiles_x) * p.TW; q /= p.tiles_x;
        const int py = (q % p.tiles_y) * p.TH; q /= p.tiles_y;
        const int pn = q * p.TN;
        { const long long t0 = clock64(); mbar_wait(empty(s), ph ^ 1u); t_wait += clock64() - t0; }
        const unsigned st = base + s * C::STAGE_BYTES;
        if (elect_one()) {
          mbar_expect_tx(full(s), (unsigned)(A_BYTES + C::G_BYTES));
#pragma unroll
          for (int j = 0; j < BM / 32; ++j)       // channels past R are TMA zero fill
            tma_4d(st + j * 4096, &mapP, full(s), w.rb * BM + 32 * j, px, py, pn);
#pragma unroll
          for (int j = 0; j < GROUPS; ++j)
            tma_4d(st + C::G_RAW + j * 4096, &mapG, full(s), gch[j], p.stride_x * px + gdx[j],
                   p.stride * py + gdy[j], pn);
        }
        __syncwarp();
        if (++s == C::STAGES) { s = 0; ph ^= 1u; }
      }
    }
    if (p.dbg && blockIdx.x == 0 && lane == 0) { p.dbg[0] = t_wait; p.dbg[1] = clock64() - t_all; }
  } else if (warp >= 4) {
    // ===================== consumers: split + transpose, wgmma, red.add into dW =====================
    const int cw = (warp >> 2) - 1;                  // rows [64 cw, 64 cw + 64) of the 128-row block
    const int ct = threadIdx.x - 128 * (cw + 1);
    const int row0 = 64 * cw + 16 * (ct >> 5) + (lane >> 2);
    const int col0 = 2 * (lane & 3);
    int s = 0;
    unsigned ph = 0;
    long long t_wait = 0, t_all = clock64();
    float sum[R], acc[R];
    for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
      const Item w = decode_item(p, item);
      const int iters = chunk_len(p, w.chunk);
#pragma unroll
      for (int c = 0; c < R; ++c) sum[c] = 0.f;
      int pending = -1;
      for (int it = 0; it < iters; ++it) {
        const int in_chunk = it % p.chunk;
        const bool chunk_end = in_chunk == p.chunk - 1 || it == iters - 1;
        { const long long t0 = clock64(); mbar_wait(full(s), ph); t_wait += clock64() - t0; }
        unsigned char *stp = gbase + s * C::STAGE_BYTES;
        split_transpose<64>(reinterpret_cast<const float *>(stp), stp + C::A_HI, stp + C::A_LO, 64 * cw, ct);
        split_transpose<BN / 2>(reinterpret_cast<const float *>(stp + C::G_RAW), stp + C::B_HI, stp + C::B_LO,
                                cw * (BN / 2), ct);
        fence_proxy_async();
        named_bar_sync(1, 256);                      // both halves of G are split
        const unsigned st = base + s * C::STAGE_BYTES;
        const unsigned long long a_hi = wgmma_desc_k128(st + C::A_HI + cw * (A_BYTES / 2));
        const unsigned long long a_lo = wgmma_desc_k128(st + C::A_LO + cw * (A_BYTES / 2));
        const unsigned long long b_hi = wgmma_desc_k128(st + C::B_HI), b_lo = wgmma_desc_k128(st + C::B_LO);
        fence_regs(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < KP / 8; ++k) {
          const unsigned long long adv = (unsigned long long)(2 * k);
          Wgmma<BN>::mma(acc, a_lo + adv, b_hi + adv, (in_chunk | k) != 0);
          Wgmma<BN>::mma(acc, a_hi + adv, b_lo + adv, 1);
          Wgmma<BN>::mma(acc, a_hi + adv, b_hi + adv, 1);
        }
        wgmma_commit();
        if (chunk_end) wgmma_wait<0>(); else wgmma_wait<1>();
        fence_regs(acc);
        __syncwarp();
        if (pending >= 0 && lane == 0) mbar_arrive(empty(pending));
        pending = s;
        if (chunk_end) {
          if (lane == 0) mbar_arrive(empty(s));
          pending = -1;
#pragma unroll
          for (int c = 0; c < R; ++c) sum[c] += acc[c];
        }
        if (++s == C::STAGES) { s = 0; ph ^= 1u; }
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
    if (p.dbg && blockIdx.x == 0 && threadIdx.x == 128) { p.dbg[2] = t_wait; p.dbg[3] = clock64() - t_all; }
  }
}

template <int BN>
static int launch(const CUtensorMap &mP, const CUtensorMap &mG, const WgradParams &p, cudaStream_t stream) {
  using C = Cfg<BN>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(tc_wgrad_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
    if (e != cudaSuccess) { set_error("tc_wgrad: cannot opt in to %d bytes of shared memory: %s", C::SMEM_BYTES, cudaGetErrorString(e)); return UNFLOW_ECUDA; }
    attr_set = true;
  }
  const long long total = (long long)p.n_chunks * p.r_blocks * p.c_blocks;
  const int grid = total < kNumSMs ? (int)total : kNumSMs;
  tc_wgrad_kernel<BN><<<grid, NTHREADS, C::SMEM_BYTES, stream>>>(mP, mG, p);
  count_launch();
  return check_launch("tc_wgrad_kernel");
}

static int launch_bn(int BN, const CUtensorMap &mP, const CUtensorMap &mG, const WgradParams &p, cudaStream_t stream) {
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
    rc = tc::encode(&mP, P, 4, dims, strides, box, estr, CU_TENSOR_MAP_SWIZZLE_NONE);   // split + transposed by the consumers
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
    rc = tc::encode(&mP, P, 4, dims, strides, box, estr, CU_TENSOR_MAP_SWIZZLE_NONE);   // split + transposed by the consumers
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
