// correlation_tiled.cu -- the FlowNetC cost volume on sm_90a: TMA-staged, register-tiled fp32.
//
// Serves kernel_size=1, stride_1=1, stride_2=2, pad == max_displacement <= 20, H even, W % 4 == 0
// (reference call site src/e2eflow/core/flownet.py:221-222; math of CorrelateData,
// ops/correlation_op.cu.cc:52-117):
//
//   out[b,(p,o),y,x] = (1/C) * sum_c in0[b,c,y,x] * in1[b,c,y+2p,x+2o]     (0 outside the image)
//
// This is a banded batched contraction, FMA-bound on CUDA cores in exact fp32 (59 FLOP/B,
// SURVEY.md R5), so the design goal is to keep the FMA pipe busy with few shared-memory
// wavefronts per FMA and to touch HBM exactly once:
//
//  * work item = (image b, 4 consecutive in1 rows y2, 16-pixel column tile).  All (y, y2) row
//    pairs with y2 in the group and |y2-y| <= 2r, y2-y even, are compacted into a pair list
//    (<= 84 pairs); row pairs whose in1 row is outside the image are never computed -- their
//    outputs are exact zeros and are written by a zero-fill pass of the same kernel
//    (22% of the nominal FLOPs at H=48 are such zeros).
//  * a warp owns 8 row pairs; lane = (pair 0..7, pixel group 0..1, displacement half 0..1).
//    Each thread keeps an 8-pixel x 11-displacement register tile: per channel it loads
//    8 in0 values and a 28-float in1 window (the Toeplitz structure x2 = x + 2o makes 88 FMAs
//    need only 36 operands), all as 128-bit shared loads.  Lanes that share an in1 row read the
//    same window addresses (shared-memory broadcast).
//  * in0 is staged as two row-parity planes (TMA 5-D view [B][C][H/2][2][W]) with a 20-float
//    row pitch so the 8 row pairs of a quarter warp hit 8 different bank groups;
//    in1 is staged as a dense [c][4][56] box.  Out-of-image rows/columns are TMA zero fill --
//    there is no padded copy of the inputs (the reference writes 2 x 144 MB of them).
//  * one producer warp feeds a 4-stage mbarrier ring of 8-channel slices; 11 consumer warps.
//  * every output element is written exactly once, as float4, by the thread that owns it.
//
// Algorithmic bytes: 4*B*H*W*(2C + D^2); FLOPs: 2*B*H*W*C*D^2 (DESIGN.md).
#include "correlation.cuh"
#include "tma.cuh"

namespace unflow {

using namespace tc;

namespace ct {
constexpr int S2 = 2;
constexpr int RMAX = 10;                   // max neighbourhood radius (md/stride_2)
constexpr int NY2 = 4;                     // in1 rows per work item
constexpr int TX = 16;                     // output columns per work item
constexpr int WIN = TX + 2 * S2 * RMAX;    // 56 staged in1 columns
constexpr int P0 = 20;                     // in0 row pitch in floats (TX used)
constexpr int ROWS0 = NY2 + 2 * S2 * RMAX; // 44 in0 rows reachable from the in1 group
constexpr int R0H = ROWS0 / 2;             // 22 rows per parity plane
constexpr int CC = 8;                      // channels per pipeline stage
constexpr int STAGES = 4;
constexpr int NCW = 11;                    // consumer warps (11*8 = 88 >= 84 pair slots)
constexpr int NTHREADS = (NCW + 1) * 32;   // + 1 producer warp
constexpr int DO = 11;                     // displacements per thread (two halves overlap at o=0)
constexpr int PX = 8;                      // pixels per thread
constexpr int MAXPAIRS = NY2 * (2 * RMAX + 1);

constexpr int IN0_PLANE_FLOATS = CC * R0H * P0;     // 3520
constexpr int IN1_FLOATS = CC * NY2 * WIN;          // 1792
constexpr int STAGE_FLOATS = 2 * IN0_PLANE_FLOATS + IN1_FLOATS;
constexpr int STAGE_BYTES = STAGE_FLOATS * 4;       // 35328
static_assert((IN0_PLANE_FLOATS * 4) % 128 == 0 && (IN1_FLOATS * 4) % 128 == 0, "TMA dst alignment");

struct Smem {
  float stage[STAGES][STAGE_FLOATS];
  unsigned long long full[STAGES];
  unsigned long long empty[STAGES];
  int npairs, nzero;
  short pair_y[MAXPAIRS], pair_y2r[MAXPAIRS], pair_p[MAXPAIRS];
  short zero_y[MAXPAIRS], zero_p[MAXPAIRS];
};
}  // namespace ct

// ------------------------------------------------------------------------------------------
// Forward kernel
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(ct::NTHREADS, 1)
corr_fwd_tiled_kernel(const __grid_constant__ CUtensorMap map0,  // in0 as [B][C][H/2][2][W]
                      const __grid_constant__ CUtensorMap map1,  // in1 as [B][C][H][W]
                      float *__restrict__ out, float *__restrict__ out_rev, int C, int H, int W, int r,
                      int y2_first) {
  using namespace ct;
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  Smem &sm = *reinterpret_cast<Smem *>(smem_raw);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int x0 = blockIdx.x * TX;
  const int Y2 = y2_first + blockIdx.y * NY2;  // first in1 row of this group (multiple of 4)
  const int b = blockIdx.z;
  const int D = 2 * r + 1;
  const int ybase = Y2 - S2 * RMAX;  // first staged in0 row (even)

  // Work lists, built in parallel: warp y2r scans the 2r+1 displacement rows of in1 row Y2+y2r
  // (lane <-> p), ballots the valid ones and ranks them; the producer warp initialises the barriers.
  // (A serial build by thread 0 cost 4.5 % of the kernel in the first ncu profile.)
  __shared__ int s_cnt[NY2], s_zcnt[NY2];
  unsigned vmask = 0, zmask = 0;
  int my_y = 0;
  if (warp < NY2) {
    const int y2 = Y2 + warp;
    const bool inside = y2 >= 0 && y2 < H;
    my_y = y2 - S2 * (lane - r);
    const bool ok = lane < D && my_y >= 0 && my_y < H;
    vmask = __ballot_sync(0xffffffffu, ok && inside);
    zmask = __ballot_sync(0xffffffffu, ok && !inside);
    if (lane == 0) { s_cnt[warp] = __popc(vmask); s_zcnt[warp] = __popc(zmask); }
  }
  if (warp == NCW && lane == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(s32(&sm.full[s]), 1); mbar_init(s32(&sm.empty[s]), NCW); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (warp < NY2) {
    int pbase = 0, zbase = 0;
    for (int k = 0; k < warp; ++k) { pbase += s_cnt[k]; zbase += s_zcnt[k]; }
    const unsigned lt = (1u << lane) - 1u;
    if ((vmask >> lane) & 1u) {
      const int pi = pbase + __popc(vmask & lt);
      sm.pair_y[pi] = (short)my_y; sm.pair_y2r[pi] = (short)warp; sm.pair_p[pi] = (short)lane;
    }
    if ((zmask >> lane) & 1u) {
      const int zi = zbase + __popc(zmask & lt);
      sm.zero_y[zi] = (short)my_y; sm.zero_p[zi] = (short)lane;
    }
    if (warp == NY2 - 1 && lane == 0) { sm.npairs = pbase + s_cnt[warp]; sm.nzero = zbase + s_zcnt[warp]; }
  }
  __syncthreads();
  const int npairs = sm.npairs, nzero = sm.nzero;
  const size_t plane_out = (size_t)H * W;        // out_h == H, out_w == W on this path
  float *outb = out + (size_t)b * D * D * plane_out;

  // ---- exact zeros: row pairs whose in1 row lies outside the image -------------------------
  if (nzero > 0) {
    const int per_pair = D * (TX / 4);
    for (int i = tid; i < nzero * per_pair; i += NTHREADS) {
      const int zp = i / per_pair, rem = i - zp * per_pair;
      const int o = rem / (TX / 4), q = rem - o * (TX / 4);
      const int x = x0 + 4 * q;
      if (x < W) {
        float *dst = outb + ((size_t)(sm.zero_p[zp] * D + o)) * plane_out + (size_t)sm.zero_y[zp] * W + x;
        *reinterpret_cast<float4 *>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
  }
  if (npairs == 0) return;

  const int nchunks = (C + CC - 1) / CC;

  if (warp == NCW) {
    // ---------------- producer warp: one lane drives TMA -----------------------------------
    if (lane == 0) {
      for (int it = 0; it < nchunks; ++it) {
        const int s = it % STAGES;
        const unsigned ph = (unsigned)(it / STAGES) & 1u;
        mbar_wait(s32(&sm.empty[s]), ph ^ 1u);
        mbar_expect_tx(s32(&sm.full[s]), STAGE_BYTES);
        float *st = sm.stage[s];
        const int c0 = it * CC;
        // in0 parity planes: coords (x, parity, hh, c, b)
        tma_5d(s32(st), &map0, s32(&sm.full[s]), x0, 0, ybase >> 1, c0, b);
        tma_5d(s32(st + IN0_PLANE_FLOATS), &map0, s32(&sm.full[s]), x0, 1, ybase >> 1, c0, b);
        // in1 window: coords (x, y, c, b)
        tma_4d(s32(st + 2 * IN0_PLANE_FLOATS), &map1, s32(&sm.full[s]), x0 - S2 * RMAX, Y2, c0, b);
      }
    }
    return;
  }

  // ---------------- consumer warps ----------------------------------------------------------
  const int slot = warp * 8 + (lane & 7);
  const bool active = slot < npairs;
  const int pslot = active ? slot : 0;
  const int pxg = (lane >> 3) & 1, og = lane >> 4;
  const int y = sm.pair_y[pslot], y2r = sm.pair_y2r[pslot], pidx = sm.pair_p[pslot];
  const int yrel = y - ybase;
  // float offsets inside a stage (channel 0)
  const int off0 = (yrel & 1) * IN0_PLANE_FLOATS + (yrel >> 1) * P0 + pxg * PX;
  const int off1 = 2 * IN0_PLANE_FLOATS + y2r * WIN + pxg * PX + og * (S2 * RMAX);

  float acc[DO][PX];
#pragma unroll
  for (int t = 0; t < DO; ++t)
#pragma unroll
    for (int i = 0; i < PX; ++i) acc[t][i] = 0.0f;

  const bool warp_active = warp * 8 < npairs;
  for (int it = 0; it < nchunks; ++it) {
    const int s = it % STAGES;
    const unsigned ph = (unsigned)(it / STAGES) & 1u;
    mbar_wait(s32(&sm.full[s]), ph);
    if (warp_active) {
      const float *p0 = sm.stage[s] + off0;
      const float *p1 = sm.stage[s] + off1;
      // explicit register double buffering: the operands of channel cc+1 are loaded before the
      // 88 FMAs of channel cc are issued, so the shared-memory latency hides behind the math even
      // with only ~3 warps per scheduler
      float4 an[2], wn[(PX + S2 * (DO - 1)) / 4];
      an[0] = *reinterpret_cast<const float4 *>(p0);
      an[1] = *reinterpret_cast<const float4 *>(p0 + 4);
#pragma unroll
      for (int k = 0; k < (PX + S2 * (DO - 1)) / 4; ++k) wn[k] = *reinterpret_cast<const float4 *>(p1 + 4 * k);
#pragma unroll
      for (int cc = 0; cc < CC; ++cc) {
        float a[PX], w[PX + S2 * (DO - 1)];
        a[0] = an[0].x; a[1] = an[0].y; a[2] = an[0].z; a[3] = an[0].w;
        a[4] = an[1].x; a[5] = an[1].y; a[6] = an[1].z; a[7] = an[1].w;
#pragma unroll
        for (int k = 0; k < (PX + S2 * (DO - 1)) / 4; ++k) {
          w[4 * k] = wn[k].x; w[4 * k + 1] = wn[k].y; w[4 * k + 2] = wn[k].z; w[4 * k + 3] = wn[k].w;
        }
        if (cc + 1 < CC) {
          an[0] = *reinterpret_cast<const float4 *>(p0 + (cc + 1) * (R0H * P0));
          an[1] = *reinterpret_cast<const float4 *>(p0 + (cc + 1) * (R0H * P0) + 4);
#pragma unroll
          for (int k = 0; k < (PX + S2 * (DO - 1)) / 4; ++k)
            wn[k] = *reinterpret_cast<const float4 *>(p1 + (cc + 1) * (NY2 * WIN) + 4 * k);
        }
#pragma unroll
        for (int t = 0; t < DO; ++t)
#pragma unroll
          for (int i = 0; i < PX; ++i) acc[t][i] = fmaf(a[i], w[i + S2 * t], acc[t][i]);
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(s32(&sm.empty[s]));
  }

  // ---------------- epilogue: each thread stores its 8 x 11 tile ----------------------------
  if (active) {
    const float denom = (float)C;  // sumelems = K*K*C with K = 1; true division as the reference
    const int x = x0 + pxg * PX;
#pragma unroll
    for (int t = 0; t < DO; ++t) {
      const int o = og == 0 ? t - RMAX : t;
      if (o < -r || o > r || (og == 1 && t == 0)) continue;
      float *dst = outb + ((size_t)(pidx * D + (o + r))) * plane_out + (size_t)y * W + x;
      if (x < W)
        *reinterpret_cast<float4 *>(dst) =
            make_float4(acc[t][0] / denom, acc[t][1] / denom, acc[t][2] / denom, acc[t][3] / denom);
      if (x + 4 < W)
        *reinterpret_cast<float4 *>(dst + 4) =
            make_float4(acc[t][4] / denom, acc[t][5] / denom, acc[t][6] / denom, acc[t][7] / denom);
      if (out_rev) {
        // The cost volume of the OTHER direction is a re-indexing of this one (SURVEY.md H1b):
        //   corr(in1,in0)[(-p,-o)](y2, x+2o) == corr(in0,in1)[(p,o)](y, x),   y2 = y + 2p
        // (same products, same summation order over the channels -> bit-identical to a second launch
        // with swapped inputs).  Elements of the reverse volume whose displaced pixel is outside the
        // image are never produced here: the launcher zero-fills the volume first.
        float *rev = out_rev + (size_t)b * D * D * plane_out +
                     ((size_t)((2 * r - pidx) * D + (r - o))) * plane_out + (size_t)(Y2 + y2r) * W;
#pragma unroll
        for (int j = 0; j < PX / 2; ++j) {
          const int xs = x + 2 * j, xr = xs + S2 * o;      // source column, reverse-volume column (both even)
          if (xs < W && xr >= 0 && xr < W)
            *reinterpret_cast<float2 *>(rev + xr) = make_float2(acc[t][2 * j] / denom, acc[t][2 * j + 1] / denom);
        }
      }
    }
  }
}

// gout_eff[(p,o)](y,x) = gout[(p,o)](y,x) + gout_rev[(-p,-o)](y+2p, x+2o): folds the gradient of the
// reverse cost volume into the forward one, so ONE pair of backward launches serves both directions.
__global__ void __launch_bounds__(256)
corr_fold_grad_kernel(const float *__restrict__ g, const float *__restrict__ grev, float *__restrict__ geff,
                      int D, int H, int W, long long total2) {
  const int r = D / 2, W2 = W / 2;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total2;
       i += (long long)gridDim.x * blockDim.x) {
    long long t = i;
    const int x = (int)(t % W2) * 2; t /= W2;
    const int y = (int)(t % H); t /= H;
    const int ch = (int)(t % (D * D));
    const long long b = t / (D * D);
    const int p = ch / D - r, o = ch % D - r;
    float2 v = *reinterpret_cast<const float2 *>(g + 2 * i);
    const int yr = y + ct::S2 * p, xr = x + ct::S2 * o;
    if (yr >= 0 && yr < H && xr >= 0 && xr < W) {
      const float2 w = *reinterpret_cast<const float2 *>(
          grev + ((b * D * D + (long long)((r - p) * D + (r - o))) * H + yr) * W + xr);
      v.x += w.x; v.y += w.y;
    }
    *reinterpret_cast<float2 *>(geff + 2 * i) = v;
  }
}

// ------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------
static int encode_map(CUtensorMap *m, const float *base, int rank, const cuuint64_t *dims,
                      const cuuint64_t *strides_bytes, const cuuint32_t *box) {
  const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  return tc::encode(m, base, rank, dims, strides_bytes, box, estr, CU_TENSOR_MAP_SWIZZLE_NONE,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
}

bool corr_tiled_supported(const CorrGeom &g) {
  return g.ks == 1 && g.s1 == 1 && g.s2 == ct::S2 && g.pad == g.md && g.ngr <= ct::RMAX &&
         g.H % 2 == 0 && g.W % 4 == 0 && g.W >= ct::TX && g.H >= 2 && g.B <= 65535;
}

int corr_fold_grad(const float *gout, const float *gout_rev, float *geff, const CorrGeom &g, cudaStream_t s) {
  const int D = 2 * g.ngr + 1;
  const long long total2 = (long long)g.B * D * D * g.H * (g.W / 2);
  corr_fold_grad_kernel<<<grid_for(total2, 256, 16), 256, 0, s>>>(gout, gout_rev, geff, D, g.H, g.W, total2);
  count_launch();
  return check_launch("correlation_fold_grad");
}

int corr_fwd_tiled(const float *in0, const float *in1, float *out, float *out_rev, const CorrGeom &g,
                   cudaStream_t s) {
  using namespace ct;
  if (out_rev) {
    if ((uintptr_t)out_rev & 15) { set_error("correlation: pointers must be 16-byte aligned"); return UNFLOW_EINVAL; }
    const int D = 2 * g.ngr + 1;
    cudaError_t e = cudaMemsetAsync(out_rev, 0, sizeof(float) * (size_t)g.B * D * D * g.H * g.W, s);
    if (e != cudaSuccess) { set_error("correlation memset: %s", cudaGetErrorString(e)); return UNFLOW_ECUDA; }
  }
  if (((uintptr_t)in0 | (uintptr_t)in1 | (uintptr_t)out) & 15) {
    set_error("correlation: pointers must be 16-byte aligned");
    return UNFLOW_EINVAL;
  }
  const cuuint64_t B = g.B, C = g.C, H = g.H, W = g.W;
  CUtensorMap map0, map1;
  {
    // in0 viewed as [B][C][H/2][2][W]; strides (bytes) of dims 1..4
    cuuint64_t dims[5] = {W, 2, H / 2, C, B};
    cuuint64_t str[4] = {W * 4, 2 * W * 4, H * W * 4, C * H * W * 4};
    cuuint32_t box[5] = {P0, 1, R0H, CC, 1};
    int rc = encode_map(&map0, in0, 5, dims, str, box);
    if (rc) return rc;
  }
  {
    cuuint64_t dims[4] = {W, H, C, B};
    cuuint64_t str[3] = {W * 4, H * W * 4, C * H * W * 4};
    cuuint32_t box[4] = {WIN, NY2, CC, 1};
    int rc = encode_map(&map1, in1, 4, dims, str, box);
    if (rc) return rc;
  }
  static bool attr_set = false;
  const int smem_bytes = (int)sizeof(Smem);
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(corr_fwd_tiled_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         smem_bytes);
    if (e != cudaSuccess) { set_error("correlation smem attribute: %s", cudaGetErrorString(e)); return UNFLOW_ECUDA; }
    attr_set = true;
  }
  const int r = g.ngr;
  const int y2_first = -((S2 * r + NY2 - 1) / NY2) * NY2;
  const int y2_end = g.H + S2 * r;  // exclusive
  dim3 grid(ceil_div(g.W, TX), ceil_div(y2_end - y2_first, NY2), g.B);
  corr_fwd_tiled_kernel<<<grid, NTHREADS, smem_bytes, s>>>(map0, map1, out, out_rev, g.C, g.H, g.W, r, y2_first);
  count_launch();
  return check_launch("correlation_fwd(tiled)");
}

// ------------------------------------------------------------------------------------------
// Backward kernels.  Both gradients have the form
//
//   OUT[c,y,x] = (1/C) * sum_{p,o} G(p,o;y,x) * SRC[c, y+2p, x+2o]
//
//   g0 (CorrelateDataBackward0, reference :120-181): SRC = in1, G = gout[(p,o)][y][x]
//   g1 (CorrelateDataBackward1, reference :184-248): SRC = in0, G = gout[(-p,-o)][y+2p][x+2o]
//
// i.e. 441 taps per output element, the tap weight shared by all C channels.  Tiling:
//   * CTA = (image b, 128-channel slab, row pair {y, y+2}, 64 columns); 8 consumer warps, one per
//     8-pixel group, + 1 TMA producer warp.  lane <-> 4 channels {lane, lane+32, lane+64, lane+96},
//     so every tap weight is a shared-memory BROADCAST and every SRC load is a conflict-free
//     128-bit load (channel pitch 108 floats == 12 mod 32).
//   * register tile = 2 rows x 4 channels x 8 pixels (64 accumulators).  The SRC window of a
//     channel slides by 2 columns per displacement o: it is kept in a 12-float rotating register
//     window refilled with ONE 128-bit load per channel per two displacements.
//   * pipeline stage = one SRC row y2 (box 108 x 128 channels) + the two tap-weight tiles that
//     use it (row y with p=(y2-y)/2, row y+2 with p-1): each SRC row is staged once per row pair.
// ------------------------------------------------------------------------------------------
namespace cb {
constexpr int RMAX = 10, S2 = 2;
constexpr int NPXG = 8, PXW = 8, TXB = NPXG * PXW;     // 64 output columns per CTA
constexpr int CCH = 128;                               // channels per CTA
constexpr int SW = TXB + 2 * S2 * RMAX;                // 104 SRC columns needed
constexpr int PITCH = 108;                             // SRC channel pitch (floats)
constexpr int STAGES = 3;
constexpr int NTHREADS = (NPXG + 1) * 32;
constexpr int DMAX = 2 * RMAX + 1;
constexpr int S_FLOATS = CCH * PITCH;                  // 13824
constexpr int G0_FLOATS = DMAX * TXB;                  // 1344  (g0: [o][64])
constexpr int G1_FLOATS = 2208;                        // >= DMAX*SW = 2184 (g1: [o][104]), 128 B multiple
template <bool G1> struct Cfg {
  static constexpr int GW = G1 ? SW : TXB;
  static constexpr int G_FLOATS = G1 ? G1_FLOATS : G0_FLOATS;
  static constexpr int STAGE_FLOATS = S_FLOATS + 2 * G_FLOATS;
};
template <bool G1> struct Smem {
  float stage[STAGES][Cfg<G1>::STAGE_FLOATS];
  float zero_tile[Cfg<G1>::G_FLOATS];     // tap weights of a row that does not use this SRC row
  unsigned long long full[STAGES];
  unsigned long long empty[STAGES];
};
static_assert((S_FLOATS * 4) % 128 == 0 && (G0_FLOATS * 4) % 128 == 0 && (G1_FLOATS * 4) % 128 == 0, "");
}  // namespace cb

// RT > 0: neighbourhood radius known at compile time (RT = 10 is FlowNetC): the displacement loop
// is branch-free, so the compiler can hoist the shared loads of the next displacement pair above
// the FMAs of the current one.  RT = 0: radius read at run time (any even r <= 10).
template <bool G1, int RT>
__global__ void __launch_bounds__(cb::NTHREADS, 1)
corr_bwd_tiled_kernel(const __grid_constant__ CUtensorMap map_src,   // SRC [B][C][H][W], box (108,1,128,1)
                      const __grid_constant__ CUtensorMap map_g,     // gout [B][D*D][H][W], box (GW,1,D,1)
                      float *__restrict__ outp, int C, int H, int W, int r, int slabs) {
  using namespace cb;
  using CF = Cfg<G1>;
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  Smem<G1> &sm = *reinterpret_cast<Smem<G1> *>(smem_raw);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int x0 = blockIdx.x * TXB;
  const int ya = (blockIdx.y >> 1) * 4 + (blockIdx.y & 1), yb = ya + 2;   // row pair
  const int b = blockIdx.z / slabs, c0 = (blockIdx.z % slabs) * CCH;
  if (RT > 0) r = RT;
  const int D = 2 * r + 1;
  const int joff = S2 * (RMAX - r);        // column offset of displacement o=-r inside the staged window

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(s32(&sm.full[s]), 1); mbar_init(s32(&sm.empty[s]), NPXG); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = tid; i < CF::G_FLOATS; i += NTHREADS) sm.zero_tile[i] = 0.0f;
  __syncthreads();

  // stages: SRC rows y2 = ya - 2r + 2k, k = 0 .. 2r+1, inside the image
  const int nk = 2 * r + 2;

  if (warp == NPXG) {
    if (lane == 0) {
      int it = 0;
      for (int k = 0; k < nk; ++k) {
        const int y2 = ya - S2 * r + S2 * k;
        if (y2 < 0 || y2 >= H) continue;
        const int pa = k - r, pb = pa - 1;                 // displacement rows used by ya / yb
        const bool va = pa <= r && ya < H, vb = pb >= -r && yb < H;
        const int s = it % STAGES;
        const unsigned ph = (unsigned)(it / STAGES) & 1u;
        mbar_wait(s32(&sm.empty[s]), ph ^ 1u);
        const unsigned bytes = (unsigned)(S_FLOATS + (va ? D * CF::GW : 0) + (vb ? D * CF::GW : 0)) * 4u;
        mbar_expect_tx(s32(&sm.full[s]), bytes);
        float *st = sm.stage[s];
        tma_4d(s32(st), &map_src, s32(&sm.full[s]), x0 - S2 * RMAX, y2, c0, b);
        if (!G1) {
          if (va) tma_4d(s32(st + S_FLOATS), &map_g, s32(&sm.full[s]), x0, ya, (pa + r) * D, b);
          if (vb) tma_4d(s32(st + S_FLOATS + CF::G_FLOATS), &map_g, s32(&sm.full[s]), x0, yb, (pb + r) * D, b);
        } else {
          if (va) tma_4d(s32(st + S_FLOATS), &map_g, s32(&sm.full[s]), x0 - S2 * RMAX, y2, (r - pa) * D, b);
          if (vb) tma_4d(s32(st + S_FLOATS + CF::G_FLOATS), &map_g, s32(&sm.full[s]), x0 - S2 * RMAX, y2, (r - pb) * D, b);
        }
        ++it;
      }
    }
    return;
  }

  const int pxg = warp;
  const bool warp_active = x0 + pxg * PXW < W;
  float acc[2][4][PXW];
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int cc = 0; cc < 4; ++cc)
#pragma unroll
      for (int i = 0; i < PXW; ++i) acc[a][cc][i] = 0.0f;

  int it = 0;
  for (int k = 0; k < nk; ++k) {
    const int y2 = ya - S2 * r + S2 * k;
    if (y2 < 0 || y2 >= H) continue;
    const int pa = k - r, pb = pa - 1;
    const bool va = pa <= r && ya < H, vb = pb >= -r && yb < H;
    const int s = it % STAGES;
    const unsigned ph = (unsigned)(it / STAGES) & 1u;
    mbar_wait(s32(&sm.full[s]), ph);
    if (warp_active) {
      const float *S = sm.stage[s] + lane * PITCH + pxg * PXW + joff;
      // a row that does not use this SRC row reads an all-zero tap tile: no branch in the hot loop
      const float *Ga = va ? sm.stage[s] + S_FLOATS : sm.zero_tile;
      const float *Gb = vb ? sm.stage[s] + S_FLOATS + CF::G_FLOATS : sm.zero_tile;
      // rotating 12-float window per channel: column col (relative to S) lives in slot col % 12
      float win[4][12];
#pragma unroll
      for (int cc = 0; cc < 4; ++cc) {
        const float4 v0 = *reinterpret_cast<const float4 *>(S + cc * 32 * PITCH);
        const float4 v1 = *reinterpret_cast<const float4 *>(S + cc * 32 * PITCH + 4);
        win[cc][0] = v0.x; win[cc][1] = v0.y; win[cc][2] = v0.z; win[cc][3] = v0.w;
        win[cc][4] = v1.x; win[cc][5] = v1.y; win[cc][6] = v1.z; win[cc][7] = v1.w;
      }
#pragma unroll
      for (int tp = 0; tp <= RMAX; ++tp) {       // displacement pairs t = 2tp, 2tp+1
        if (RT > 0 || 2 * tp < D) {
#pragma unroll
          for (int cc = 0; cc < 4; ++cc) {
            const float4 v = *reinterpret_cast<const float4 *>(S + cc * 32 * PITCH + 4 * tp + 8);
            win[cc][(4 * tp + 8) % 12] = v.x; win[cc][(4 * tp + 9) % 12] = v.y;
            win[cc][(4 * tp + 10) % 12] = v.z; win[cc][(4 * tp + 11) % 12] = v.w;
          }
#pragma unroll
          for (int tt = 0; tt < 2; ++tt) {
            const int t = 2 * tp + tt;
            if (RT > 0 ? t < 2 * RT + 1 : t < D) {
#pragma unroll
              for (int a = 0; a < 2; ++a) {
                const float *G = a == 0 ? Ga : Gb;
                float g[PXW];
                if (!G1) {
                  const float4 g0 = *reinterpret_cast<const float4 *>(G + t * TXB + pxg * PXW);
                  const float4 g1 = *reinterpret_cast<const float4 *>(G + t * TXB + pxg * PXW + 4);
                  g[0] = g0.x; g[1] = g0.y; g[2] = g0.z; g[3] = g0.w;
                  g[4] = g1.x; g[5] = g1.y; g[6] = g1.z; g[7] = g1.w;
                } else {
                  const float *gp = G + (D - 1 - t) * SW + pxg * PXW + joff + 2 * t;
#pragma unroll
                  for (int h2 = 0; h2 < 4; ++h2) {
                    const float2 gv = *reinterpret_cast<const float2 *>(gp + 2 * h2);
                    g[2 * h2] = gv.x; g[2 * h2 + 1] = gv.y;
                  }
                }
#pragma unroll
                for (int cc = 0; cc < 4; ++cc)
#pragma unroll
                  for (int i = 0; i < PXW; ++i)
                    acc[a][cc][i] = fmaf(g[i], win[cc][(2 * t + i) % 12], acc[a][cc][i]);
              }
            }
          }
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(s32(&sm.empty[s]));
    ++it;
  }

  if (warp_active) {
    const float denom = (float)C;
    const int x = x0 + pxg * PXW;
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      const int y = a == 0 ? ya : yb;
      if (y >= H) continue;
#pragma unroll
      for (int cc = 0; cc < 4; ++cc) {
        const int c = c0 + lane + 32 * cc;
        if (c >= C) continue;
        float *dst = outp + (((size_t)b * C + c) * H + y) * W + x;
        *reinterpret_cast<float4 *>(dst) = make_float4(acc[a][cc][0] / denom, acc[a][cc][1] / denom,
                                                       acc[a][cc][2] / denom, acc[a][cc][3] / denom);
        if (x + 4 < W)
          *reinterpret_cast<float4 *>(dst + 4) = make_float4(acc[a][cc][4] / denom, acc[a][cc][5] / denom,
                                                             acc[a][cc][6] / denom, acc[a][cc][7] / denom);
      }
    }
  }
}

bool corr_bwd_tiled_supported(const CorrGeom &g) {
  return corr_tiled_supported(g) && g.ngr % 2 == 0 && g.ngr >= 2 && (long long)g.B * ceil_div(g.C, cb::CCH) <= 65535;
}

template <bool G1>
static int launch_bwd(const float *src, const float *gout, float *outp, const CorrGeom &g, cudaStream_t s) {
  using namespace cb;
  const cuuint64_t B = g.B, C = g.C, H = g.H, W = g.W, D = g.ngw;
  CUtensorMap map_src, map_g;
  {
    cuuint64_t dims[4] = {W, H, C, B};
    cuuint64_t str[3] = {W * 4, H * W * 4, C * H * W * 4};
    cuuint32_t box[4] = {PITCH, 1, CCH, 1};
    int rc = encode_map(&map_src, src, 4, dims, str, box);
    if (rc) return rc;
  }
  {
    cuuint64_t dims[4] = {W, H, D * D, B};
    cuuint64_t str[3] = {W * 4, H * W * 4, D * D * H * W * 4};
    cuuint32_t box[4] = {(cuuint32_t)Cfg<G1>::GW, 1, (cuuint32_t)D, 1};
    int rc = encode_map(&map_g, gout, 4, dims, str, box);
    if (rc) return rc;
  }
  static bool attr_set = false;
  const int smem_bytes = (int)sizeof(Smem<G1>);
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(corr_bwd_tiled_kernel<G1, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         smem_bytes);
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(corr_bwd_tiled_kernel<G1, RMAX>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes);
    if (e != cudaSuccess) { set_error("correlation_grad smem attribute: %s", cudaGetErrorString(e)); return UNFLOW_ECUDA; }
    attr_set = true;
  }
  const int slabs = ceil_div(g.C, CCH);
  dim3 grid(ceil_div(g.W, TXB), ceil_div(g.H, 4) * 2, g.B * slabs);
  if (g.ngr == RMAX)
    corr_bwd_tiled_kernel<G1, RMAX><<<grid, NTHREADS, smem_bytes, s>>>(map_src, map_g, outp, g.C, g.H, g.W, g.ngr, slabs);
  else
    corr_bwd_tiled_kernel<G1, 0><<<grid, NTHREADS, smem_bytes, s>>>(map_src, map_g, outp, g.C, g.H, g.W, g.ngr, slabs);
  count_launch();
  return check_launch(G1 ? "correlation_bwd1(tiled)" : "correlation_bwd0(tiled)");
}

int corr_bwd_tiled(const float *gout, const float *in0, const float *in1, float *g0, float *g1,
                   const CorrGeom &g, cudaStream_t s) {
  if (!corr_bwd_tiled_supported(g)) return corr_bwd_generic(gout, in0, in1, g0, g1, g, s);
  if (((uintptr_t)in0 | (uintptr_t)in1 | (uintptr_t)gout | (uintptr_t)g0 | (uintptr_t)g1) & 15) {
    set_error("correlation_grad: pointers must be 16-byte aligned");
    return UNFLOW_EINVAL;
  }
  int rc = launch_bwd<false>(in1, gout, g0, g, s);
  if (rc) return rc;
  return launch_bwd<true>(in0, gout, g1, g, s);
}

}  // namespace unflow
