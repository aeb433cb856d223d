// narrow_conv_tma.cu -- forward of the flow heads (3x3, stride 1, SAME, C_out = 2; reference flownet.py:92-131)
// with TMA-staged input tiles.  Second version of narrow_fwd_kernel (narrow_conv.cu), which stages its window
// with one 4-byte cp.async per element into a transposed [channel][row][col] tile: issue-bound (ncu: 68 % of
// the issue slots, 14 % of the HBM roofline, no overlap of staging and arithmetic inside a CTA).
//
// Here the (16+2) x (32+2) pixel window of a 16-channel chunk arrives as ONE TMA box in the layout the tensor
// already has, [row][col][16 channels] (64 bytes per pixel, 64-byte swizzle), through a 3-stage mbarrier ring,
// so loading costs one instruction per chunk and overlaps the arithmetic of the previous chunks.
//   lane = output column, warp = 4 output rows: a thread owns a 1 x 4 column strip x 2 outputs; per 8-channel
//   half and window column it keeps the 6 input rows in registers (12 LDS.128, conflict-free: 8 consecutive
//   pixels x 64 B under the 64-byte swizzle cover all 32 banks) and applies the three filter rows to them
//   (12 broadcast LDS.128 of weights) for 576 FMAs: 8 FMAs per shared-memory instruction.
// The layer's weights are staged once per CTA as [chunk][output][tap][16].
// Small images (flow4..flow6: 8..48 tiles on 132 SMs) split the channel chunks over several CTAs per tile that
// add their parts with atomics into a zeroed output, as narrow_fwd_kernel does.
#include "tma.cuh"

namespace unflow {
namespace nct {

using namespace unflow::tc;

constexpr int TH = 16, TW = 32;              // output tile
constexpr int SR = TH + 2, SC = TW + 2;      // window
constexpr int KC = 16;                       // channels per chunk
constexpr int STAGE_BYTES = SR * SC * KC * 4;            // 39168
constexpr int STAGE_PITCH = (STAGE_BYTES + 1023) / 1024 * 1024;   // swizzle pattern = 512 B: keep stages 1 KB aligned
constexpr int THREADS = 128;

// STAGES = 3 with one CTA per SM, or 2 with two CTAs per SM when the layer's weights are small enough (flow2 /
// flow3: 8 warps per SM hide the shared-memory latency better than a third stage does)
template <int STAGES>
__global__ void __launch_bounds__(THREADS, STAGES == 2 ? 2 : 1)
narrow_fwd_tma_kernel(const __grid_constant__ CUtensorMap mapX, const float *__restrict__ w,
                      const float *__restrict__ bias, float *__restrict__ y, int H, int W, int C, long long YP,
                      int csplit) {
  extern __shared__ unsigned char smem_raw[];
  const unsigned base = (s32(smem_raw) + 1023u) & ~1023u;
  unsigned char *gbase = smem_raw + (base - s32(smem_raw));
  const unsigned bars = base + STAGES * STAGE_PITCH;
  float *ws = reinterpret_cast<float *>(gbase + STAGES * STAGE_PITCH + 64);       // [chunks][2][9][16]
  auto full = [&](int s) { return bars + 8u * s; };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n = blockIdx.z / csplit, split = blockIdx.z - n * csplit;
  const int y0 = blockIdx.y * TH, x0 = blockIdx.x * TW;
  const int chunks = (C + KC - 1) / KC, per = (chunks + csplit - 1) / csplit;
  const int k_begin = split * per, k_end = (split + 1) * per < chunks ? (split + 1) * per : chunks;
  const int nk = k_end > k_begin ? k_end - k_begin : 0;

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) mbar_init(full(s), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapX) : "memory");
  }
  // this CTA's weights: ws[(k * 2 + o) * 144 + tap * 16 + c]  (zero beyond C)
  for (int idx = tid; idx < nk * 288; idx += THREADS) {
    const int c = idx & 15, r = idx >> 4, tap = r % 9, ko = r / 9, o = ko & 1, k = ko >> 1;
    const int ch = (k_begin + k) * KC + c;
    ws[idx] = ch < C ? __ldg(w + ((long long)(o * 9 + tap)) * C + ch) : 0.f;
  }
  __syncthreads();
  if (tid == 0) {
    for (int k = 0; k < STAGES && k < nk; ++k) {
      mbar_expect_tx(full(k), STAGE_BYTES);
      tma_4d(base + k * STAGE_PITCH, &mapX, full(k), (k_begin + k) * KC, x0 - 1, y0 - 1, n);
    }
  }

  float acc[4][2];
#pragma unroll
  for (int r = 0; r < 4; ++r) acc[r][0] = acc[r][1] = 0.f;

  for (int k = 0; k < nk; ++k) {
    const int s = k % STAGES;
    mbar_wait(full(s), (unsigned)(k / STAGES) & 1u);
    const unsigned char *tile = gbase + s * STAGE_PITCH;
    const float *wk = ws + k * 288;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
#pragma unroll
      for (int dx = 0; dx < 3; ++dx) {
        // the 6 window rows of column lane + dx, 8 channels each
        float v[6][8];
#pragma unroll
        for (int r = 0; r < 6; ++r) {
          const int p = (4 * warp + r) * SC + lane + dx;            // pixel index inside the box
          const unsigned char *pp = tile + p * 64;
          const int sw = (p >> 1) & 3;                              // 64-byte swizzle: chunk ^= address bits [7, 9)
          const float4 a = *reinterpret_cast<const float4 *>(pp + (((2 * half) ^ sw) << 4));
          const float4 b = *reinterpret_cast<const float4 *>(pp + (((2 * half + 1) ^ sw) << 4));
          v[r][0] = a.x; v[r][1] = a.y; v[r][2] = a.z; v[r][3] = a.w;
          v[r][4] = b.x; v[r][5] = b.y; v[r][6] = b.z; v[r][7] = b.w;
        }
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
          float wv[2][8];
#pragma unroll
          for (int o = 0; o < 2; ++o) {
            const float4 a = *reinterpret_cast<const float4 *>(wk + o * 144 + (ky * 3 + dx) * 16 + 8 * half);
            const float4 b = *reinterpret_cast<const float4 *>(wk + o * 144 + (ky * 3 + dx) * 16 + 8 * half + 4);
            wv[o][0] = a.x; wv[o][1] = a.y; wv[o][2] = a.z; wv[o][3] = a.w;
            wv[o][4] = b.x; wv[o][5] = b.y; wv[o][6] = b.z; wv[o][7] = b.w;
          }
#pragma unroll
          for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int c = 0; c < 8; ++c) {
              acc[r][0] = fmaf(v[r + ky][c], wv[0][c], acc[r][0]);
              acc[r][1] = fmaf(v[r + ky][c], wv[1][c], acc[r][1]);
            }
        }
      }
    }
    __syncthreads();                           // every warp is done with stage s
    if (tid == 0 && k + STAGES < nk) {
      mbar_expect_tx(full(s), STAGE_BYTES);
      tma_4d(base + s * STAGE_PITCH, &mapX, full(s), (k_begin + k + STAGES) * KC, x0 - 1, y0 - 1, n);
    }
  }

  const int gx = x0 + lane;
  if (gx < W && nk > 0) {
    const float b0 = (bias && split == 0) ? bias[0] : 0.f, b1 = (bias && split == 0) ? bias[1] : 0.f;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int gy = y0 + 4 * warp + r;
      if (gy < H) {
        float *out = y + (((long long)n * H + gy) * W + gx) * YP;
        if (csplit == 1) {
          *reinterpret_cast<float2 *>(out) = make_float2(acc[r][0] + b0, acc[r][1] + b1);
        } else {
          atomicAdd(out, acc[r][0] + b0);
          atomicAdd(out + 1, acc[r][1] + b1);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------
// Weight gradient of the same layers:  gw[o][ky][kx][c] = sum_{n,y,x} g[n,y,x,o] * x[n, y+ky-1, x+kx-1, c]
// Same TMA-staged window.  warp = 4 channels of the chunk, lane = tile column: a thread walks down its
// column with a 3 x 3 window of float4 (4 channels) in registers -- 3 LDS.128 + 1 LDS.64 (the two gradient
// values) per 72 FMAs -- and owns 72 partial sums (9 taps x 4 channels x 2 outputs).  At the end of the chunk the
// 32 lanes of a warp are summed through a per-warp shared-memory transpose (fixed order), and the CTA writes its
// partial sums in the layout of narrow_wgrad_kernel, so narrow_wgrad_reduce_kernel finishes the job as before
// (deterministic: no atomics).
// ------------------------------------------------------------------------------------------------------
constexpr int WG_STAGES = 3;
constexpr int RED_PITCH = 33;

__global__ void __launch_bounds__(THREADS, 1)
narrow_wgrad_tma_kernel(const __grid_constant__ CUtensorMap mapX, const float *__restrict__ g, long long gsN,
                        long long gsC, long long gsH, long long gsW, float *__restrict__ partial, int H, int W,
                        int C, int csplit) {
  extern __shared__ unsigned char smem_raw[];
  const unsigned base = (s32(smem_raw) + 1023u) & ~1023u;
  unsigned char *gbase = smem_raw + (base - s32(smem_raw));
  const unsigned bars = base + WG_STAGES * STAGE_PITCH;
  float2 *gs = reinterpret_cast<float2 *>(gbase + WG_STAGES * STAGE_PITCH + 64);          // [TH][TW]
  float *red = reinterpret_cast<float *>(gbase + WG_STAGES * STAGE_PITCH + 64 + TH * TW * 8);   // [4][72][RED_PITCH]
  auto full = [&](int s) { return bars + 8u * s; };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n = blockIdx.z / csplit, split = blockIdx.z - n * csplit;
  const int y0 = blockIdx.y * TH, x0 = blockIdx.x * TW;
  const long long bid = ((long long)n * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
  const int chunks = (C + KC - 1) / KC, per = (chunks + csplit - 1) / csplit;
  const int k_begin = split * per, k_end = (split + 1) * per < chunks ? (split + 1) * per : chunks;
  const int nk = k_end > k_begin ? k_end - k_begin : 0;

  if (tid == 0) {
    for (int s = 0; s < WG_STAGES; ++s) mbar_init(full(s), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapX) : "memory");
  }
  for (int idx = tid; idx < TH * TW; idx += THREADS) {
    const int r = idx / TW, c = idx - r * TW;
    const int gy = y0 + r, gx = x0 + c;
    float2 v = make_float2(0.f, 0.f);
    if (gy < H && gx < W) {
      const float *gp = g + n * gsN + gy * gsH + gx * gsW;
      v.x = __ldg(gp); v.y = __ldg(gp + gsC);
    }
    gs[idx] = v;
  }
  __syncthreads();
  if (tid == 0) {
    for (int k = 0; k < WG_STAGES && k < nk; ++k) {
      mbar_expect_tx(full(k), STAGE_BYTES);
      tma_4d(base + k * STAGE_PITCH, &mapX, full(k), (k_begin + k) * KC, x0 - 1, y0 - 1, n);
    }
  }
  float *myred = red + warp * 72 * RED_PITCH;

  for (int k = 0; k < nk; ++k) {
    const int s = k % WG_STAGES;
    mbar_wait(full(s), (unsigned)(k / WG_STAGES) & 1u);
    const unsigned char *tile = gbase + s * STAGE_PITCH;
    auto ldx = [&](int row, int col) -> float4 {        // 4 channels (this warp's quad) of box pixel (row, col)
      const int p = row * SC + col;
      return *reinterpret_cast<const float4 *>(tile + p * 64 + ((warp ^ ((p >> 1) & 3)) << 4));
    };
    float acc[9][4][2];
#pragma unroll
    for (int t = 0; t < 9; ++t)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[t][e][0] = acc[t][e][1] = 0.f;
    float4 xw[3][3];
#pragma unroll
    for (int ky = 0; ky < 2; ++ky)
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) xw[ky][kx] = ldx(ky, lane + kx);
#pragma unroll 4
    for (int r = 0; r < TH; ++r) {
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) xw[2][kx] = ldx(r + 2, lane + kx);
      const float2 gv = gs[r * TW + lane];
#pragma unroll
      for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
          const float xv[4] = {xw[ky][kx].x, xw[ky][kx].y, xw[ky][kx].z, xw[ky][kx].w};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            acc[ky * 3 + kx][e][0] = fmaf(gv.x, xv[e], acc[ky * 3 + kx][e][0]);
            acc[ky * 3 + kx][e][1] = fmaf(gv.y, xv[e], acc[ky * 3 + kx][e][1]);
          }
        }
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) { xw[0][kx] = xw[1][kx]; xw[1][kx] = xw[2][kx]; }
    }
    // sum over the 32 lanes (columns) of this warp: j = (o * 9 + tap) * 4 + e
    __syncwarp();
#pragma unroll
    for (int t = 0; t < 9; ++t)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        myred[((0 * 9 + t) * 4 + e) * RED_PITCH + lane] = acc[t][e][0];
        myred[((1 * 9 + t) * 4 + e) * RED_PITCH + lane] = acc[t][e][1];
      }
    __syncwarp();
    const int c0 = (k_begin + k) * KC + 4 * warp;
    for (int j = lane; j < 72; j += 32) {
      float sum = 0.f;
#pragma unroll 8
      for (int l = 0; l < 32; ++l) sum += myred[j * RED_PITCH + l];
      const int e = j & 3, i = j >> 2;                 // i = o * 9 + tap
      if (c0 + e < C) partial[(bid * 18 + i) * C + c0 + e] = sum;
    }
    __syncthreads();                           // every warp is done with stage s (and with its red buffer)
    if (tid == 0 && k + WG_STAGES < nk) {
      mbar_expect_tx(full(s), STAGE_BYTES);
      tma_4d(base + s * STAGE_PITCH, &mapX, full(s), (k_begin + k + WG_STAGES) * KC, x0 - 1, y0 - 1, n);
    }
  }
}

}  // namespace nct

// Launch the TMA-staged weight-gradient kernel (partials only; the caller runs the reduce kernel); -1: cannot take it.
int narrow_wgrad_tma(const float *x, long long x_pitch, const float *g, long long gsN, long long gsC, long long gsH,
                     long long gsW, float *partial, int N, int H, int W, int C, int csplit, cudaStream_t st) {
  using namespace nct;
  if (((uintptr_t)x & 15) != 0 || x_pitch % 4 != 0) return -1;
  const size_t smem = (size_t)WG_STAGES * STAGE_PITCH + 64 + TH * TW * 8 + 4 * 72 * RED_PITCH * sizeof(float) + 1024;
  CUtensorMap mX;
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)x_pitch * 4, (cuuint64_t)x_pitch * 4 * W, (cuuint64_t)x_pitch * 4 * W * H};
  cuuint32_t box[4] = {(cuuint32_t)KC, (cuuint32_t)SC, (cuuint32_t)SR, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  if (tc::encode(&mX, x, 4, dims, strides, box, estr, CU_TENSOR_MAP_SWIZZLE_64B)) return -1;
  static bool attr = false;
  if (!attr) {
    if (cudaFuncSetAttribute(narrow_wgrad_tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
      (void)cudaGetLastError();
      return -1;
    }
    attr = true;
  }
  const dim3 grid((W + TW - 1) / TW, (H + TH - 1) / TH, N * csplit);
  narrow_wgrad_tma_kernel<<<grid, THREADS, smem, st>>>(mX, g, gsN, gsC, gsH, gsW, partial, H, W, C, csplit);
  count_launch();
  return check_launch("conv3x3_narrow_wgrad(tma)");
}

// Launch the TMA-staged forward; returns -1 when the arguments do not fit it (the caller falls back to
// narrow_fwd_kernel): TMA needs a 16-byte aligned base and pixel pitch; the staged weights must fit shared memory.
int narrow_fwd_tma(const float *x, long long x_pitch, const float *w, const float *bias, float *y, long long y_pitch,
                   int N, int H, int W, int C, int csplit, cudaStream_t st) {
  using namespace nct;
  if (((uintptr_t)x & 15) != 0 || x_pitch % 4 != 0) return -1;
  const int chunks = (C + KC - 1) / KC, per = (chunks + csplit - 1) / csplit;
  const size_t wbytes = 64 + (size_t)per * 288 * sizeof(float) + 1024;
  const int stages = (2 * (size_t)STAGE_PITCH + wbytes <= 110 * 1024) ? 2 : 3;
  const size_t smem = (size_t)stages * STAGE_PITCH + wbytes;
  if (smem > 220 * 1024) return -1;
  CUtensorMap mX;
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)x_pitch * 4, (cuuint64_t)x_pitch * 4 * W, (cuuint64_t)x_pitch * 4 * W * H};
  cuuint32_t box[4] = {(cuuint32_t)KC, (cuuint32_t)SC, (cuuint32_t)SR, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  if (tc::encode(&mX, x, 4, dims, strides, box, estr, CU_TENSOR_MAP_SWIZZLE_64B)) return -1;
  static size_t attr[2] = {0, 0};
  if (smem > attr[stages - 2]) {
    cudaError_t e = stages == 2
        ? cudaFuncSetAttribute(narrow_fwd_tma_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
        : cudaFuncSetAttribute(narrow_fwd_tma_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { (void)cudaGetLastError(); return -1; }
    attr[stages - 2] = smem;
  }
  const dim3 grid((W + TW - 1) / TW, (H + TH - 1) / TH, N * csplit);
  if (stages == 2) narrow_fwd_tma_kernel<2><<<grid, THREADS, smem, st>>>(mX, w, bias, y, H, W, C, y_pitch, csplit);
  else narrow_fwd_tma_kernel<3><<<grid, THREADS, smem, st>>>(mX, w, bias, y, H, W, C, y_pitch, csplit);
  count_launch();
  return check_launch("conv3x3_narrow_fwd(tma)");
}

}  // namespace unflow
