// narrow_conv.cu -- the flow-prediction heads of the decoder: 3x3, stride 1, SAME, C_in = 194..1026,
// C_out = 2 (reference flownet.py:92-131, `slim.conv2d(concatN, 2, 3, scope='flowN', activation_fn=None)`).
//
// A convolution with two output channels is no tensor-core shape: as an implicit GEMM its N
// dimension is 2 (padded to 4, computed on 64-wide tiles), so the library kernels of the 3xTF32
// path spend their time streaming the 3x-wide split operand (flow2: 144 us operand pass + 516 us
// fprop, 141 us + 886 us wgrad per step in the ncu launch list) for 1.7 GFLOP of useful work.  In
// exact fp32 on the FMA pipes the same layer reads its input once:
//
//   forward  y[n,y,x,co]      = b[co] + sum_{ky,kx,c} x[n,y+ky-1,x+kx-1,c] * w[co,ky,kx,c]
//   wgrad    gw[co,ky,kx,c]   = sum_{n,y,x} g[n,y,x,co] * x[n,y+ky-1,x+kx-1,c]
//
// Both kernels work on a 16x32 output tile per CTA and walk the input channels in chunks of 16:
// the (16+2)x(32+2) input window of the chunk is staged in shared memory TRANSPOSED to
// [channel][row][col] (global reads: one 8-byte channel pair per lane, lanes on consecutive pixels;
// shared stores: consecutive banks), so that the arithmetic reads it conflict-free:
//   forward: a thread owns 4 adjacent pixels x 2 outputs; per (channel, ky) it loads 6 inputs
//            (LDS.128 + LDS.64) and 6 weights (2 broadcast LDS.128) for 24 FMAs;
//   wgrad:   a thread owns one channel and two tile rows, slides a 3x3 window along the row
//            (3 LDS + 1 broadcast LDS.64 per 18 FMAs), partial sums are reduced over the 8 row
//            groups in shared memory and written per CTA; a second kernel adds the per-CTA
//            partials in a fixed order (deterministic, no atomics).
// HBM bytes: forward 4*N*H*W*(C + 2), wgrad 4*N*H*W*(C + 2) + the partials.
// The input gradient of these layers stays on the library path (its output is C_in wide).
#include "common.cuh"

namespace unflow {
int narrow_fwd_tma(const float *x, long long x_pitch, const float *w, const float *bias, float *y, long long y_pitch,
                   int N, int H, int W, int C, int csplit, cudaStream_t st);     // narrow_conv_tma.cu
int narrow_wgrad_tma(const float *x, long long x_pitch, const float *g, long long gsN, long long gsC, long long gsH,
                     long long gsW, float *partial, int N, int H, int W, int C, int csplit, cudaStream_t st);
namespace nc {

constexpr int TH = 16, TW = 32;            // output tile
constexpr int SR = TH + 2, SC = TW + 2;    // staged input window (halo 1)
constexpr int PITCH = 36;                  // floats per staged row (SC rounded up to a multiple of 4)
constexpr int KC = 16;                     // input channels per chunk
constexpr int THREADS = 128;
constexpr int NOUT = 18;                   // 2 output channels x 9 taps
constexpr int GPITCH = 2 * TW + 2;         // floats per row of the staged gradient tile (wgrad)
constexpr int FWD_PITCH = 38, FWD_CHS = 706;   // forward staging layout (see narrow_fwd_kernel)
static_assert(FWD_CHS >= SR * FWD_PITCH && FWD_CHS % 32 == 2 && FWD_PITCH % 4 == 2, "forward smem layout");

__device__ __forceinline__ void cp_async_4(unsigned dst, const float *src, unsigned bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst), "l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// Stage the window of chunk [c0, c0+KC) as xs[ch * CHS + row * PITCH_ + col]; zero outside the image
// and beyond C.  x is NHWC with XP floats between pixels (XP >= C: a channel slice of a concat buffer).
// Asynchronous 4-byte copies (LDGSTS), nothing passes through registers, so all ~77 copies of a thread
// are in flight at once and the DRAM latency is paid once per chunk.  A warp instruction covers 2
// consecutive pixels x 16 channels = two 64-byte runs; out-of-image / beyond-C elements are
// zero-filled by a copy of size 0.  The copies are issued row by row: the row pointer and the bounds
// test of a window row are computed once, the columns of a thread are a fixed unrolled set.
template <int CHS, int PITCH_>
__device__ __forceinline__ void stage(float *xs, const float *__restrict__ x, int n, int y0, int x0, int c0,
                                      int H, int W, int C, long long XP, int tid) {
  const int ch = tid & 15, q = tid >> 4;                  // 8 column slots: pc = q, q+8, q+16, q+24, (q+32)
  const bool chan_ok = c0 + ch < C;
  const float *xc = x + (long long)n * H * W * XP + c0 + ch;
  const unsigned dbase = (unsigned)__cvta_generic_to_shared(xs + ch * CHS) + (unsigned)q * 4u;
  int gxs[5];
  bool cok[5];
#pragma unroll
  for (int j = 0; j < 5; ++j) {
    const int pc = q + 8 * j;
    gxs[j] = x0 - 1 + pc;
    cok[j] = chan_ok && pc < SC && gxs[j] >= 0 && gxs[j] < W;
  }
#pragma unroll 3
  for (int pr = 0; pr < SR; ++pr) {
    const int gy = y0 - 1 + pr;
    const bool rok = gy >= 0 && gy < H;
    const float *rowp = xc + (long long)(rok ? gy : 0) * W * XP;
    const unsigned drow = dbase + (unsigned)(pr * PITCH_) * 4u;
#pragma unroll
    for (int j = 0; j < 5; ++j) {
      if (q + 8 * j < SC) {                               // the fifth column exists for q < 2 only
        const bool ok = rok && cok[j];
        const float *src = ok ? rowp + (long long)gxs[j] * XP : x;
        cp_async_4(drow + (unsigned)(8 * j) * 4u, src, ok ? 4u : 0u);
      }
    }
  }
  cp_async_wait_all();
}

__global__ void __launch_bounds__(THREADS, 4)
narrow_fwd_kernel(const float *__restrict__ x, const float *__restrict__ w, const float *__restrict__ bias,
                  float *__restrict__ y, int H, int W, int C, long long XP, long long YP, int csplit) {
  // rows 38 floats apart: a half-warp's 8-byte reads (two tile rows) fall on disjoint banks;
  // channels 706 = 2 (mod 32) floats apart: the staging stores are conflict-free
  constexpr int CHS = FWD_CHS, FP = FWD_PITCH;
  extern __shared__ __align__(16) float smem[];
  float *xs = smem;                           // [KC][CHS]
  float *ws = smem + KC * CHS;                // [KC][3][8]: co0 kx0..2, co1 kx0..2, 0, 0
  // csplit > 1 (small images: flow4..flow6 have 8..48 tiles for 132 SMs): blockIdx.z also selects a slice of
  // the input channels; the slices' partial sums meet in y (zeroed by the launcher) through atomics
  const int tid = threadIdx.x, n = blockIdx.z / csplit, split = blockIdx.z - n * csplit;
  const int y0 = blockIdx.y * TH, x0 = blockIdx.x * TW;
  const int row = tid >> 3, cg = tid & 7;     // 16 rows x 8 groups of 4 pixels
  float acc0[4] = {0.f, 0.f, 0.f, 0.f}, acc1[4] = {0.f, 0.f, 0.f, 0.f};
  const int chunks = (C + KC - 1) / KC, per = (chunks + csplit - 1) / csplit;
  const int c_begin = split * per * KC, c_end = (split + 1) * per * KC < C ? (split + 1) * per * KC : C;

  for (int c0 = c_begin; c0 < c_end; c0 += KC) {
    __syncthreads();                          // the previous chunk has been consumed
    stage<CHS, FP>(xs, x, n, y0, x0, c0, H, W, C, XP, tid);
    for (int idx = tid; idx < KC * 24; idx += THREADS) {
      const int ch = idx % KC, r = idx / KC, ky = r >> 3, e = r & 7;
      float v = 0.f;
      if (e < 6 && c0 + ch < C) {
        const int co = e / 3, kx = e - co * 3;
        v = __ldg(w + ((long long)(co * 3 + ky) * 3 + kx) * C + c0 + ch);
      }
      ws[(ch * 3 + ky) * 8 + e] = v;
    }
    __syncthreads();
#pragma unroll 2
    for (int ch = 0; ch < KC; ++ch) {
#pragma unroll
      for (int ky = 0; ky < 3; ++ky) {
        const float *xp = xs + ch * CHS + (row + ky) * FP + 4 * cg;
        const float2 a = *reinterpret_cast<const float2 *>(xp);
        const float2 b = *reinterpret_cast<const float2 *>(xp + 2);
        const float2 c = *reinterpret_cast<const float2 *>(xp + 4);
        const float4 wa = *reinterpret_cast<const float4 *>(ws + (ch * 3 + ky) * 8);
        const float4 wb = *reinterpret_cast<const float4 *>(ws + (ch * 3 + ky) * 8 + 4);
        const float xv[6] = {a.x, a.y, b.x, b.y, c.x, c.y};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          acc0[j] = fmaf(xv[j], wa.x, acc0[j]);
          acc0[j] = fmaf(xv[j + 1], wa.y, acc0[j]);
          acc0[j] = fmaf(xv[j + 2], wa.z, acc0[j]);
          acc1[j] = fmaf(xv[j], wa.w, acc1[j]);
          acc1[j] = fmaf(xv[j + 1], wb.x, acc1[j]);
          acc1[j] = fmaf(xv[j + 2], wb.y, acc1[j]);
        }
      }
    }
  }

  const int gy = y0 + row;
  if (gy < H) {
    const float b0 = (bias && split == 0) ? bias[0] : 0.f, b1 = (bias && split == 0) ? bias[1] : 0.f;
    float *out = y + ((long long)n * H + gy) * W * YP;          // YP floats between output pixels (even)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gx = x0 + 4 * cg + j;
      if (gx < W) {
        if (csplit == 1) {
          *reinterpret_cast<float2 *>(out + gx * YP) = make_float2(acc0[j] + b0, acc1[j] + b1);
        } else {
          atomicAdd(out + gx * YP, acc0[j] + b0);
          atomicAdd(out + gx * YP + 1, acc1[j] + b1);
        }
      }
    }
  }
}

__global__ void __launch_bounds__(THREADS, 4)
narrow_wgrad_kernel(const float *__restrict__ x, const float *__restrict__ g, long long gsN, long long gsC,
                    long long gsH, long long gsW, float *__restrict__ partial, int H, int W, int C, long long XP,
                    int csplit) {
  constexpr int CHS = SR * PITCH + 1;         // 649: odd -> lanes on consecutive channels hit distinct banks
  extern __shared__ __align__(16) float smem[];
  float *xs = smem;                           // [KC][CHS]; reused as red[8][KC][NOUT] after the arithmetic
  float *gs = smem + KC * CHS;                // [TH][GPITCH] (even offset: 8-byte aligned float2 reads)
  // csplit > 1: several CTAs per tile, each with its own slice of the input channels (disjoint outputs)
  const int tid = threadIdx.x, n = blockIdx.z / csplit, split = blockIdx.z - n * csplit;
  const int y0 = blockIdx.y * TH, x0 = blockIdx.x * TW;
  const long long bid = ((long long)n * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
  const int chunks = (C + KC - 1) / KC, per = (chunks + csplit - 1) / csplit;
  const int c_begin = split * per * KC, c_end = (split + 1) * per * KC < C ? (split + 1) * per * KC : C;
  const int ch = tid & 15, h = tid >> 4;      // channel, row group (0..7)
  // rows {base, base + 8}; the two row groups of a warp sit 4 rows apart (bank offset 16)
  const int base = (h >> 1) + 4 * (h & 1);

  for (int idx = tid; idx < TH * TW * 2; idx += THREADS) {
    const int co = idx & 1, px = idx >> 1, r = px / TW, c = px - r * TW;
    const int gy = y0 + r, gx = x0 + c;
    float v = 0.f;
    if (gy < H && gx < W) v = __ldg(g + n * gsN + co * gsC + gy * gsH + gx * gsW);
    gs[r * GPITCH + 2 * c + co] = v;
  }

  for (int c0 = c_begin; c0 < c_end; c0 += KC) {
    __syncthreads();                          // red (aliasing xs) has been read; gs is complete
    stage<CHS, PITCH>(xs, x, n, y0, x0, c0, H, W, C, XP, tid);
    __syncthreads();
    float acc0[9], acc1[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) acc0[i] = acc1[i] = 0.f;
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int r = base + 8 * rr;
      const float *xr = xs + ch * CHS + r * PITCH;
      float xw[3][3];
#pragma unroll
      for (int ky = 0; ky < 3; ++ky) {
        xw[ky][0] = xr[ky * PITCH];
        xw[ky][1] = xr[ky * PITCH + 1];
      }
#pragma unroll 4
      for (int c = 0; c < TW; ++c) {
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) xw[ky][2] = xr[ky * PITCH + c + 2];
        const float2 gv = *reinterpret_cast<const float2 *>(gs + r * GPITCH + 2 * c);
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
#pragma unroll
          for (int kx = 0; kx < 3; ++kx) {
            acc0[ky * 3 + kx] = fmaf(gv.x, xw[ky][kx], acc0[ky * 3 + kx]);
            acc1[ky * 3 + kx] = fmaf(gv.y, xw[ky][kx], acc1[ky * 3 + kx]);
          }
          xw[ky][0] = xw[ky][1];
          xw[ky][1] = xw[ky][2];
        }
      }
    }
    __syncthreads();                          // every thread is done reading xs
    float *red = xs;
#pragma unroll
    for (int i = 0; i < 9; ++i) {
      red[(h * KC + ch) * NOUT + i] = acc0[i];
      red[(h * KC + ch) * NOUT + 9 + i] = acc1[i];
    }
    __syncthreads();
    for (int idx = tid; idx < KC * NOUT; idx += THREADS) {
      const int cc = idx % KC, i = idx / KC;
      float s = 0.f;
#pragma unroll
      for (int hh = 0; hh < 8; ++hh) s += red[(hh * KC + cc) * NOUT + i];
      if (c0 + cc < C) partial[(bid * NOUT + i) * C + c0 + cc] = s;
    }
  }
}

// gw[i] = sum over CTAs (fixed order) of partial[b][i];  32 outputs x 8 CTA groups per block
__global__ void __launch_bounds__(256)
narrow_wgrad_reduce_kernel(const float *__restrict__ partial, float *__restrict__ gw, int nblocks, int total) {
  __shared__ float red[8][32];
  const int lane = threadIdx.x & 31, grp = threadIdx.x >> 5;
  const int i = blockIdx.x * 32 + lane;
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  if (i < total) {
    int b = grp;
    for (; b + 24 < nblocks; b += 32) {
      s0 += __ldg(partial + (long long)b * total + i);
      s1 += __ldg(partial + (long long)(b + 8) * total + i);
      s2 += __ldg(partial + (long long)(b + 16) * total + i);
      s3 += __ldg(partial + (long long)(b + 24) * total + i);
    }
    for (; b < nblocks; b += 8) s0 += __ldg(partial + (long long)b * total + i);
  }
  red[grp][lane] = (s0 + s1) + (s2 + s3);
  __syncthreads();
  if (grp == 0 && i < total) {
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) s += red[k][lane];
    gw[i] = s;
  }
}

inline long long tiles(int N, int H, int W) { return (long long)N * ceil_div(H, TH) * ceil_div(W, TW); }

}  // namespace nc
}  // namespace unflow

extern "C" size_t unflow_conv3x3_narrow_wgrad_workspace_bytes(int N, int H, int W, int C) {
  if (N <= 0 || H <= 0 || W <= 0 || C <= 0) return 0;
  return (size_t)unflow::nc::tiles(N, H, W) * unflow::nc::NOUT * (size_t)C * sizeof(float);
}

static int narrow_check(const char *what, int N, int H, int W, int C, int Co) {
  using namespace unflow;
  UNFLOW_REQUIRE(Co == 2, "%s: only 2 output channels (the flow heads) are supported, got %d", what, Co);
  UNFLOW_REQUIRE(N >= 0 && H >= 1 && W >= 1 && C >= 2 && C % 2 == 0, "%s: need H, W >= 1 and an even C", what);
  UNFLOW_REQUIRE(N <= 65535 && ceil_div(H, nc::TH) <= 65535, "%s: grid too large", what);
  return UNFLOW_OK;
}

extern "C" int unflow_conv3x3_narrow_fwd(const float *x, long long x_pitch, const float *w, const float *bias,
                                         float *y, long long y_pitch, int N, int H, int W, int C, int Co,
                                         void *stream) {
  using namespace unflow;
  if (int rc = narrow_check("conv3x3_narrow_fwd", N, H, W, C, Co)) return rc;
  if (N == 0) return UNFLOW_OK;
  UNFLOW_REQUIRE(x && w && y, "conv3x3_narrow_fwd: null pointer");
  UNFLOW_REQUIRE(((uintptr_t)y & 7) == 0, "conv3x3_narrow_fwd: y must be 8-byte aligned");
  UNFLOW_REQUIRE(x_pitch >= C, "conv3x3_narrow_fwd: pixel pitch smaller than C");
  UNFLOW_REQUIRE(y_pitch >= 2 && y_pitch % 2 == 0, "conv3x3_narrow_fwd: output pitch must be even and >= 2");
  // few tiles (the coarse pyramid levels): split the channel range over several CTAs per tile
  const long long tiles = nc::tiles(N, H, W);
  const int chunks = ceil_div(C, nc::KC);
  int csplit = 1;
  if (tiles < 2 * kNumSMs) {
    csplit = (int)((2ll * kNumSMs + tiles - 1) / tiles);
    if (csplit > chunks / 2) csplit = chunks / 2 > 0 ? chunks / 2 : 1;
    if ((long long)N * csplit > 65535) csplit = 65535 / N;
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (csplit > 1) {
    cudaError_t e = cudaMemsetAsync(y, 0, sizeof(float) * (size_t)N * H * W * y_pitch, st);
    if (e != cudaSuccess) { set_error("conv3x3_narrow_fwd memset: %s", cudaGetErrorString(e)); return UNFLOW_ECUDA; }
  }
  // the TMA-staged version (narrow_conv_tma.cu) takes every call it can; it returns -1 for a base or pixel pitch
  // that is not 16-byte aligned, weights that do not fit shared memory or a failed encode, and the cp.async
  // kernel below runs instead
  if (const int rc = narrow_fwd_tma(x, x_pitch, w, bias, y, y_pitch, N, H, W, C, csplit, st); rc >= 0) return rc;
  const dim3 grid(ceil_div(W, nc::TW), ceil_div(H, nc::TH), N * csplit);
  const size_t smem = (size_t)(nc::KC * nc::FWD_CHS + nc::KC * 24) * sizeof(float);
  nc::narrow_fwd_kernel<<<grid, nc::THREADS, smem, st>>>(x, w, bias, y, H, W, C, x_pitch, y_pitch, csplit);
  count_launch();
  return check_launch("conv3x3_narrow_fwd");
}

extern "C" int unflow_conv3x3_narrow_wgrad(const float *x, long long x_pitch, const float *g, long long gsN, long long gsC,
                                           long long gsH, long long gsW, float *gw, void *workspace, int N,
                                           int H, int W, int C, int Co, void *stream) {
  using namespace unflow;
  if (int rc = narrow_check("conv3x3_narrow_wgrad", N, H, W, C, Co)) return rc;
  UNFLOW_REQUIRE(gw, "conv3x3_narrow_wgrad: null pointer");
  cudaStream_t s = (cudaStream_t)stream;
  if (N == 0) {
    cudaError_t e = cudaMemsetAsync(gw, 0, sizeof(float) * nc::NOUT * C, s);
    if (e != cudaSuccess) { set_error("conv3x3_narrow_wgrad memset: %s", cudaGetErrorString(e)); return UNFLOW_ECUDA; }
    return UNFLOW_OK;
  }
  UNFLOW_REQUIRE(x && g && workspace, "conv3x3_narrow_wgrad: null pointer");
  UNFLOW_REQUIRE(x_pitch >= C, "conv3x3_narrow_wgrad: pixel pitch smaller than C");
  const int nblocks = (int)nc::tiles(N, H, W);
  const int chunks = ceil_div(C, nc::KC);
  int csplit = 1;
  if (nblocks < 2 * kNumSMs) {
    csplit = (2 * kNumSMs + nblocks - 1) / nblocks;
    if (csplit > chunks / 2) csplit = chunks / 2 > 0 ? chunks / 2 : 1;
    if ((long long)N * csplit > 65535) csplit = 65535 / N;
  }
  const dim3 grid(ceil_div(W, nc::TW), ceil_div(H, nc::TH), N * csplit);
  const size_t smem = (size_t)(nc::KC * (nc::SR * nc::PITCH + 1) + nc::TH * nc::GPITCH) * sizeof(float);
  float *part = (float *)workspace;
  const int rc_tma = narrow_wgrad_tma(x, x_pitch, g, gsN, gsC, gsH, gsW, part, N, H, W, C, csplit, s);
  if (rc_tma > 0) return rc_tma;
  if (rc_tma < 0) {
    nc::narrow_wgrad_kernel<<<grid, nc::THREADS, smem, s>>>(x, g, gsN, gsC, gsH, gsW, part, H, W, C, x_pitch, csplit);
    count_launch();
    if (int rc = check_launch("conv3x3_narrow_wgrad")) return rc;
  }
  const int total = nc::NOUT * C;
  nc::narrow_wgrad_reduce_kernel<<<ceil_div(total, 32), 256, 0, s>>>((const float *)workspace, gw, nblocks, total);
  count_launch();
  return check_launch("conv3x3_narrow_wgrad_reduce");
}
