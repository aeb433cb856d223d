// conv_fma.cu -- unflow_tc_conv for contractions over at most 4 channels, in exact fp32 on the FMA pipes: the input
// gradients of the flow heads (2 -> C_in of the concat, 3x3) and the flow up-sampling deconvs (2 -> 2, k4 s2, forward
// and input gradient).
//
// On the wgmma kernel such a layer pays a whole 32-channel K block per tap for at most 4 real channels, three MMA
// passes each: at most 495 / 3 * 4 / 32 ~ 21 TFLOP/s of useful work, below the 67 TFLOP/s of the FMA pipes, while
// both paths move the same output bytes.  Here the layer costs what it reads and writes.
//
// Same plan as the wgmma kernel (make_plan, tc_conv_plan.cuh): per output-parity class a list of taps over an
// iteration space of positions,
//     out[n, s_out*iy + py, s_out*ix + px, co] (+)= act( bias[co] +
//         sum_{t in taps(class)} sum_{ci < Cin}  in[n, s_in*iy + dy_t, s_in*ix + dx_t, ci] * W[t.widx][co][ci] )
// with the positions outside the input contributing zero.
//
// Grid: (position blocks, channel blocks, classes).  A CTA stages the weights of its class's taps for its channel
// block once (w_hi + w_lo: exactly the fp32 variable, since lo = w - hi is exact) and then walks batches of
// positions.  A thread owns 4 consecutive output channels -- a warp covers 128 contiguous channels of one pixel --
// of FMA_PIX consecutive positions, whose input loads (one vector load of the Cin channels per pixel and tap) and
// output read-modify-writes are independent and in flight together.  Every output element is written by exactly
// one thread, channels >= Cout never (the output is often a slice of a concat buffer): no atomics, no zero fill, no
// separate epilogue pass, and repeated launches are bit-identical.
//
// Accuracy: each output is a sequential fp32 FMA chain of taps(class) x Cin <= 256 products (in the training step
// at most 9 x 2), so its error is at most about that many units of 2^-24 of the sum of |products|.
#include <algorithm>

#include "tc_conv_plan.cuh"

namespace unflow {
namespace tc {

constexpr int FMA_THREADS = 256;                // most threads per CTA
constexpr int FMA_PIX = 8;                     // positions per thread and batch
constexpr int FMA_SMEM = 48 * 1024;            // staged weights per CTA (no opt-in needed)

struct FmaParams {
  const float *x;
  const float *w_hi, *w_lo;                    // [taps][Cout][4]
  float *y;
  const float *bias;
  int x_pitch, y_pitch;
  int Hin, Win, Hout, Wout, Cout;
  int N, Hit, Wit, s_in, s_out;
  int pixels;                                  // positions per class: N * Hit * Wit
  int G, GB, PB;                               // channel groups of 4; groups per CTA; position lanes per CTA
  float slope;
  int act, accumulate;
  int class_start[5];
  short class_px[4], class_py[4];
  short dx[MAX_TAPS], dy[MAX_TAPS];
  short widx[MAX_TAPS];
};

// the Cin input channels of one pixel in one load (the pixel is 16-byte aligned, its pitch a multiple of 4)
template <int CIN> struct XVec { typedef float4 T; };
template <> struct XVec<1> { typedef float2 T; };
template <> struct XVec<2> { typedef float2 T; };
template <int CIN>
__device__ __forceinline__ float xcomp(const typename XVec<CIN>::T &v, int c);
template <> __device__ __forceinline__ float xcomp<1>(const float2 &v, int c) { return c == 0 ? v.x : v.y; }
template <> __device__ __forceinline__ float xcomp<2>(const float2 &v, int c) { return c == 0 ? v.x : v.y; }
template <> __device__ __forceinline__ float xcomp<3>(const float4 &v, int c) {
  return c == 0 ? v.x : (c == 1 ? v.y : (c == 2 ? v.z : v.w));
}
template <> __device__ __forceinline__ float xcomp<4>(const float4 &v, int c) {
  return c == 0 ? v.x : (c == 1 ? v.y : (c == 2 ? v.z : v.w));
}
__device__ __forceinline__ float wcomp(const float4 &v, int c) {
  return c == 0 ? v.x : (c == 1 ? v.y : (c == 2 ? v.z : v.w));
}

template <int CIN>
__global__ void __launch_bounds__(FMA_THREADS, 2)
conv_fma_kernel(const __grid_constant__ FmaParams p) {
  typedef typename XVec<CIN>::T XV;
  extern __shared__ float4 wsm[];              // [tap of the class][j][GB]: the Cin weights of channel 4 (g0 + g) + j
  const int cls = blockIdx.z;
  const int t0 = p.class_start[cls], nt = p.class_start[cls + 1] - t0;
  const int g0 = blockIdx.y * p.GB;
  for (int i = threadIdx.x; i < nt * 4 * p.GB; i += blockDim.x) {
    const int g = i % p.GB, j = (i / p.GB) & 3, t = i / (4 * p.GB);
    const int co = 4 * (g0 + g) + j;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (co < p.Cout) {
      const long long o = ((long long)p.widx[t0 + t] * p.Cout + co) * 4;
      const float4 h = __ldg(reinterpret_cast<const float4 *>(p.w_hi + o));
      const float4 l = __ldg(reinterpret_cast<const float4 *>(p.w_lo + o));
      v = make_float4(h.x + l.x, h.y + l.y, h.z + l.z, h.w + l.w);
    }
    wsm[i] = v;
  }
  __syncthreads();
  const int g = threadIdx.x % p.GB, pl = threadIdx.x / p.GB;
  if (pl >= p.PB || g0 + g >= p.G) return;
  const int co = 4 * (g0 + g), rem = p.Cout - co;          // rem < 4: the channel tail, stored channel by channel
  const int px = p.class_px[cls], py = p.class_py[cls];
  float b[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) b[j] = p.bias && j < rem ? __ldg(p.bias + co + j) : 0.f;

  const int step = p.PB * FMA_PIX;
  for (int first = blockIdx.x * step + pl * FMA_PIX; first - pl * FMA_PIX < p.pixels; first += gridDim.x * step) {
    // FMA_PIX consecutive positions of the class: (n, iy, ix), n == N past the end
    int n[FMA_PIX], iy[FMA_PIX], ix[FMA_PIX];
    {
      int a = first < p.pixels ? first : p.pixels;
      int x0 = a % p.Wit, r = a / p.Wit, y0 = r % p.Hit, n0 = r / p.Hit;
#pragma unroll
      for (int k = 0; k < FMA_PIX; ++k) {
        n[k] = n0; iy[k] = y0; ix[k] = x0;
        if (n0 < p.N && ++x0 == p.Wit) {
          x0 = 0;
          if (++y0 == p.Hit) { y0 = 0; ++n0; }
        }
      }
    }
    float acc[FMA_PIX][4];
#pragma unroll
    for (int k = 0; k < FMA_PIX; ++k)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[k][j] = 0.f;
    for (int t = 0; t < nt; ++t) {
      const int dx = p.dx[t0 + t], dy = p.dy[t0 + t];
      float4 w[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) w[j] = wsm[(t * 4 + j) * p.GB + g];
      XV xv[FMA_PIX];
#pragma unroll
      for (int k = 0; k < FMA_PIX; ++k) {
        const int yy = p.s_in * iy[k] + dy, xx = p.s_in * ix[k] + dx;
        if (n[k] < p.N && (unsigned)yy < (unsigned)p.Hin && (unsigned)xx < (unsigned)p.Win)
          xv[k] = __ldg(reinterpret_cast<const XV *>(p.x + (long long)((n[k] * p.Hin + yy) * p.Win + xx) * p.x_pitch));
        else
          xv[k] = XV{};
      }
#pragma unroll
      for (int k = 0; k < FMA_PIX; ++k)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int c = 0; c < CIN; ++c) acc[k][j] = fmaf(xcomp<CIN>(xv[k], c), wcomp(w[j], c), acc[k][j]);
    }
    // epilogue: act(bias + sum), then (accumulate) += what y held; the old values of all positions are loaded first
    int opix[FMA_PIX];                        // output pixel, -1 past the end
#pragma unroll
    for (int k = 0; k < FMA_PIX; ++k) {
      opix[k] = n[k] < p.N ? (n[k] * p.Hout + p.s_out * iy[k] + py) * p.Wout + p.s_out * ix[k] + px : -1;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float v = acc[k][j] + b[j];
        if (p.act) v = v > 0.f ? v : p.slope * v;
        acc[k][j] = v;
      }
    }
    auto out = [&](int k) { return p.y + (long long)opix[k] * p.y_pitch + co; };
    if (p.accumulate) {
      float old[FMA_PIX][4];
#pragma unroll
      for (int k = 0; k < FMA_PIX; ++k) {
        old[k][0] = old[k][1] = old[k][2] = old[k][3] = 0.f;
        if (opix[k] < 0) continue;
        const float *o = out(k);
        if (rem >= 4) {
          const float4 v = *reinterpret_cast<const float4 *>(o);
          old[k][0] = v.x; old[k][1] = v.y; old[k][2] = v.z; old[k][3] = v.w;
        } else {
#pragma unroll
          for (int j = 0; j < 3; ++j)
            if (j < rem) old[k][j] = o[j];
        }
      }
#pragma unroll
      for (int k = 0; k < FMA_PIX; ++k)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[k][j] += old[k][j];
    }
#pragma unroll
    for (int k = 0; k < FMA_PIX; ++k) {
      if (opix[k] < 0) continue;
      float *o = out(k);
      if (rem >= 4) {
        *reinterpret_cast<float4 *>(o) = make_float4(acc[k][0], acc[k][1], acc[k][2], acc[k][3]);
      } else {
        // co and the pitch are multiples of 4: o is 16-byte aligned
        if (rem >= 2) *reinterpret_cast<float2 *>(o) = make_float2(acc[k][0], acc[k][1]);
        if (rem == 1) o[0] = acc[k][0];
        if (rem == 3) o[2] = acc[k][2];
      }
    }
  }
}

template <int CIN>
static int launch_fma(const FmaParams &f, dim3 grid, int threads, int smem, cudaStream_t stream) {
  conv_fma_kernel<CIN><<<grid, threads, smem, stream>>>(f);
  count_launch();
  return check_launch("conv_fma_kernel");
}

// CTAs of conv_fma_kernel<CIN> that fit on one SM with `smem` bytes of staged weights
template <int CIN>
static int ctas_per_sm(int smem) {
  static int regs_limit = 0;
  if (!regs_limit) {
    int b = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, conv_fma_kernel<CIN>, FMA_THREADS, 0) != cudaSuccess || b < 1)
      b = 1;
    regs_limit = b;
  }
  const int by_smem = (SMEM_LIMIT - 1024) / (smem + 1024);
  return std::max(1, std::min(regs_limit, by_smem));
}

int conv_fma(const ConvParams &p, const float *x, int Hin, int Win, long long x_pitch, const float *w_hi,
             const float *w_lo, cudaStream_t stream) {
  UNFLOW_REQUIRE(p.Cin >= 1 && p.Cin <= 4 && p.s_in_x == p.s_in_y, "conv_fma: bad plan");
  UNFLOW_REQUIRE((long long)p.N * Hin * Win < (1ll << 30) && (long long)p.N * p.Hout * p.Wout < (1ll << 30) &&
                 x_pitch < (1ll << 31) && p.out_pitch < (1ll << 31), "conv_fma: tensors too large");
  FmaParams f{};
  f.x = x; f.w_hi = w_hi; f.w_lo = w_lo; f.y = p.out; f.bias = p.bias;
  f.x_pitch = (int)x_pitch; f.y_pitch = (int)p.out_pitch;
  f.Hin = Hin; f.Win = Win; f.Hout = p.Hout; f.Wout = p.Wout; f.Cout = p.Cout;
  f.N = p.N; f.Hit = p.Hit; f.Wit = p.Wit; f.s_in = p.s_in_y; f.s_out = p.s_out;
  f.pixels = p.N * p.Hit * p.Wit;
  f.slope = p.slope; f.act = p.act; f.accumulate = p.accumulate;
  int max_nt = 0;
  for (int c = 0; c <= p.n_classes; ++c) f.class_start[c] = p.class_start[c];
  for (int c = 0; c < p.n_classes; ++c) {
    f.class_px[c] = p.class_px[c]; f.class_py[c] = p.class_py[c];
    max_nt = std::max(max_nt, p.class_start[c + 1] - p.class_start[c]);
  }
  for (int t = 0; t < p.class_start[p.n_classes]; ++t) {
    f.dx[t] = p.taps[t].dx; f.dy[t] = p.taps[t].dy; f.widx[t] = (short)p.taps[t].widx;
  }
  // channel blocks: at most 32 groups (128 channels) and FMA_SMEM of weights per CTA, as even as possible
  f.G = (p.Cout + 3) / 4;
  const int gb_max = std::max(1, std::min(32, FMA_SMEM / (max_nt * 4 * 16)));
  const int n_cb = (f.G + gb_max - 1) / gb_max;
  f.GB = (f.G + n_cb - 1) / n_cb;
  const int smem = max_nt * 4 * f.GB * 16;
  // position lanes: FMA_THREADS / GB, halved down to one warp per CTA while the launch would have fewer than two
  // CTAs per SM (the few-pixel layers: more, smaller CTAs spread their positions over more SMs)
  f.PB = FMA_THREADS / f.GB;
  auto batches_of = [&](int pb) { return ((long long)f.pixels + (long long)pb * FMA_PIX - 1) / ((long long)pb * FMA_PIX); };
  while (f.PB * f.GB > 32 && batches_of(f.PB) * n_cb * p.n_classes < 2 * kNumSMs) f.PB = std::max(1, f.PB / 2);
  const int threads = (f.PB * f.GB + 31) / 32 * 32;
  const long long batches = batches_of(f.PB);
  const int per_sm = p.Cin <= 2 ? (p.Cin == 1 ? ctas_per_sm<1>(smem) : ctas_per_sm<2>(smem))
                                : (p.Cin == 3 ? ctas_per_sm<3>(smem) : ctas_per_sm<4>(smem));
  const long long wave = std::max<long long>(1, (long long)kNumSMs * per_sm * (FMA_THREADS / threads) / ((long long)n_cb * p.n_classes));
  const dim3 grid((unsigned)std::min(batches, wave), (unsigned)n_cb, (unsigned)p.n_classes);
  switch (p.Cin) {
    case 1: return launch_fma<1>(f, grid, threads, smem, stream);
    case 2: return launch_fma<2>(f, grid, threads, smem, stream);
    case 3: return launch_fma<3>(f, grid, threads, smem, stream);
    default: return launch_fma<4>(f, grid, threads, smem, stream);
  }
}

}  // namespace tc
}  // namespace unflow
