// supervised_loss.cu -- the supervised fine-tuning loss of one network, fused.
//
// Replaces the graph of supervised_loss (reference src/e2eflow/core/supervised.py:45-57) for one
// network of the stack:
//   final = resize_bilinear(flow, [H, W]) * scale          (legacy TF kernel; scale = FLOW_SCALE * 4)
//   loss  = charbonnier_loss(final - flow_gt, mask_gt)     (losses.py:298-323)
//         = sum(mask * ((final - gt)^2 + 0.001^2)^0.45) / (B*H*W*2)
// The upsampled flow is never written to memory.  The forward kernel evaluates one full-resolution
// pixel (both channels) per thread and reduces deterministically (per-CTA partials in double, the
// last CTA sums them in a fixed order).  The backward kernel writes d loss / d flow [B,h,w,2]
// directly as a GATHER: one thread per coarse pixel sums, in a fixed order, the gradient of every
// full-resolution pixel whose interpolation reads it, times the interpolation weight.  No float
// atomics, so two runs are bit-identical.
//
// Resize mapping (tf.image.resize_bilinear, align_corners=False, no half-pixel centres), per axis:
//   s = float32(h / H);  src = float32(Y) * s;  lo = floor(src);  hi = min(ceil(src), h - 1);
//   lerp = src - lo.
// Any ratio h / H is allowed (1 for full_res networks, non-integer for odd sizes).  On the last
// coarse row / column lo == hi, which then receives both lerp weights.
//
// HBM-bound: algorithmic bytes fwd = 4*B*H*W*3 (flow_gt, mask) + 4*B*h*w*2 (flow);
// bwd = the same + 4*B*h*w*2 (dflow).  The gathers of the coarse flow and the overlapping
// full-resolution windows of neighbouring coarse pixels hit L1.
#include "common.cuh"

namespace unflow {
namespace sl {

constexpr int FWD_THREADS = 256;
constexpr int BX = 32, BY = 8;     // backward CTA: 32 x 8 coarse pixels
constexpr float kEps2 = 1e-6f;     // epsilon^2, epsilon = 0.001
constexpr float kAlpha = 0.45f;

struct Axis {
  int lo, hi;
  float lerp;
};

// tf_image._bilinear_axis: float32 source coordinate of output index i
__device__ __forceinline__ Axis axis_map(int i, float s, int n_in) {
  const float src = __fmul_rn((float)i, s);
  const float f = floorf(src);
  Axis a;
  a.lo = (int)f;
  a.hi = min((int)ceilf(src), n_in - 1);
  a.lerp = __fsub_rn(src, f);
  return a;
}

// ((x)^2 + eps^2)^alpha: the argument is >= 1e-6 > 0, so pow is exp2(alpha * log2(.))
__device__ __forceinline__ float pow_pos(float x, float a) { return exp2f(a * __log2f(x)); }

// the upsampled, scaled flow at full-resolution pixel (Y, X) of image b, op by op as
// top = tl + (tr - tl) * lx;  bot = bl + (br - bl) * lx;  v = top + (bot - top) * ly;  v * scale
__device__ __forceinline__ float2 upsample(const float2 *f, int w, const Axis &ay, const Axis &ax, float scale) {
  const float2 tl = __ldg(f + ay.lo * w + ax.lo), tr = __ldg(f + ay.lo * w + ax.hi);
  const float2 bl = __ldg(f + ay.hi * w + ax.lo), br = __ldg(f + ay.hi * w + ax.hi);
  float2 v;
  {
    const float top = __fadd_rn(tl.x, __fmul_rn(__fsub_rn(tr.x, tl.x), ax.lerp));
    const float bot = __fadd_rn(bl.x, __fmul_rn(__fsub_rn(br.x, bl.x), ax.lerp));
    v.x = __fmul_rn(__fadd_rn(top, __fmul_rn(__fsub_rn(bot, top), ay.lerp)), scale);
  }
  {
    const float top = __fadd_rn(tl.y, __fmul_rn(__fsub_rn(tr.y, tl.y), ax.lerp));
    const float bot = __fadd_rn(bl.y, __fmul_rn(__fsub_rn(br.y, bl.y), ax.lerp));
    v.y = __fmul_rn(__fadd_rn(top, __fmul_rn(__fsub_rn(bot, top), ay.lerp)), scale);
  }
  return v;
}

struct Params {
  const float *flow, *gt, *mask;   // [B,h,w,2], [B,H,W,2], [B,H,W,1] or null
  const float *grad_loss;          // bwd: d L / d loss (device scalar)
  float *loss, *dflow;
  double *partials;                // fwd: [gridDim.x]
  unsigned *counter;
  int B, h, w, H, W;
  float sy, sx, scale;
};

__global__ void __launch_bounds__(FWD_THREADS)
supervised_loss_fwd_kernel(Params p) {
  __shared__ double sred[FWD_THREADS / 32];
  __shared__ bool s_last;
  const long long hw = (long long)p.H * p.W, n = hw * p.B;
  double acc = 0.0;
  for (long long q = (long long)blockIdx.x * FWD_THREADS + threadIdx.x; q < n;
       q += (long long)gridDim.x * FWD_THREADS) {
    const int b = (int)(q / hw);
    const int r = (int)(q - (long long)b * hw);
    const int Y = r / p.W, X = r - Y * p.W;
    const Axis ay = axis_map(Y, p.sy, p.h), ax = axis_map(X, p.sx, p.w);
    const float2 v = upsample(reinterpret_cast<const float2 *>(p.flow) + (long long)b * p.h * p.w, p.w, ay, ax,
                              p.scale);
    const float2 g = __ldg(reinterpret_cast<const float2 *>(p.gt) + q);
    const float m = p.mask ? __ldg(p.mask + q) : 1.0f;
    const float dx = __fsub_rn(v.x, g.x), dy = __fsub_rn(v.y, g.y);
    const float e = pow_pos(__fadd_rn(__fmul_rn(dx, dx), kEps2), kAlpha) +
                    pow_pos(__fadd_rn(__fmul_rn(dy, dy), kEps2), kAlpha);
    acc += (double)(m * e);
  }
  // warp shuffle -> CTA -> per-CTA partial -> the last CTA sums all partials in a fixed order
  const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, off);
  if (lane == 0) sred[wrp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double v = 0.0;
    for (int i = 0; i < FWD_THREADS / 32; ++i) v += sred[i];
    p.partials[blockIdx.x] = v;
    __threadfence();
    const unsigned ticket = atomicAdd(p.counter, 1u);
    s_last = (ticket == gridDim.x - 1);
  }
  __syncthreads();
  if (s_last && wrp == 0) {
    __threadfence();
    double v = 0.0;
    for (int i = lane; i < (int)gridDim.x; i += 32) v += __ldcg(p.partials + i);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += __shfl_down_sync(0xffffffffu, v, off);
    if (lane == 0) {
      *p.loss = (float)(v / ((double)n * 2.0));
      *p.counter = 0u;
    }
  }
}

// Weight with which full-resolution index i (mapped to `a`) reads coarse index j; 0 if it does not.
__device__ __forceinline__ float tap_weight(const Axis &a, int j) {
  float wgt = 0.0f;
  if (a.lo == j) wgt += 1.0f - a.lerp;
  if (a.hi == j) wgt += a.lerp;
  return wgt;
}

// Full-resolution indices that can read coarse index j: src = i * s in (j - 1, j + 1), padded by one
// on both sides against the rounding of the float32 product (tap_weight decides exactly).
__device__ __forceinline__ void gather_range(int j, float s, int n_out, int &first, int &last) {
  const double sd = (double)s;
  first = max(0, (int)floor((double)(j - 1) / sd) - 1);
  last = min(n_out - 1, (int)ceil((double)(j + 1) / sd) + 1);
}

__global__ void __launch_bounds__(BX * BY)
supervised_loss_bwd_kernel(Params p) {
  const int i = blockIdx.x * BX + threadIdx.x, j = blockIdx.y * BY + threadIdx.y, b = blockIdx.z;
  if (i >= p.w || j >= p.h) return;
  // u = dL/dloss * scale / N: the chain through `final = v * scale` and the mean
  const float u = (float)((double)__ldg(p.grad_loss) * (double)p.scale / ((double)p.B * p.H * p.W * 2.0));
  const float2 *f = reinterpret_cast<const float2 *>(p.flow) + (long long)b * p.h * p.w;
  const long long base = (long long)b * p.H * p.W;
  const float2 *gt = reinterpret_cast<const float2 *>(p.gt) + base;
  const float *mk = p.mask ? p.mask + base : nullptr;
  int y0, y1, x0, x1;
  gather_range(j, p.sy, p.H, y0, y1);
  gather_range(i, p.sx, p.W, x0, x1);
  float gx = 0.0f, gy = 0.0f;
  for (int Y = y0; Y <= y1; ++Y) {
    const Axis ay = axis_map(Y, p.sy, p.h);
    const float wy = tap_weight(ay, j);
    if (wy == 0.0f) continue;
    for (int X = x0; X <= x1; ++X) {
      const Axis ax = axis_map(X, p.sx, p.w);
      const float wx = tap_weight(ax, i);
      if (wx == 0.0f) continue;
      const int q = Y * p.W + X;
      const float m = mk ? __ldg(mk + q) : 1.0f;
      if (m == 0.0f) continue;
      const float2 v = upsample(f, p.w, ay, ax, p.scale);
      const float2 g = __ldg(gt + q);
      const float dx = v.x - g.x, dy = v.y - g.y;
      // d/dx (x^2 + eps^2)^alpha = 2 alpha x (x^2 + eps^2)^(alpha - 1)
      const float cx = 2.0f * kAlpha * dx * pow_pos(dx * dx + kEps2, kAlpha - 1.0f);
      const float cy = 2.0f * kAlpha * dy * pow_pos(dy * dy + kEps2, kAlpha - 1.0f);
      const float wgt = wy * wx * m;
      gx += wgt * cx;
      gy += wgt * cy;
    }
  }
  reinterpret_cast<float2 *>(p.dflow)[((long long)b * p.h + j) * p.w + i] = make_float2(u * gx, u * gy);
}

static int check_shape(int B, int h, int w, int H, int W) {
  UNFLOW_REQUIRE(B >= 1 && h >= 1 && w >= 1 && H >= 1 && W >= 1, "supervised_loss: bad shape");
  UNFLOW_REQUIRE(B <= 65535 && h <= 65535 * BY, "supervised_loss: batch or height too large");
  UNFLOW_REQUIRE((long long)H * W * 2 < (1ll << 31) && (long long)h * w * 2 < (1ll << 31),
                 "supervised_loss: image too large");
  return UNFLOW_OK;
}

static int fwd_grid(int B, int H, int W) { return grid_for((long long)B * H * W, FWD_THREADS); }

static void fill(Params &p, const float *flow, const float *gt, const float *mask, int B, int h, int w, int H,
                 int W, float scale) {
  p.flow = flow; p.gt = gt; p.mask = mask;
  p.B = B; p.h = h; p.w = w; p.H = H; p.W = W; p.scale = scale;
  p.sy = (float)((double)h / (double)H);
  p.sx = (float)((double)w / (double)W);
}

}  // namespace sl
}  // namespace unflow

using namespace unflow;
using namespace unflow::sl;

extern "C" size_t unflow_supervised_loss_workspace_bytes(int B, int H, int W) {
  if (B < 1 || H < 1 || W < 1) return 0;
  return (size_t)fwd_grid(B, H, W) * sizeof(double) + 256;
}

extern "C" int unflow_supervised_loss_fwd(const float *flow, const float *flow_gt, const float *mask_gt,
                                          float *loss, void *workspace, int B, int h, int w, int H, int W,
                                          float scale, void *stream) {
  int rc = check_shape(B, h, w, H, W);
  if (rc) return rc;
  UNFLOW_REQUIRE(flow && flow_gt && loss && workspace, "supervised_loss: null pointer");
  Params p{};
  fill(p, flow, flow_gt, mask_gt, B, h, w, H, W, scale);
  const int grid = fwd_grid(B, H, W);
  p.loss = loss;
  p.partials = (double *)workspace;
  p.counter = (unsigned *)((char *)workspace + (size_t)grid * sizeof(double));
  cudaStream_t s = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(p.counter, 0, sizeof(unsigned), s);
  if (e != cudaSuccess) { set_error("supervised_loss memset: %s", cudaGetErrorString(e)); return UNFLOW_ECUDA; }
  supervised_loss_fwd_kernel<<<grid, FWD_THREADS, 0, s>>>(p);
  count_launch();
  return check_launch("supervised_loss_fwd");
}

extern "C" int unflow_supervised_loss_bwd(const float *grad_loss, const float *flow, const float *flow_gt,
                                          const float *mask_gt, float *dflow, int B, int h, int w, int H, int W,
                                          float scale, void *stream) {
  int rc = check_shape(B, h, w, H, W);
  if (rc) return rc;
  UNFLOW_REQUIRE(grad_loss && flow && flow_gt && dflow, "supervised_loss_grad: null pointer");
  Params p{};
  fill(p, flow, flow_gt, mask_gt, B, h, w, H, W, scale);
  p.grad_loss = grad_loss;
  p.dflow = dflow;
  dim3 grid(ceil_div(w, BX), ceil_div(h, BY), B), block(BX, BY);
  supervised_loss_bwd_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(p);
  count_launch();
  return check_launch("supervised_loss_bwd");
}
