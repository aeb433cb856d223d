// bias_act.cu -- the leaky-ReLU layer epilogue outside the conv kernels: bias + leaky ReLU in place
// (unflow_bias_lrelu, tc_conv.cu's K-split path) and the activation backward with the bias gradient
// (unflow_lrelu_bwd_bias: gpre = g * lrelu'(act), the operand of the input / weight gradient kernels).
#include "common.cuh"

namespace unflow {

// ---------------------------------------------------------------------------------------------
// Fused bias + leaky ReLU (in place, dense NHWC) and its bias gradient.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
bias_lrelu_kernel(float4 *__restrict__ y, const float *__restrict__ bias, long long n4, int c4n, float slope) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % c4n) * 4;
    float4 v = y[i];
    // the bias is a view into the flat parameter buffer: only 4-byte aligned
    v.x += __ldg(bias + c); v.y += __ldg(bias + c + 1); v.z += __ldg(bias + c + 2); v.w += __ldg(bias + c + 3);
    v.x = v.x > 0.f ? v.x : v.x * slope; v.y = v.y > 0.f ? v.y : v.y * slope;
    v.z = v.z > 0.f ? v.z : v.z * slope; v.w = v.w > 0.f ? v.w : v.w * slope;
    y[i] = v;
  }
}

// gb[c] += sum over pixels of g * lrelu'(act); one CTA = 32 channels x a strip of pixels.
// LINEAR: the gradient is NHWC-like (possibly a channel slice of a wider buffer), so pixel p lives
// at p*pix_stride -- no per-element div/mod (the first version spent most of its time on them).
template <bool LINEAR>
__global__ void __launch_bounds__(256)
bias_grad_lrelu_kernel(const float *__restrict__ g, long long sN, long long sC, long long sH, long long sW,
                       const float *__restrict__ act, float *__restrict__ gb, int N, int C, int H, int W,
                       float slope, int pix_per_cta, float *__restrict__ gpre, long long AP, long long GP) {
  __shared__ float red[8][32];
  const int lane = threadIdx.x & 31, row = threadIdx.x >> 5;
  const int c = blockIdx.y * 32 + lane;
  const long long npix = (long long)N * H * W;
  const long long p0 = (long long)blockIdx.x * pix_per_cta;
  const long long p1 = p0 + pix_per_cta < npix ? p0 + pix_per_cta : npix;
  float s0 = 0.f, s1 = 0.f;
  if (c < C) {
    if (LINEAR) {
      const float *gp = g + c * sC;
      const float *ap = act ? act + c : nullptr;
      long long p = p0 + row;
      for (; p + 8 < p1; p += 16) {           // two independent loads in flight per thread
        float v0 = __ldg(gp + p * sW), v1 = __ldg(gp + (p + 8) * sW);
        if (ap) {
          if (__ldg(ap + p * AP) <= 0.0f) v0 *= slope;
          if (__ldg(ap + (p + 8) * AP) <= 0.0f) v1 *= slope;
        }
        if (gpre) { gpre[p * GP + c] = v0; gpre[(p + 8) * GP + c] = v1; }
        s0 += v0; s1 += v1;
      }
      for (; p < p1; p += 8) {
        float v = __ldg(gp + p * sW);
        if (ap && __ldg(ap + p * AP) <= 0.0f) v *= slope;
        if (gpre) gpre[p * GP + c] = v;
        s0 += v;
      }
    } else {
      for (long long p = p0 + row; p < p1; p += 8) {
        const int x = (int)(p % W);
        const int y = (int)((p / W) % H);
        const long long n = p / ((long long)W * H);
        float v = __ldg(g + n * sN + y * sH + x * sW + c * sC);
        if (act && __ldg(act + p * AP + c) <= 0.0f) v *= slope;
        if (gpre) gpre[p * GP + c] = v;
        s0 += v;
      }
    }
  }
  red[row][lane] = s0 + s1;
  __syncthreads();
  if (row == 0 && c < C) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += red[k][lane];
    atomicAdd(gb + c, t);
  }
}

// Vector form of the LINEAR case (NHWC gradient, channels contiguous, everything 16-byte aligned):
// a lane owns 4 channels (one 128-bit load per tensor and pixel), a warp 128 channels, the 8 warps of a
// CTA walk the pixel strip with two pixels in flight each.  The scalar kernel above reaches 39 % of the
// HBM roofline (one 4-byte load per lane in flight); this one moves 4x the bytes per instruction.
// Layers with fewer than 128 channels (conv1 / deconv2: 64, the largest tensors of the step) would leave
// lanes without channels: `cl` = lanes per pixel (a power of two <= 32, cl * 4 >= min(C, 128)), the other
// 32 / cl lane groups of a warp take the following pixels.
__global__ void __launch_bounds__(256)
bias_grad_lrelu_vec_kernel(const float *__restrict__ g, long long GS, const float *__restrict__ act, long long AP,
                           float *__restrict__ gpre, long long GP, float *__restrict__ gb, int C, long long npix,
                           float slope, int pix_per_cta, int cl) {
  __shared__ float4 red[8][32];
  const int lane = threadIdx.x & 31, row = threadIdx.x >> 5;
  const int sub = 32 / cl;                        // pixels per warp and step
  const int c = blockIdx.y * 128 + (lane & (cl - 1)) * 4;
  const long long p0 = (long long)blockIdx.x * pix_per_cta;
  const long long p1 = p0 + pix_per_cta < npix ? p0 + pix_per_cta : npix;
  const int step = 8 * sub;
  float4 s0 = make_float4(0.f, 0.f, 0.f, 0.f), s1 = s0;
  if (c < C) {                                   // C % 4 == 0: a lane's four channels are all inside or all outside
    long long p = p0 + row * sub + lane / cl;
    for (; p + step < p1; p += 2 * step) {
      float4 v0 = __ldg(reinterpret_cast<const float4 *>(g + p * GS + c));
      float4 v1 = __ldg(reinterpret_cast<const float4 *>(g + (p + step) * GS + c));
      if (act) {
        const float4 a0 = __ldg(reinterpret_cast<const float4 *>(act + p * AP + c));
        const float4 a1 = __ldg(reinterpret_cast<const float4 *>(act + (p + step) * AP + c));
        if (a0.x <= 0.f) v0.x *= slope; if (a0.y <= 0.f) v0.y *= slope; if (a0.z <= 0.f) v0.z *= slope; if (a0.w <= 0.f) v0.w *= slope;
        if (a1.x <= 0.f) v1.x *= slope; if (a1.y <= 0.f) v1.y *= slope; if (a1.z <= 0.f) v1.z *= slope; if (a1.w <= 0.f) v1.w *= slope;
      }
      if (gpre) {
        *reinterpret_cast<float4 *>(gpre + p * GP + c) = v0;
        *reinterpret_cast<float4 *>(gpre + (p + step) * GP + c) = v1;
      }
      s0.x += v0.x; s0.y += v0.y; s0.z += v0.z; s0.w += v0.w;
      s1.x += v1.x; s1.y += v1.y; s1.z += v1.z; s1.w += v1.w;
    }
    for (; p < p1; p += step) {
      float4 v = __ldg(reinterpret_cast<const float4 *>(g + p * GS + c));
      if (act) {
        const float4 a = __ldg(reinterpret_cast<const float4 *>(act + p * AP + c));
        if (a.x <= 0.f) v.x *= slope; if (a.y <= 0.f) v.y *= slope; if (a.z <= 0.f) v.z *= slope; if (a.w <= 0.f) v.w *= slope;
      }
      if (gpre) *reinterpret_cast<float4 *>(gpre + p * GP + c) = v;
      s0.x += v.x; s0.y += v.y; s0.z += v.z; s0.w += v.w;
    }
  }
  red[row][lane] = make_float4(s0.x + s1.x, s0.y + s1.y, s0.z + s1.z, s0.w + s1.w);
  __syncthreads();
  if (row == 0 && lane < cl && c < C) {
    float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int k = 0; k < 8; ++k)
      for (int u = 0; u < sub; ++u) { const float4 r = red[k][lane + u * cl]; t.x += r.x; t.y += r.y; t.z += r.z; t.w += r.w; }
    atomicAdd(gb + c, t.x); atomicAdd(gb + c + 1, t.y); atomicAdd(gb + c + 2, t.z); atomicAdd(gb + c + 3, t.w);
  }
}

}  // namespace unflow

extern "C" int unflow_bias_lrelu(float *y, const float *bias, long long pixels, int C, float slope,
                                 void *stream) {
  using namespace unflow;
  UNFLOW_REQUIRE(pixels >= 0 && C >= 4 && C % 4 == 0, "bias_lrelu: C must be a positive multiple of 4");
  if (pixels == 0) return UNFLOW_OK;
  UNFLOW_REQUIRE(y && bias, "bias_lrelu: null pointer");
  UNFLOW_REQUIRE(((uintptr_t)y & 15) == 0, "bias_lrelu: y must be 16-byte aligned");
  const long long n4 = pixels * (C / 4);
  bias_lrelu_kernel<<<grid_for(n4, 256, 16), 256, 0, (cudaStream_t)stream>>>((float4 *)y, bias, n4, C / 4, slope);
  count_launch();
  return check_launch("bias_lrelu");
}

extern "C" int unflow_lrelu_bwd_bias(const float *g, long long sN, long long sC, long long sH, long long sW,
                                     const float *act, long long act_pitch, float *gpre, long long gpre_pitch,
                                     float *gb, int N, int C, int H, int W, float slope, void *stream);

extern "C" int unflow_bias_grad_lrelu(const float *g, long long sN, long long sC, long long sH,
                                      long long sW, const float *act, float *gb, int N, int C, int H,
                                      int W, float slope, void *stream) {
  return unflow_lrelu_bwd_bias(g, sN, sC, sH, sW, act, C, nullptr, C, gb, N, C, H, W, slope, stream);
}

extern "C" int unflow_lrelu_bwd_bias(const float *g, long long sN, long long sC, long long sH, long long sW,
                                     const float *act, long long act_pitch, float *gpre, long long gpre_pitch,
                                     float *gb, int N, int C, int H, int W, float slope, void *stream) {
  using namespace unflow;
  UNFLOW_REQUIRE(!gpre || gpre_pitch >= C, "lrelu_bwd_bias: gpre pitch smaller than C");
  UNFLOW_REQUIRE(!act || act_pitch >= C, "lrelu_bwd_bias: activation pitch smaller than C");
  UNFLOW_REQUIRE(N >= 0 && C >= 1 && H >= 1 && W >= 1, "bias_grad: bad shape");
  UNFLOW_REQUIRE(g && gb, "bias_grad: null pointer");
  cudaStream_t s = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(gb, 0, sizeof(float) * C, s);
  if (e != cudaSuccess) { set_error("bias_grad memset: %s", cudaGetErrorString(e)); return UNFLOW_ECUDA; }
  const long long npix = (long long)N * H * W;
  if (npix == 0) return UNFLOW_OK;
  const int cblocks = ceil_div(C, 32);
  long long strips = (long long)kNumSMs * 8 / cblocks;
  if (strips < 1) strips = 1;
  int pix_per_cta = (int)((npix + strips - 1) / strips);
  if (pix_per_cta < 64) pix_per_cta = 64;
  dim3 grid(ceil_div(npix, pix_per_cta), cblocks);
  const bool linear = sH == (long long)W * sW && sN == (long long)H * sH;
  const bool vec = linear && sC == 1 && C % 4 == 0 && sW % 4 == 0 && ((uintptr_t)g & 15) == 0 &&
                   (!act || (act_pitch % 4 == 0 && ((uintptr_t)act & 15) == 0)) &&
                   (!gpre || (gpre_pitch % 4 == 0 && ((uintptr_t)gpre & 15) == 0));
  if (vec) {
    const int cb = ceil_div(C, 128);
    long long st = (long long)kNumSMs * 8 / cb;
    if (st < 1) st = 1;
    int ppc = (int)((npix + st - 1) / st);
    if (ppc < 64) ppc = 64;
    dim3 vgrid(ceil_div(npix, ppc), cb);
    int cl = 32;                                  // lanes per pixel: the smallest power of two covering min(C, 128) / 4
    while (cl > 1 && (cl / 2) * 4 >= (C < 128 ? C : 128)) cl /= 2;
    bias_grad_lrelu_vec_kernel<<<vgrid, 256, 0, s>>>(g, sW, act, act_pitch, gpre, gpre_pitch, gb, C, npix, slope, ppc, cl);
    count_launch();
    return check_launch("bias_grad_lrelu(vec)");
  }
  if (linear) bias_grad_lrelu_kernel<true><<<grid, 256, 0, s>>>(g, sN, sC, sH, sW, act, gb, N, C, H, W, slope, pix_per_cta, gpre, act_pitch, gpre_pitch);
  else bias_grad_lrelu_kernel<false><<<grid, 256, 0, s>>>(g, sN, sC, sH, sW, act, gb, N, C, H, W, slope, pix_per_cta, gpre, act_pitch, gpre_pitch);
  count_launch();
  return check_launch("bias_grad_lrelu");
}
