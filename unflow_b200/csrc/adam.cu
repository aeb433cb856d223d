// adam.cu -- one fused Adam update over the flat parameter buffer of the data-parallel step.
//
// The reference uses tf.train.AdamOptimizer(beta1=0.9, beta2=0.999) (src/e2eflow/core/train.py:
// 151-152; TF default epsilon 1e-8) and averages tower gradients on the CPU (train.py:388-422).
// Here all trainable variables live in ONE contiguous fp32 buffer (so the gradient mean is one
// NCCL all-reduce) and the update is one pass: TF's formulation
//     lr_t = lr * sqrt(1 - beta2^t) / (1 - beta1^t)
//     m <- beta1*m + (1-beta1)*g ;  v <- beta2*v + (1-beta2)*g^2 ;  p <- p - lr_t * m / (sqrt(v) + eps)
// The gradient is cleared in the same pass (it is accumulated into by the next backward), which
// saves a separate 157 MB memset.  HBM-bound: 16 B read + 16 B written per parameter.
#include "common.cuh"

namespace unflow {

// hyper (device, optional): [lr, beta1, beta2, eps, grad_scale, step] -- read at run time so that a
// CUDA graph of the whole training step can be replayed: the step counter lives on the device and
// is advanced by a one-thread kernel after the update, the host only rewrites `lr` when the
// schedule changes it.
//
// l2mask / l2 (optional): slim.l2_regularizer on the `weights` variables (flownet.py:176,200,218) adds
// l2 * w to their gradient.  One bit per parameter (bits 0-3 of byte i for the float4 i) marks the
// regularised elements; the term is added here, after the gradient mean -- (sum_r g_r) / N + l2 * w is what
// every tower's own `g_r + l2 * w` averages to -- instead of as 36 scaled copies of the weights that autograd
// then adds to the gradients (0.17 ms per step).
__global__ void __launch_bounds__(256)
adam_kernel(float4 *__restrict__ p, float4 *__restrict__ g, float4 *__restrict__ m,
            float4 *__restrict__ v, long long n4, float lr_t, float b1, float b2, float eps,
            float grad_scale, int zero_grad, const float *__restrict__ hyper,
            const unsigned char *__restrict__ l2mask, float l2) {
  if (hyper) {
    b1 = __ldg(hyper + 1); b2 = __ldg(hyper + 2); eps = __ldg(hyper + 3);
    grad_scale = __ldg(hyper + 4);
    // in double, as unflow_adam_step_l2 forms it on the host: in fp32, 1 - powf(0.999f, t) cancels the rounding
    // of the power into a 3e-6 error of lr_t from t = 2 on
    const double t = __ldg(hyper + 5);
    lr_t = (float)((double)__ldg(hyper) * sqrt(1.0 - pow((double)b2, t)) / (1.0 - pow((double)b1, t)));
  }
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    float4 pp = p[i], gg = g[i], mm = m[i], vv = v[i];
    const unsigned mk = l2mask ? (unsigned)__ldg(l2mask + i) : 0u;
    const float l2x = (mk & 1u) ? l2 : 0.f, l2y = (mk & 2u) ? l2 : 0.f, l2z = (mk & 4u) ? l2 : 0.f, l2w = (mk & 8u) ? l2 : 0.f;
#define UNFLOW_ADAM1(c)                                     \
    {                                                       \
      const float gr = gg.c * grad_scale + l2##c * pp.c;    \
      mm.c = b1 * mm.c + (1.0f - b1) * gr;                  \
      vv.c = b2 * vv.c + (1.0f - b2) * gr * gr;             \
      pp.c = pp.c - lr_t * mm.c / (sqrtf(vv.c) + eps);      \
    }
    UNFLOW_ADAM1(x) UNFLOW_ADAM1(y) UNFLOW_ADAM1(z) UNFLOW_ADAM1(w)
#undef UNFLOW_ADAM1
    p[i] = pp; m[i] = mm; v[i] = vv;
    if (zero_grad) g[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

__global__ void adam_advance_kernel(float *step) { *step += 1.0f; }

}  // namespace unflow

extern "C" int unflow_adam_step_l2(float *params, float *grads, float *m, float *v, long long n,
                                   float lr, float beta1, float beta2, float eps, long long step,
                                   float grad_scale, int zero_grad, const unsigned char *l2mask, float l2,
                                   void *stream);
extern "C" int unflow_adam_step(float *params, float *grads, float *m, float *v, long long n,
                                float lr, float beta1, float beta2, float eps, long long step,
                                float grad_scale, int zero_grad, void *stream) {
  return unflow_adam_step_l2(params, grads, m, v, n, lr, beta1, beta2, eps, step, grad_scale, zero_grad, nullptr,
                             0.f, stream);
}

extern "C" int unflow_adam_step_l2(float *params, float *grads, float *m, float *v, long long n,
                                   float lr, float beta1, float beta2, float eps, long long step,
                                   float grad_scale, int zero_grad, const unsigned char *l2mask, float l2,
                                   void *stream) {
  using namespace unflow;
  UNFLOW_REQUIRE(n >= 0 && n % 4 == 0, "adam: the flat buffer length must be a multiple of 4");
  UNFLOW_REQUIRE(step >= 1, "adam: step counts from 1");
  if (n == 0) return UNFLOW_OK;
  UNFLOW_REQUIRE(params && grads && m && v, "adam: null pointer");
  UNFLOW_REQUIRE((((uintptr_t)params | (uintptr_t)grads | (uintptr_t)m | (uintptr_t)v) & 15) == 0,
                 "adam: buffers must be 16-byte aligned");
  const double lr_t = (double)lr * sqrt(1.0 - pow((double)beta2, (double)step)) /
                      (1.0 - pow((double)beta1, (double)step));
  const long long n4 = n / 4;
  adam_kernel<<<grid_for(n4, 256, 8), 256, 0, (cudaStream_t)stream>>>(
      (float4 *)params, (float4 *)grads, (float4 *)m, (float4 *)v, n4, (float)lr_t, beta1, beta2, eps,
      grad_scale, zero_grad, nullptr, l2mask, l2);
  count_launch();
  return check_launch("adam_step");
}

extern "C" int unflow_adam_step_dev_l2(float *params, float *grads, float *m, float *v, long long n,
                                       float *hyper, int zero_grad, const unsigned char *l2mask, float l2,
                                       void *stream);
extern "C" int unflow_adam_step_dev(float *params, float *grads, float *m, float *v, long long n,
                                    float *hyper, int zero_grad, void *stream) {
  return unflow_adam_step_dev_l2(params, grads, m, v, n, hyper, zero_grad, nullptr, 0.f, stream);
}

extern "C" int unflow_adam_step_dev_l2(float *params, float *grads, float *m, float *v, long long n,
                                       float *hyper, int zero_grad, const unsigned char *l2mask, float l2,
                                       void *stream) {
  using namespace unflow;
  UNFLOW_REQUIRE(n >= 0 && n % 4 == 0, "adam: the flat buffer length must be a multiple of 4");
  if (n == 0) return UNFLOW_OK;
  UNFLOW_REQUIRE(params && grads && m && v && hyper, "adam: null pointer");
  UNFLOW_REQUIRE((((uintptr_t)params | (uintptr_t)grads | (uintptr_t)m | (uintptr_t)v) & 15) == 0,
                 "adam: buffers must be 16-byte aligned");
  const long long n4 = n / 4;
  adam_kernel<<<grid_for(n4, 256, 8), 256, 0, (cudaStream_t)stream>>>(
      (float4 *)params, (float4 *)grads, (float4 *)m, (float4 *)v, n4, 0.f, 0.f, 0.f, 0.f, 0.f, zero_grad, hyper,
      l2mask, l2);
  adam_advance_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(hyper + 5);
  count_launch(2);
  return check_launch("adam_step_dev");
}
