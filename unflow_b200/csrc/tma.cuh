// tma.cuh -- PTX wrappers for mbarriers and TMA loads, and the tensor-map encoder, shared by every kernel that
// stages its tiles with TMA (correlation_tiled.cu, narrow_conv_tma.cu, tc_conv.cu, tc_wgrad.cu).
#pragma once
#include <cuda.h>

#include "common.cuh"

namespace unflow {
namespace tc {

__device__ __forceinline__ unsigned s32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(unsigned bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(unsigned bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned bar, unsigned parity) {
  unsigned done;
  do {
    asm volatile(
        "{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        " selp.u32 %0, 1, 0, p;\n}\n"
        : "=r"(done) : "r"(bar), "r"(parity) : "memory");
  } while (!done);
}
// One lane of a fully converged warp (elect.sync): the TMA producer runs its loop with all lanes converged and
// issues under this predicate.
__device__ __forceinline__ bool elect_one() {
  unsigned pred = 0;
  asm volatile("{\n .reg .pred p;\n elect.sync _|p, 0xFFFFFFFF;\n selp.u32 %0, 1, 0, p;\n}\n" : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void tma_3d(unsigned dst, const CUtensorMap *map, unsigned bar, int c0, int c1,
                                       int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_4d(unsigned dst, const CUtensorMap *map, unsigned bar, int c0, int c1,
                                       int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_5d(unsigned dst, const CUtensorMap *map, unsigned bar, int c0, int c1,
                                       int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---- host: tensor maps --------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);
inline EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void *ptr = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)ptr;
  }
  return fn;
}

// cuTensorMapEncodeTiled is a driver-API call and needs a current context on the calling thread.  A host thread
// whose first CUDA work is a launcher of this library (autograd's backward worker, for one) has none until a
// runtime call binds the device's primary context, and the encode then fails with CUDA_ERROR_INVALID_CONTEXT.
// cudaSetDevice binds it.
inline int bind_primary_context() {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaSetDevice(dev);
  if (e != cudaSuccess) {
    set_error("cannot make the device's primary context current: %s", cudaGetErrorString(e));
    return UNFLOW_ECUDA;
  }
  return UNFLOW_OK;
}

inline int encode(CUtensorMap *m, const float *basep, int rank, const cuuint64_t *dims,
                  const cuuint64_t *strides_bytes, const cuuint32_t *box, const cuuint32_t *estr,
                  CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B,
                  CUtensorMapL2promotion l2 = CU_TENSOR_MAP_L2_PROMOTION_L2_256B) {
  if (bind_primary_context()) return UNFLOW_ECUDA;
  EncodeTiledFn fn = encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled entry point not available"); return UNFLOW_ECUDA; }
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, (void *)basep, dims, strides_bytes, box,
                  estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, l2, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d)", (int)r); return UNFLOW_ECUDA; }
  return UNFLOW_OK;
}

}  // namespace tc
}  // namespace unflow
