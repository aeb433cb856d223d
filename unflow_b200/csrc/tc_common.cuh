// tc_common.cuh -- PTX wrappers (mbarrier, TMA, wgmma) and the tensor-map encoder shared by the tensor-core
// kernels (tc_conv.cu: forward / input gradient, tc_wgrad.cu: weight gradient).
#pragma once
#include <cuda.h>

#include "common.cuh"

namespace unflow {
namespace tc {

constexpr int BM = 128;          // rows of a tile: two consumer warpgroups of 64 rows (the wgmma M)
constexpr int BK = 32;           // fp32 elements per K block = 128 bytes = one swizzle row
// K blocks accumulated by wgmma in one register accumulator before it is added, with round to nearest, to a
// second fp32 register accumulator (default of the "tc_chunk" option).  A tensor-core accumulation adds with
// truncation, an error that grows linearly with K; cutting K into chunks bounds it (tc_conv.cu, "Accuracy").
constexpr int CHUNK = 8;
constexpr int A_BYTES = BM * BK * 4;   // 16 KB
extern long long *g_dbg;               // tc_conv.cu: role-timer buffer (unflow_tc_conv_debug)
extern int g_chunk;                    // tc_conv.cu: K blocks per wgmma accumulation between register adds (default CHUNK)

// ------------------------------------------------------------------------------------------
// PTX helpers
// ------------------------------------------------------------------------------------------
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
__device__ __forceinline__ void tma_4d(unsigned dst, const CUtensorMap *map, unsigned bar, int c0, int c1,
                                       int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_3d(unsigned dst, const CUtensorMap *map, unsigned bar, int c0, int c1,
                                       int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// barrier over `count` threads (whole warps) with hardware barrier `id` (0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

__device__ __forceinline__ float tf32_rna(float x) {
  unsigned u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}
// The same rounding (to nearest, ties away from zero) on the integer pipes without cvt's NaN / Inf handling:
// 2 instead of 4 instructions per element in the split (activations and gradients are finite).
__device__ __forceinline__ float tf32_rna_fast(float x) {
  return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u);
}
__device__ __forceinline__ float4 tf32_hi4(float4 v) {
  return make_float4(tf32_rna_fast(v.x), tf32_rna_fast(v.y), tf32_rna_fast(v.z), tf32_rna_fast(v.w));
}
__device__ __forceinline__ float4 sub4(float4 a, float4 b) { return make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w); }

__device__ __forceinline__ void red_add_f32(float *addr, float v) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(addr), "f"(v) : "memory");
}

// ---- wgmma (sm_90a warpgroup MMA) ----------------------------------------------------------------
// K-major operand tile in the 128-byte swizzle (what TMA writes with CU_TENSOR_MAP_SWIZZLE_128B): rows of
// 128 B = 32 tf32, 16-byte chunk j of row r stored at chunk j ^ (r & 7), 8-row atoms of 1024 B (stride byte
// offset), layout type 1 = SWIZZLE_128B.  The tile must start 1024-byte aligned; one K step of 8 tf32 is
// +32 bytes on the start address (+2 in the descriptor's 16-byte units).
__device__ __forceinline__ unsigned long long wgmma_desc_k128(unsigned saddr) {
  return (unsigned long long)((saddr >> 4) & 0x3FFFu) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
// byte offset of element (row r, k) in such a tile
__device__ __forceinline__ unsigned sw128_offset(int r, int k) {
  return (unsigned)(r * 128 + ((((k >> 2) ^ (r & 7)) & 7) << 4) + ((k & 3) << 2));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving reads / writes of the accumulator registers across a wgmma fence or wait
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x N] (+)= A[64 x 8] * B[N x 8]^T, tf32 inputs from shared memory (K-major descriptors), fp32 accumulators
// in registers.  Thread t of the warpgroup holds rows 16 * (t / 32) + (t % 32) / 4 (+ 8) and, in d[4j .. 4j + 3],
// columns 8j + 2 (t % 4) (+ 1): d[4j + 2h + e] = D[row + 8h][8j + 2 (t % 4) + e].
template <int N> struct Wgmma;
template <> struct Wgmma<32> {
  static __device__ __forceinline__ void mma(float (&d)[16], unsigned long long da, unsigned long long db, int scale_d) {
    asm volatile(
        "{\n .reg .pred p;\n setp.ne.b32 p, %18, 0;\n"
        " wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(scale_d));
  }
};
template <> struct Wgmma<64> {
  static __device__ __forceinline__ void mma(float (&d)[32], unsigned long long da, unsigned long long db, int scale_d) {
    asm volatile(
        "{\n .reg .pred p;\n setp.ne.b32 p, %34, 0;\n"
        " wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d));
  }
};
template <> struct Wgmma<128> {
  static __device__ __forceinline__ void mma(float (&d)[64], unsigned long long da, unsigned long long db, int scale_d) {
    asm volatile(
        "{\n .reg .pred p;\n setp.ne.b32 p, %66, 0;\n"
        " wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(scale_d));
  }
};

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
inline int encode(CUtensorMap *m, const float *basep, int rank, const cuuint64_t *dims,
                  const cuuint64_t *strides_bytes, const cuuint32_t *box, const cuuint32_t *estr,
                  CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
  if (bind_primary_context()) return UNFLOW_ECUDA;
  EncodeTiledFn fn = encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled entry point not available"); return UNFLOW_ECUDA; }
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, (void *)basep, dims, strides_bytes, box,
                  estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d)", (int)r); return UNFLOW_ECUDA; }
  return UNFLOW_OK;
}

}  // namespace tc
}  // namespace unflow
