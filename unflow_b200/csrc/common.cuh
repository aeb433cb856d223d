// common.cuh -- shared host/device helpers for libunflow.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cstdarg>
#include <cstdint>
#include <cstdio>

#include "../../include/unflow.h"

namespace unflow {

// thread-local last-error string (unflow_last_error)
void set_error(const char *fmt, ...);
// every launcher calls this once per kernel it enqueues
void count_launch(int n = 1);

inline int check_launch(const char *what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    return UNFLOW_ECUDA;
  }
  return UNFLOW_OK;
}

#define UNFLOW_REQUIRE(cond, ...)      \
  do {                                 \
    if (!(cond)) {                     \
      ::unflow::set_error(__VA_ARGS__);\
      return UNFLOW_EINVAL;            \
    }                                  \
  } while (0)

constexpr int kNumSMs = 132;  // H100 SXM

inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

// grid size for a grid-stride pixel-parallel kernel: enough CTAs to fill the
// SMs a whole number of times, capped by the work available.
inline int grid_for(long long work_items, int threads, int ctas_per_sm = 8) {
  long long need = (work_items + threads - 1) / threads;
  long long cap = (long long)kNumSMs * ctas_per_sm;
  if (need < 1) need = 1;
  return (int)(need < cap ? need : cap);
}

}  // namespace unflow
