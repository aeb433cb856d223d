// correlation.cuh -- shared declarations of the correlation translation units.
#pragma once
#include "common.cuh"

namespace unflow {

// ops/correlation_op.h:28-52 (CorrelationState)
struct CorrGeom {
  int B, C, H, W;
  int ks, md, pad, s1, s2;
  int kr, border, ngr, ngw;
  int oh, ow, oc;
};

int make_corr_geom(CorrGeom &g, int B, int C, int H, int W, int ks, int md, int pad, int s1, int s2);

int corr_fwd_generic(const float *in0, const float *in1, float *out, const CorrGeom &g, cudaStream_t s);
int corr_bwd_generic(const float *gout, const float *in0, const float *in1, float *g0, float *g1,
                     const CorrGeom &g, cudaStream_t s);

// correlation_tiled.cu
bool corr_tiled_supported(const CorrGeom &g);
int corr_fwd_tiled(const float *in0, const float *in1, float *out, float *out_rev, const CorrGeom &g,
                   cudaStream_t s);
int corr_fold_grad(const float *gout, const float *gout_rev, float *geff, const CorrGeom &g, cudaStream_t s);
int corr_bwd_tiled(const float *gout, const float *in0, const float *in1, float *g0, float *g1,
                   const CorrGeom &g, cudaStream_t s);

}  // namespace unflow
