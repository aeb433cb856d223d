// tc_conv_plan.cuh -- the description of one unflow_tc_conv layer that make_plan (tc_conv.cu) builds: taps,
// output-parity classes, iteration extents, the wgmma kernel's tiles and epilogue.  The wgmma kernel (tc_conv.cu)
// and the FMA kernel for contractions over at most 4 channels (conv_fma.cu) both run from it.
#pragma once
#include "tc_common.cuh"

namespace unflow {
namespace tc {

constexpr int MAX_TAPS = 64;

struct Tap {
  short dx, dy;
  int widx;
  int widx2;                  // pair_px: the weight tap of the px = 1 class for this input offset (-1: none)
};

struct ConvParams {
  int N, Hit, Wit;            // images; iteration rows / columns of one class
  int TW, TH, TN;             // tile box, TW*TH*TN <= 128
  int tiles_x, tiles_y, tiles_n, n_blocks, n_classes;
  int s_in_x, s_in_y, s_out;    // input strides per axis (the row-window form folds the x stride into the tensor map)
  int Cin, Cout, kblocks;
  float *out;
  long long out_pitch;        // floats between consecutive output pixels
  int Hout, Wout;
  const float *bias;          // [Cout] or nullptr
  float slope;                // leaky-ReLU slope when act != 0
  int act, accumulate;
  int chunk;                  // K blocks per wgmma accumulation between two register adds (g_chunk)
  long long *dbg;             // role timers of CTA 0 (unflow_tc_conv_debug), or nullptr
  int pair_px;                // two output-parity classes (px = 0, 1) of a narrow transposed layer share one tile, see
                              // pair_px_plan()
  int ksplit;                 // > 1: the K loop of a tile is cut into ksplit work items whose partial sums meet in the
                              // (zeroed) output through red.global.add; bias / activation run as a separate pass
  int class_start[5];
  short class_px[4], class_py[4];
  Tap taps[MAX_TAPS];
  SkSchedule sk;              // the segments of each CTA (tc_schedule.h)
  float *sk_part;             // stream-K fixup: partial sums of split tiles, 2 slots per CTA (see sk_storage)
  unsigned *sk_count;         // stream-K fixup: arrivals per SK item and consumer warp, zero between launches
};

// conv_fma.cu: the layer of plan `p` (epilogue fields set, p.Cin <= 4) as one FMA-pipe launch.  x: NHWC
// [N, Hin, Win, Cin] with `x_pitch` floats per pixel; w_hi / w_lo: the weight planes [taps][Cout][4].
int conv_fma(const ConvParams &p, const float *x, int Hin, int Win, long long x_pitch, const float *w_hi,
             const float *w_lo, cudaStream_t stream);

}  // namespace tc
}  // namespace unflow
