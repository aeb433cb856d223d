/*
 * unflow.h -- C ABI of libunflow.so, the sm_90a kernels behind the UnFlow hot path.
 *
 * This is the drop-in boundary: the reference binds its ops through
 * TensorFlow's C++ OpKernel interface (tf.load_op_library, reference
 * src/e2eflow/ops.py:56-63); a maintainer replacing those four .so files binds
 * the entry points below instead (INTEGRATION.md shows the ctypes stub).  Each
 * entry point cites the reference interface it replaces (file:line under
 * /root/reference).
 *
 * Conventions (SURVEY.md section 8b):
 *   - every pointer is a DEVICE pointer to float32 data, densely packed, in the
 *     layout the reference op uses (NCHW for correlation, NHWC elsewhere);
 *   - the caller allocates and owns every buffer, including outputs;
 *   - `stream` is a cudaStream_t (CUstream) passed as void*; kernels are only
 *     enqueued on it; nothing here synchronises or allocates device memory;
 *   - return value: UNFLOW_OK, UNFLOW_EINVAL (argument check failed -- mirrors
 *     the reference's OP_REQUIRES -> InvalidArgument), UNFLOW_ECUDA (launch
 *     failed); unflow_last_error() returns a thread-local message;
 *   - re-entrant: safe to call from several host threads on distinct streams.
 *     Process-global state: the atomic launch counter, the thread-local error
 *     string, the once-resolved driver entry point used to encode TMA tensor
 *     maps, and the accumulation chunk set through
 *     unflow_set_int_option() (set it before launching, not while other
 *     threads launch).
 */
#ifndef UNFLOW_H_
#define UNFLOW_H_

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define UNFLOW_OK 0
#define UNFLOW_EINVAL 1
#define UNFLOW_ECUDA 2

#define UNFLOW_BORDER_ZERO 0  /* BackwardWarp op: taps outside the image contribute 0 */
#define UNFLOW_BORDER_CLAMP 1 /* image_warp: tap indices clamped to the image       */
#define UNFLOW_BORDER_STN 2   /* spatial_transformer sampler (augmentation): `flows` holds ABSOLUTE
                                 sample coordinates; forward only (the reference stops gradients) */

/* Library / diagnostics. */
int unflow_abi_version(void);
const char *unflow_last_error(void);
/* Number of kernels this library has launched since load (or since the last
 * reset); bench.py reports it as gpu_launches. */
unsigned long long unflow_launch_count(void);
void unflow_reset_launch_count(void);
/* Accuracy knob for tests / benchmarks; the only option is "tc_chunk" (1..64): K blocks per tensor-core
 * accumulation of the tc_* kernels, default 8 (the accumulator truncates, so the error grows with the chunk:
 * about 8x at 64).  Any other name or value: UNFLOW_EINVAL. */
int unflow_set_int_option(const char *name, int value);

/* ------------------------------------------------------------------------
 * Correlation   (reference: REGISTER_OP("Correlation") ops/correlation_op.cc:133-168,
 * CorrelationOp::Compute ops/correlation_op.cc:38-85, geometry ops/correlation_op.h:28-52,
 * kernels ops/correlation_op.cu.cc:31-117,250-315)
 *   in0,in1 : [B,C,H,W]    out : [B, D*D, out_h, out_w],  D = 2*(max_displacement/stride_2)+1
 * The reference's padded_0/padded_1 outputs are an implementation detail of
 * its kernels (consumed only by its own gradient) and are not produced.
 * EINVAL: even kernel_size (correlation_op.h:16-17), out_h<=0 or out_w<=0
 * (correlation_op.cc:60-61), non-positive strides/sizes.
 * ---------------------------------------------------------------------- */
int unflow_correlation_out_shape(int H, int W, int kernel_size, int max_displacement, int pad,
                                 int stride_1, int stride_2, int *out_c, int *out_h, int *out_w);
size_t unflow_correlation_workspace_bytes(int B, int C, int H, int W, int kernel_size,
                                          int max_displacement, int pad, int stride_1,
                                          int stride_2);
int unflow_correlation_fwd(const float *in0, const float *in1, float *out, int B, int C, int H,
                           int W, int kernel_size, int max_displacement, int pad, int stride_1,
                           int stride_2, void *stream);
/* CorrelationGrad (REGISTER_OP ops/correlation_op.cc:170-187, Compute :87-129, kernels
 * ops/correlation_op.cu.cc:120-248,317-390): gout [B,D*D,out_h,out_w] -> g0,g1 [B,C,H,W].
 * Reads the original inputs directly (no padded copies). */
int unflow_correlation_bwd(const float *gout, const float *in0, const float *in1, float *g0,
                           float *g1, int B, int C, int H, int W, int kernel_size,
                           int max_displacement, int pad, int stride_1, int stride_2,
                           void *stream);
/* Which implementation the dispatcher picks for these attributes:
 * 0 = generic kernel, 1 = tiled TMA kernel (the FlowNetC path). */
int unflow_correlation_fwd_path(int C, int H, int W, int kernel_size, int max_displacement,
                                int pad, int stride_1, int stride_2);
/* Both cost volumes of the bidirectional pass (reference call site src/e2eflow/core/flownet.py:34-44:
 * flownet_c(conv3_a, conv3_b, ..) and flownet_c(conv3_b, conv3_a, ..)) in ONE launch:
 *   out = Correlation(in0, in1),  out_rev = Correlation(in1, in0)
 * using corr(in1,in0)[(-p,-o)](y+s2*p, x+s2*o) == corr(in0,in1)[(p,o)](y,x): the second volume is a
 * second store of the first one's accumulators (zero where the displaced pixel leaves the image) and is
 * bit-identical to a second launch.  unflow_correlation_fold_grad adds the re-indexed gradient of the
 * reverse volume to the forward one's, so unflow_correlation_bwd(gout_eff, in0, in1) yields the
 * gradients of BOTH volumes.  Served for the attribute / shape set of the tiled kernel only
 * (unflow_correlation_fwd_path == 1), UNFLOW_EINVAL otherwise. */
int unflow_correlation_fwd_bidir(const float *in0, const float *in1, float *out, float *out_rev, int B,
                                 int C, int H, int W, int kernel_size, int max_displacement, int pad,
                                 int stride_1, int stride_2, void *stream);
int unflow_correlation_fold_grad(const float *gout, const float *gout_rev, float *gout_eff, int B, int C,
                                 int H, int W, int kernel_size, int max_displacement, int pad,
                                 int stride_1, int stride_2, void *stream);
/* Layout bridge around the correlation op.  The op keeps the reference's tensor layout -- inputs and cost
 * volume are [B, C, H, W] (ops/correlation_op.cc:15-27, ops/correlation_op.cu.cc:250-315) -- while the conv
 * stack keeps activations NHWC inside pitch-padded concat buffers (src/e2eflow/core/flownet.py:34-44 is the
 * call site: conv3 features in, concat([conv_redir, corr]) out).  These two tiled transposes replace the
 * strided library copies at that border:
 *   planar_to_interleaved: dst[b][p][c] (+)= src[b][c][p]     src dense [C][P] per image (P = H*W)
 *   interleaved_to_planar: dst[b][c][p]  =  src[b][p][c]      interleaved side: pixel pitch >= C floats
 * `*_batch` = floats between consecutive images on that side (lets the interleaved side be a channel and
 * batch slice of a larger buffer); accumulate != 0 adds into dst. */
int unflow_planar_to_interleaved(const float *src, long long src_batch, float *dst, long long dst_batch,
                                 long long pitch, int B, int C, int P, int accumulate, void *stream);
int unflow_interleaved_to_planar(const float *src, long long src_batch, long long pitch, float *dst,
                                 long long dst_batch, int B, int C, int P, void *stream);

/* ------------------------------------------------------------------------
 * BackwardWarp / image_warp
 *   reference op: REGISTER_OP("BackwardWarp") ops/backward_warp_op.cc:77-91, kernel
 *   ops/backward_warp_op.cu.cc:14-68 (border_mode = UNFLOW_BORDER_ZERO);
 *   reference training path: image_warp, src/e2eflow/core/image_warp.py:4-76
 *   (border_mode = UNFLOW_BORDER_CLAMP).
 *   images [B,H,W,C], flows [B,H,W,2] -> out [B,H,W,C]
 * ---------------------------------------------------------------------- */
int unflow_backward_warp_fwd(const float *images, const float *flows, float *out, int B, int H,
                             int W, int C, int border_mode, void *stream);
/* BackwardWarpGrad (ops/backward_warp_op.cu.cc:70-138) -> dflow [B,H,W,2].
 * dimage may be NULL (the op returns no image gradient, src/e2eflow/ops.py:80-84);
 * when non-NULL it must be zero-initialised by the caller and receives the
 * scatter-add gradient TF autodiff produces for image_warp (tf.gather -> scatter). */
int unflow_backward_warp_bwd(const float *grad, const float *images, const float *flows,
                             float *dflow, float *dimage, int B, int H, int W, int C,
                             int border_mode, void *stream);

/* ------------------------------------------------------------------------
 * ForwardWarp  (REGISTER_OP ops/forward_warp_op.cc:81-100; kernels
 * ops/forward_warp_op.cu.cc:16-125).  flows [B,H,W,2] -> out [B,H,W,1].
 * The launcher zeroes `out` itself (the reference runs SetZero first, :139-143).
 * ---------------------------------------------------------------------- */
int unflow_forward_warp_fwd(const float *flows, float *out, int B, int H, int W, void *stream);
int unflow_forward_warp_bwd(const float *grad, const float *flows, float *dflow, int B, int H,
                            int W, void *stream);

/* ------------------------------------------------------------------------
 * Downsample  (REGISTER_OP ops/downsample_op.cc:63-81, Compute :30-57, kernel
 * ops/downsample_op.cu.cc:15-72).  images [B,H,W,C] -> out [B,H/scale,W/scale,C].
 * EINVAL when H or W is not divisible by scale (downsample_op.cc:37-40).
 * ---------------------------------------------------------------------- */
int unflow_downsample(const float *images, float *out, int B, int H, int W, int C, int scale,
                      void *stream);

/* ------------------------------------------------------------------------
 * Fused per-level loss  (reference: compute_losses, src/e2eflow/core/losses.py:16-87, with
 * image_warp image_warp.py:4-76, ternary_loss :90-122, fb occlusion :38-56, second_order_loss
 * :258-295, smoothness_loss :206-255, charbonnier_loss :298-322, masks :325-366).
 * The reference has no native entry point here (it is a graph of TF ops); this is the fused
 * replacement the Python mirror (e2eflow.core.losses.compute_losses) calls.
 *   im1, im2            [B,h,w,3] in [0,1]
 *   flow_fw, flow_bw    [B,h,w,2] in pixels (already scaled)
 *   border_mask         [B,h,w,1] or NULL (NULL -> create_outgoing_mask of each flow)
 *   fwarp_fw, fwarp_bw  [B,h,w,1] outputs of unflow_forward_warp_fwd for the two flows; only
 *                       needed when mask_occlusion == 2 ('disocc') or the sym term is requested
 *   losses              [8] out: sym, occ, photo, grad, smooth_1st, smooth_2nd, fb, ternary
 *                       (UNFLOW_TERM_* order; terms not requested are written as 0)
 *   saved               [4*B*h*w] out, consumed by the backward pass (needed for ternary)
 *   masks_out           optional [2*B*h*w] out: mask_fw, mask_bw (binary; for parity tests)
 *   workspace           unflow_level_loss_workspace_bytes(B,h,w) bytes of scratch
 *   mask_occlusion      0 '' / 1 'fb' / 2 'disocc';  max_distance 1..3 (census patch 3/5/7)
 *   terms               bit k set = compute term k.  The 'grad' term (bit 3) is not fused: EINVAL.
 * Backward: grad_losses [8] (device) = dL/dloss_k -> dflow_fw, dflow_bw [B,h,w,2] (zeroed by the
 * launcher, accumulated with atomics).  Masks / occlusion maps carry no gradient (tf.cast).
 * ---------------------------------------------------------------------- */
#define UNFLOW_TERM_SYM 0
#define UNFLOW_TERM_OCC 1
#define UNFLOW_TERM_PHOTO 2
#define UNFLOW_TERM_GRAD 3
#define UNFLOW_TERM_SMOOTH_1ST 4
#define UNFLOW_TERM_SMOOTH_2ND 5
#define UNFLOW_TERM_FB 6
#define UNFLOW_TERM_TERNARY 7
size_t unflow_level_loss_workspace_bytes(int B, int h, int w);
int unflow_level_loss_fwd(const float *im1, const float *im2, const float *flow_fw,
                          const float *flow_bw, const float *border_mask, const float *fwarp_fw,
                          const float *fwarp_bw, float *losses, float *saved, float *masks_out,
                          void *workspace, int B, int h, int w, int mask_occlusion,
                          int max_distance, unsigned terms, void *stream);
int unflow_level_loss_bwd(const float *grad_losses, const float *im1, const float *im2,
                          const float *flow_fw, const float *flow_bw, const float *border_mask,
                          const float *fwarp_fw, const float *fwarp_bw, const float *saved,
                          float *dflow_fw, float *dflow_bw, int B, int h, int w,
                          int mask_occlusion, int max_distance, unsigned terms, void *stream);

/* ------------------------------------------------------------------------
 * Fused supervised flow loss of one network  (reference: supervised_loss,
 * src/e2eflow/core/supervised.py:45-57, with charbonnier_loss losses.py:298-323):
 *   loss = sum(mask * ((resize_bilinear(flow, [H,W]) * scale - flow_gt)^2 + 0.001^2)^0.45)
 *          / (B*H*W*2)
 * resize_bilinear is the legacy TF kernel (align_corners=False, no half-pixel centres):
 * per axis src = float32(i) * float32(h/H), lo = floor(src), hi = min(ceil(src), h-1).  Any
 * ratio h/H works (1 for full-resolution networks).  Masked elements add nothing but count in
 * the denominator, as in the reference.
 *   flow        [B,h,w,2] network output (network units)
 *   flow_gt     [B,H,W,2] ground truth in pixels
 *   mask_gt     [B,H,W,1] 0/1 validity, or NULL (every pixel valid)
 *   loss        [1] out (device)
 *   workspace   unflow_supervised_loss_workspace_bytes(B,H,W) bytes of scratch; one call at a
 *               time per workspace
 *   scale       FLOW_SCALE * 4 = 20 in the reference
 * The sum is reduced deterministically (per-CTA partials in double, fixed-order final sum).
 * Backward: grad_loss [1] (device) = dL/dloss -> dflow [B,h,w,2], fully written (no zeroing
 * needed, no atomics: bit-identical across runs).  flow_gt and mask_gt carry no gradient.
 * UNFLOW_EINVAL on a non-positive size, a tensor of 2^31 or more elements, or a NULL required
 * pointer (everything except mask_gt).
 * ---------------------------------------------------------------------- */
size_t unflow_supervised_loss_workspace_bytes(int B, int H, int W);
int unflow_supervised_loss_fwd(const float *flow, const float *flow_gt, const float *mask_gt,
                               float *loss, void *workspace, int B, int h, int w, int H, int W,
                               float scale, void *stream);
int unflow_supervised_loss_bwd(const float *grad_loss, const float *flow, const float *flow_gt,
                               const float *mask_gt, float *dflow, int B, int h, int w, int H,
                               int W, float scale, void *stream);

/* ------------------------------------------------------------------------
 * Fused Adam update on the flat parameter buffer (reference: tf.train.AdamOptimizer(beta1=0.9,
 * beta2=0.999), src/e2eflow/core/train.py:151-152; gradient averaging train.py:388-422 becomes
 * one NCCL all-reduce on `grads` before this call).  TF update rule:
 *   lr_t = lr*sqrt(1-beta2^step)/(1-beta1^step);  p -= lr_t * m / (sqrt(v) + eps).
 * grads are multiplied by grad_scale first (1/world_size when the all-reduce summed); when
 * zero_grad != 0 the gradient buffer is cleared in the same pass.  n must be a multiple of 4.
 * ---------------------------------------------------------------------- */
int unflow_adam_step(float *params, float *grads, float *m, float *v, long long n, float lr,
                     float beta1, float beta2, float eps, long long step, float grad_scale,
                     int zero_grad, void *stream);
/* Same update with the hyper-parameters read from DEVICE memory at run time:
 * hyper = [lr, beta1, beta2, eps, grad_scale, step]; lr_t is computed on the device from `step`
 * (1 for the first update), in double as unflow_adam_step forms it on the host.  A one-thread kernel
 * advances `step` after the update.  Lets a CUDA graph
 * of the whole training step be replayed without per-step host writes. */
int unflow_adam_step_dev(float *params, float *grads, float *m, float *v, long long n,
                         float *hyper, int zero_grad, void *stream);
/* The same two updates with the L2 regularisation gradient of slim.l2_regularizer (reference
 * src/e2eflow/core/flownet.py:176,200,218: `weights` variables only) folded in: bit k of l2mask[i] marks
 * element 4*i + k of the flat buffer as regularised; its gradient becomes grad * grad_scale + l2 * param.
 * (l2mask == NULL: identical to the functions above.) */
int unflow_adam_step_l2(float *params, float *grads, float *m, float *v, long long n, float lr,
                        float beta1, float beta2, float eps, long long step, float grad_scale,
                        int zero_grad, const unsigned char *l2mask, float l2, void *stream);
int unflow_adam_step_dev_l2(float *params, float *grads, float *m, float *v, long long n,
                            float *hyper, int zero_grad, const unsigned char *l2mask, float l2,
                            void *stream);

/* ------------------------------------------------------------------------
 * Bias and leaky ReLU of the conv / deconv layers outside the conv kernels (csrc/bias_act.cu;
 * reference activation flownet.py:84-86).  `act` is the leaky-ReLU OUTPUT of the layer whose
 * gradient `g` is, and lrelu'(act) = (act > 0 ? 1 : slope).
 * ---------------------------------------------------------------------- */
/* unflow_bias_lrelu: y = leaky_relu(y + bias[c]) in place on dense NHWC [pixels][C] (C % 4 == 0).
 * unflow_bias_grad_lrelu: gb[c] = sum_pixels g * lrelu'(act)  (act: dense NHWC [N,H,W,C]; NULL: plain
 * bias gradient); g is read through strides, gb is zeroed by the launcher. */
int unflow_bias_lrelu(float *y, const float *bias, long long pixels, int C, float slope, void *stream);
/* unflow_lrelu_bwd_bias: unflow_bias_grad_lrelu that also writes gpre = g * lrelu'(act) as dense
 * NHWC [N,H,W,C] (NULL: skip) -- the gradient w.r.t. the pre-activation output, the operand of the
 * tensor-core input / weight gradient kernels (one pass over g instead of two).  Here `act` may be a
 * channel slice of a concat buffer: `act_pitch` floats between pixels; gpre is written with
 * `gpre_pitch` floats between pixels (>= C; a multiple of 4 for the tensor-core kernels). */
int unflow_lrelu_bwd_bias(const float *g, long long sN, long long sC, long long sH, long long sW,
                          const float *act, long long act_pitch, float *gpre, long long gpre_pitch,
                          float *gb, int N, int C, int H, int W, float slope, void *stream);
int unflow_bias_grad_lrelu(const float *g, long long sN, long long sC, long long sH, long long sW,
                           const float *act, float *gb, int N, int C, int H, int W, float slope,
                           void *stream);

/* ---- flow-prediction heads: 3x3, stride 1, SAME, C_out = 2 (csrc/narrow_conv.cu) ---------------
 * The reference's `slim.conv2d(concatN, 2, 3, scope='flowN', activation_fn=None)` layers
 * (src/e2eflow/core/flownet.py:92-131) in exact fp32 on the FMA pipes; two output channels are
 * no tensor-core shape.
 *   x    NHWC [N,H,W,C] with `x_pitch` floats between pixels (>= C: a channel slice of a concat
 *        buffer is allowed), C even
 *   w    [2][3][3][C]  (OIHW weights stored channels-last = TF's HWIO with O moved to the front)
 *   bias [2] or NULL;  y NHWC [N,H,W,2] with `y_pitch` (even) floats between pixels, 8-byte aligned
 *   g    gradient w.r.t. y as a logical [N,2,H,W] tensor read through strides (floats)
 *   gw   [2][3][3][C], written (not accumulated); deterministic two-pass reduction through
 *        ``workspace`` (unflow_conv3x3_narrow_wgrad_workspace_bytes bytes).
 * UNFLOW_EINVAL unless C_out == 2 and C is even. */
int unflow_conv3x3_narrow_fwd(const float *x, long long x_pitch, const float *w, const float *bias, float *y,
                              long long y_pitch, int N, int H, int W, int C, int C_out, void *stream);
size_t unflow_conv3x3_narrow_wgrad_workspace_bytes(int N, int H, int W, int C);
int unflow_conv3x3_narrow_wgrad(const float *x, long long x_pitch, const float *g, long long gsN, long long gsC,
                                long long gsH, long long gsW, float *gw, void *workspace, int N, int H,
                                int W, int C, int C_out, void *stream);

/* ---- conv / deconv stacks on the tensor cores (csrc/tc_conv.cu) --------------------------------
 * The reference's slim.conv2d / slim.conv2d_transpose layers (src/e2eflow/core/flownet.py:166-233,
 * _flownet_upconv :89-155; cuDNN behind TensorFlow) as a hand-written wgmma implicit GEMM:
 * fp32 activations are read from HBM once (TMA), split into TF32 hi / lo planes in shared memory,
 * three tf32 wgmma per K step accumulate in registers (fp32-level accuracy, "3xTF32"),
 * the epilogue adds the bias, applies max(slope*x, x) (flownet.py:84-86) and writes -- or, with
 * `accumulate`, adds -- into the destination.
 *
 * unflow_tc_wsplit: weight planes hi = tf32(w), lo = w - hi in the layout [taps][R][Cp]
 *   (R = the GEMM's output channels, C = contraction channels, Cp = C rounded up to 4, tail zero);
 *   element (t, r, c) is read from w[t*s_t + r*s_r + c*s_c] (strides in floats).
 * unflow_tc_conv:
 *   x  NHWC [N,Hin,Win,Cin], `x_pitch` floats between pixels (a channel slice of a wider buffer is
 *      allowed); y NHWC [N,Hout,Wout,Cout] with `y_pitch`; pitches % 4 == 0; x, y and the weight
 *      planes 16-byte aligned (bias: any float address).
 *   mode 0  y[oy,ox] = sum_k x[stride*oy - pad_t + ky, stride*ox - pad_l + kx] W[ky*kw+kx]
 *           (slim.conv2d; TF SAME padding enters as the offsets pad_t / pad_l, zero outside)
 *   mode 1  y[stride*iy - pad_t + ky, stride*ix - pad_l + kx] += x[iy,ix] W[ky*kw+kx]
 *           (slim.conv2d_transpose and the input gradient of mode 0; Hout, Wout % stride == 0)
 *   stride 1 or 2, kh*kw <= 64.  UNFLOW_EINVAL otherwise.
 *   Epilogue: y = act(bias + conv), or with accumulate != 0  y += act(bias + conv) (the activation applies
 *   to this call's sum only, never to what y held before); bias may be null, act = 0 skips the activation.
 *   Cin <= 4 (the flow heads' input gradients, the flow up-sampling deconvs) runs in exact fp32 on the FMA pipes
 *   instead (csrc/conv_fma.cu): one launch, each output element written by one thread, channels >= Cout never;
 *   the weight planes are read as hi + lo. */
/* Debug hook: CTA 0 of every following tc_conv launch writes its role timers
 * (clocks blocked on each pipeline barrier / in total, see csrc/tc_conv.cu) into `buf`, device memory for 16
 * long longs; nullptr switches it off.  [0, 1]: producer wait / total, [2, 3]: consumer wait / total; tc_conv
 * launches add [5]: stages of the ring; tc_wgrad launches add [4]: consumer wait for a free split slot, [5, 6]:
 * raw and split ring slots (csrc/tc_wgrad.cu). */
int unflow_tc_conv_debug(long long *buf);
/* unflow_tc_conv_plan (host only, for the CPU tests): the tap / class / tile plan unflow_tc_conv launches,
 * as integers (layout in csrc/tc_conv.cu), including the two-parity-classes-per-tile rewrite it applies to
 * transposed layers of 33..64 output channels; returns the count written, -needed when `cap` is too
 * small, -1 on invalid arguments.  Only the low two bits of `mode` are read.  The last integer is the
 * number of K slices per tile the launcher uses when the epilogue allows slicing. */
int unflow_tc_conv_plan(int N, int Hin, int Win, int Cin, int Hout, int Wout, int Cout, int mode,
                        int stride, int kh, int kw, int pad_t, int pad_l, int *out, int cap);
int unflow_tc_wsplit(const float *w, float *w_hi, float *w_lo, int taps, int R, int C, long long s_t,
                     long long s_r, long long s_c, void *stream);
int unflow_tc_conv(const float *x, int N, int Hin, int Win, int Cin, long long x_pitch,
                   const float *w_hi, const float *w_lo, float *y, int Hout, int Wout, int Cout,
                   long long y_pitch, const float *bias, float slope, int act, int accumulate,
                   int mode, int stride, int kh, int kw, int pad_t, int pad_l, void *stream);

/* unflow_tc_wgrad (csrc/tc_wgrad.cu): weight gradient of the same layers, same arithmetic (both operands
 * split and transposed in shared memory straight from the NHWC activations, wgmma, fp32 register
 * accumulation, split-K):
 *     dw[r * pitch_r + t * pitch_t + c] += sum_p P[p][r] * G[stride * p + (k - pad)][c],   t = ky*kw + kx
 *   slim.conv2d:            P = dL/dy [N,Hp,Wp,R=C_out],  G = x     [N,Hg,Wg,C=C_in]
 *   slim.conv2d_transpose:  P = x     [N,Hp,Wp,R=C_in],   G = dL/dy [N,Hg,Wg,C=C_out], stride 2
 * P / G: NHWC with pixel pitches (multiples of 4 floats), 16-byte aligned.  dw is ACCUMULATED with
 * fp32 atomics (the caller zeroes it); the summation order is not fixed.  unflow_tc_wgrad_plan: the
 * launcher's K-block box / split-K plan as integers, host only (tests). */
int unflow_tc_wgrad_plan(int N, int Hp, int Wp, int R, int C, int stride, int kh, int kw, int pad_t,
                         int pad_l, int *out);
int unflow_tc_wgrad(const float *P, int N, int Hp, int Wp, int R, long long p_pitch, const float *G,
                    int Hg, int Wg, int C, long long g_pitch, float *dw, long long pitch_r,
                    long long pitch_t, int stride, int kh, int kw, int pad_t, int pad_l, void *stream);

/* First layers (7x7 stride 2 on 3 / 6 / 14 channels; flownet.py:174-176,203): the row-window form.
 * `xp` is the input as NHWC with Cp = 4 / 8 / 16 floats per pixel (channel tail zero) and rows of Wp
 * pixels that already contain the TF SAME padding in x (pad_l zero pixels on the left, zeros on the
 * right up to Wp >= stride*(Wout-1) + 8); rows outside [0,H) are zero fill.  The kw taps of a filter
 * row are one contiguous 8*Cp-float window, so the layer is a convolution with kh taps and an
 * 8*Cp-wide contraction: weight planes / dw are [Cout][kh][8*Cp] with column kx*Cp + c. */
int unflow_tc_conv_window(const float *xp, int N, int H, int Wp, int Cp, const float *w_hi, const float *w_lo,
                          float *y, int Hout, int Wout, int Cout, long long y_pitch, const float *bias,
                          float slope, int act, int kh, int stride, int pad_t, void *stream);
int unflow_tc_wgrad_window(const float *P, int N, int Ho, int Wo, int R, long long p_pitch, const float *xp,
                           int H, int Wp, int Cp, float *dw, int kh, int stride, int pad_t, void *stream);

/* ---- checkpoint formats (SURVEY.md section 8f, N2) --------------------------------------------
 * Host-only helper, no GPU work: CRC-32C (Castagnoli) of ``n`` bytes continuing from ``crc``
 * (0 to start).  TensorFlow's checkpoint files -- what tf.train.Saver writes and restores in the
 * reference (src/e2eflow/core/train.py:23-65,258-259) -- guard every index block and every tensor
 * with this checksum; the importer/exporter (e2eflow/core/tf_checkpoint.py) calls it for the
 * ~157 MB of weights per network. */
unsigned int unflow_crc32c(const void *data, size_t n, unsigned int crc);

#ifdef __cplusplus
}
#endif
#endif /* UNFLOW_H_ */
