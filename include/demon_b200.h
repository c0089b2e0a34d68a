/*
 * demon_b200 -- C ABI of the H100-native (sm_90a) DeMoN two-view inference path.
 *
 * This is the drop-in boundary: every entry point replaces one TensorFlow
 * custom-op kernel (or one `session.run` of a network graph) of the reference
 * lmb-freiburg/demon.  Plain pointers and sizes only; all tensor pointers are
 * DEVICE pointers on the current CUDA device unless the name ends in `_host`.
 * Every call is asynchronous on `stream` (a cudaStream_t passed as void*),
 * performs no allocation and no host synchronisation (the `_host` variants
 * excepted: they copy in, run, copy out and synchronise the stream), and is
 * CUDA-graph capturable.
 *
 * Return value: 0 on success, a negative DEMON_E_* code otherwise;
 * demon_last_error() returns a thread-local message for the last failure.
 *
 * Layout conventions follow the reference ops: NCHW with all leading
 * dimensions collapsed by the caller into `n` (warp2d.cc:150-160,
 * depthtoflow.cc:225-232, flowtodepth.cc:321-328).
 */
#ifndef DEMON_B200_H
#define DEMON_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DEMON_OK            0
#define DEMON_E_INVALID    -1   /* bad argument (shape, enum, null pointer)            */
#define DEMON_E_CUDA       -2   /* CUDA runtime / driver error (message has the code)  */
#define DEMON_E_STATE      -3   /* call order (e.g. forward before finalize)           */
#define DEMON_E_NOTFOUND   -4   /* unknown weight name                                 */

/* enum values shared with the Python layer */
#define DEMON_BORDER_CLAMP  1   /* warp2d.cc:259 enum BorderMode {CLAMP = 1, VALUE = 2} */
#define DEMON_BORDER_VALUE  2
#define DEMON_ROT_MATRIX     0  /* rotation_format.h:27 enum RotationFormat            */
#define DEMON_ROT_QUATERNION 1
#define DEMON_ROT_ANGLEAXIS3 2

const char* demon_last_error(void);
/* "demon_b200 <version> sm_90a" */
const char* demon_version(void);
/* number of kernels this library has launched in this process (bench.py's gpu_launches) */
int64_t demon_launch_count(void);

/* ------------------------------------------------------------------------
 * Geometry ops.  _f32 / _f64 mirror TypeConstraint<float|double>.
 * ---------------------------------------------------------------------- */

/* Replaces Warp2dOp / warp2d_gpu  (lmbspecialops/src/warp2d.cc:117-273, warp2d_cuda.cu:31-237).
 * input [n,c,h,w], displacements [n,2,h,w] -> output [n,c,h,w]. */
int demon_warp2d_f32(const float* input, const float* displacements, float* output,
                     int n, int c, int h, int w, int normalized, int border_mode,
                     float border_value, void* stream);
int demon_warp2d_f64(const double* input, const double* displacements, double* output,
                     int n, int c, int h, int w, int normalized, int border_mode,
                     double border_value, void* stream);

/* Replaces DepthToFlowOp (depthtoflow.cc:191-327, depthtoflow_cuda.cu:62-360).
 * depth [n,h,w], intrinsics [n,4], rotation [n,9|4|3], translation [n,3] -> flow [n,2,h,w]. */
int demon_depth_to_flow_f32(const float* depth, const float* intrinsics, const float* rotation,
                            const float* translation, float* flow, int n, int h, int w,
                            int rotation_format, int inverse_depth, int normalize_flow, void* stream);
int demon_depth_to_flow_f64(const double* depth, const double* intrinsics, const double* rotation,
                            const double* translation, double* flow, int n, int h, int w,
                            int rotation_format, int inverse_depth, int normalize_flow, void* stream);

/* Replaces FlowToDepthOp and FlowToDepth2Op (flowtodepth.cc:284-500, flowtodepth2.cc; CPU-only in
 * the reference).  flow [n,2,h,w] -> depth [n,1,h,w]. */
int demon_flow_to_depth_f32(const float* flow, const float* intrinsics, const float* rotation,
                            const float* translation, float* depth, int n, int h, int w,
                            int rotation_format, int inverse_depth, int normalized_flow, void* stream);
int demon_flow_to_depth_f64(const double* flow, const double* intrinsics, const double* rotation,
                            const double* translation, double* depth, int n, int h, int w,
                            int rotation_format, int inverse_depth, int normalized_flow, void* stream);

/* Replaces LeakyReluLmbOp (leakyrelu.cc:49-96, leakyrelu_cuda.cu:38-140). */
int demon_leaky_relu_f32(const float* input, float* output, int64_t size, float leak, void* stream);
int demon_leaky_relu_f64(const double* input, double* output, int64_t size, double leak, void* stream);

/* Replaces Median3x3DownsampleOp (median3x3downsample.cc:68-197, median3x3downsample_cuda.cu:28-180).
 * input [z,h,w] -> output [z,ceil(h/2),ceil(w/2)].  Bit exact with the CPU kernel. */
int demon_median3x3_downsample_f32(const float* input, float* output, int64_t z, int h, int w, void* stream);
int demon_median3x3_downsample_f64(const double* input, double* output, int64_t z, int h, int w, void* stream);

/* tf.image.resize_area(align_corners=False) by integer factors, the image2_2 of training/v2/training.py:179 (192x256 ->
 * 48x64).  input [n,c,h,w] float32 with `in_sn` floats between samples (>= c*h*w; a channel slice of a wider batch is read
 * in place) -> output [n,c,oh,ow] packed.  h % oh and w % ow must be 0 (DEMON_E_INVALID otherwise).  Every output is, in
 * float32: each of the fy = h/oh source rows' fx = w/ow pixels summed left to right from +0, the fy row sums summed top to
 * bottom from +0, times float32(1/(fy*fx)) -- this project's definition (DESIGN.md section 3.6). */
int demon_resize_area_f32(const float* input, int64_t in_sn, float* output, int n, int c, int h, int w, int oh, int ow, void* stream);

/* Replaces ScaleInvariantGradientOp forward (scaleinvariantgradient.cc:98-207,
 * scaleinvariantgradient_cuda.cu:56-102,205-320).  input [z,h,w] -> output [z,2,h,w].
 * deltas / weights are HOST arrays of length num (<= 16); they are op attributes in the reference. */
int demon_scale_invariant_gradient_f32(const float* input, float* output, int64_t z, int h, int w,
                                       const int* deltas, const float* weights, int num, float epsilon,
                                       void* stream);
int demon_scale_invariant_gradient_f64(const double* input, double* output, int64_t z, int h, int w,
                                       const int* deltas, const double* weights, int num, double epsilon,
                                       void* stream);

/* ------------------------------------------------------------------------
 * Training-side companions (SURVEY.md section 8 f4): the gradient kernels the reference registers for the ops above
 * and the element-wise ReplaceNonfinite of its v2 losses.  Same collapsing of leading dimensions as the forward ops.
 * ---------------------------------------------------------------------- */
/* Replaces ScaleInvariantGradientGradOp (scaleinvariantgradient.cc:294-404): gradients [z,2,h,w], input [z,h,w] -> [z,h,w] */
int demon_scale_invariant_gradient_grad_f32(const float* gradients, const float* input, float* output, int64_t z, int h, int w,
                                            const int* deltas, const float* weights, int num, float epsilon, void* stream);
int demon_scale_invariant_gradient_grad_f64(const double* gradients, const double* input, double* output, int64_t z, int h, int w,
                                            const int* deltas, const double* weights, int num, double epsilon, void* stream);
/* Replaces LeakyReluLmbGradOp (leakyrelu.cc:127-155) */
int demon_leaky_relu_grad_f32(const float* gradients, const float* input, float* output, int64_t size, float leak, void* stream);
int demon_leaky_relu_grad_f64(const double* gradients, const double* input, double* output, int64_t size, double leak, void* stream);
/* Replaces ReplaceNonfiniteOp / ReplaceNonfiniteGradOp (replacenonfinite.cc:49-80,115-150) */
int demon_replace_nonfinite_f32(const float* input, float* output, int64_t size, float value, void* stream);
int demon_replace_nonfinite_f64(const double* input, double* output, int64_t size, double value, void* stream);
int demon_replace_nonfinite_grad_f32(const float* gradients, const float* input, float* output, int64_t size, void* stream);
int demon_replace_nonfinite_grad_f64(const double* gradients, const double* input, double* output, int64_t size, void* stream);
/* Replaces DepthToNormalsOp (depthtonormals.cc:117-238): depth [z,h,w] (inverse depth if inverse_depth != 0), intrinsics [z,4]
 * normalised (fx, fy, cx, cy) -> normals [z,3,h,w] in the camera frame; NaN on the border and next to invalid depths */
int demon_depth_to_normals_f32(const float* depth, const float* intrinsics, float* output, int64_t z, int h, int w, int inverse_depth, void* stream);
int demon_depth_to_normals_f64(const double* depth, const double* intrinsics, double* output, int64_t z, int h, int w, int inverse_depth, void* stream);

/* ------------------------------------------------------------------------
 * FlowNet cost volumes: Correlation / Correlation1D and their gradients (correlation.cc, correlation_1d.cc,
 * correlation_cuda.cu, correlation_1d_cuda.cu), float32 NCHW, bit for bit the reference's CUDA kernels (NaNs included).
 * input1, input2 [n,c,h,w] -> output [n,top_c,top_h,top_w] with
 *   top_w = ceil((float)(w + 2 pad_size - 2 (max_displacement + k)) / stride1), k = (kernel_size - 1) / 2,
 *   top_h = the same over h for the 2D op, ceil((float)(h - 2 k) / stride1) for the 1D op (no vertical padding),
 *   top_c = (2 R + 1)^2 (2D), 2 R + 1 (1D, single_dir 0) or R + 1 (1D, single_dir +-1), R = max_displacement / stride2.
 * The 1D op's single_dir -1 uses the reference's displacements -(R+1) stride2 .. -stride2; a read outside the padded input
 * is 0.  do_abs is accepted and has no effect, as in the reference.  Gradients: gradient [n,top_c,top_h,top_w] ->
 * input1_grad, input2_grad [n,c,h,w], deterministic (no atomics).  DEMON_E_INVALID before any launch for an even or
 * non-positive kernel_size, stride1 or stride2 < 1, a negative max_displacement or pad_size, single_dir not in {-1,0,1}
 * or a top size < 1.  No workspace, no allocation; everything runs on `stream`.
 * ---------------------------------------------------------------------- */
#define DEMON_CORR_MULT 1   /* correlation_cuda.cu: enum CorrType {MULT = 1, SUBT = 2} */
#define DEMON_CORR_SUBT 2
int demon_correlation_f32(const float* input1, const float* input2, float* output, int n, int c, int h, int w, int corr_type,
                          int kernel_size, int max_displacement, int stride1, int stride2, int pad_size, int do_abs, void* stream);
int demon_correlation_grad_f32(const float* input1, const float* input2, const float* gradient, float* input1_grad, float* input2_grad,
                               int n, int c, int h, int w, int corr_type, int kernel_size, int max_displacement, int stride1,
                               int stride2, int pad_size, int do_abs, void* stream);
int demon_correlation_1d_f32(const float* input1, const float* input2, float* output, int n, int c, int h, int w, int corr_type,
                             int kernel_size, int max_displacement, int stride1, int stride2, int pad_size, int do_abs, int single_dir,
                             void* stream);
int demon_correlation_1d_grad_f32(const float* input1, const float* input2, const float* gradient, float* input1_grad,
                                  float* input2_grad, int n, int c, int h, int w, int corr_type, int kernel_size, int max_displacement,
                                  int stride1, int stride2, int pad_size, int do_abs, int single_dir, void* stream);

/* ------------------------------------------------------------------------
 * FlowNet warping: FlowWarp / FlowWarpGrad (flowwarp.cc, flowwarp_cuda.cu) and FlowOutOfFrame (flow_out_of_frame.cc),
 * float32 NCHW.  image [n,c,h,w], flow [n,2,h,w] (x then y displacement in pixels).
 *   flow_warp       warped [n,c,h,w]: bilinear at (x + fx, y + fy), bit for bit the reference's GPU kernel; out of frame
 *                   (a NaN flow included) the fill: 0 (DEMON_FLOW_WARP_ZERO) or the NaN with bits 0xFFE00000
 *                   (DEMON_FLOW_WARP_NAN).
 *   flow_warp_grad  gradient [n,c,h,w] -> image_grad [n,c,h,w], flow_grad [n,2,h,w].  flow_grad is bit for bit the
 *                   reference's GPU kernel (its formula, which at the clamped last row and column is not the derivative
 *                   of the forward op).  image_grad is bit for bit the reference's CPU kernel, whose GPU kernel adds
 *                   the same products with atomics in scheduling order.  workspace: device memory of at least
 *                   demon_flow_warp_grad_workspace_bytes(n, h, w) bytes, 256-byte aligned; that query returns -1 (and
 *                   sets the error) for n*h*w >= 2^31 - 1 or when the device cannot be queried.
 *   flow_out_of_frame  occ [n*h*w] -> output [n,1,h,w], bit for bit the reference's CPU kernel: occ where the rounded
 *                   target (x + fx, y + fy) lies in the image, else 1; a NaN occ passes through; a NaN, infinite or
 *                   out-of-int-range target is out of frame.
 * Deterministic: no float atomics, the same bits on every call.  DEMON_E_INVALID before any launch for a negative size,
 * an unknown fill or too small a workspace.  No allocation; everything runs on `stream`.
 * ---------------------------------------------------------------------- */
#define DEMON_FLOW_WARP_ZERO 1   /* flowwarp_cuda.cu: #define ZERO 1, NOT_A_NUMBER 2 */
#define DEMON_FLOW_WARP_NAN 2
int demon_flow_warp_f32(const float* image, const float* flow, float* warped, int n, int c, int h, int w, int fill, void* stream);
int64_t demon_flow_warp_grad_workspace_bytes(int n, int h, int w);
int demon_flow_warp_grad_f32(const float* image, const float* flow, const float* gradient, float* image_grad, float* flow_grad, int n, int c,
                             int h, int w, void* workspace, int64_t workspace_bytes, void* stream);
int demon_flow_out_of_frame_f32(const float* flow, const float* occ, float* output, int n, int h, int w, void* stream);

/* ------------------------------------------------------------------------
 * Resample (resample.cc, resample_cuda.cu): input [n,c,in_h,in_w] -> output [n,c,out_h,out_w], float32 and float64, bit
 * for bit the reference's NearestNeighborKernel / InterpolationKernel: scale fx = in_w / out_w, fy = in_h / out_h in
 * float, source position (x fx + fy/2 - 0.5, y fy + fx/2 - 0.5) (the reference's swapped half offsets), LINEAR (triangle)
 * or CUBIC (Keys, a = -0.5) weights, antialiased on both axes when `antialias` and either axis downsamples.  One
 * deviation: NEAREST clamps its source pixel to the image, where the reference reads outside it (fy / 2 >~ fx).
 * DEMON_E_INVALID for an unknown type or an output side < 1.  Deterministic, no allocation, runs on `stream`.
 * ---------------------------------------------------------------------- */
/* resample_cuda.cu: enum InterpolationType {NEAREST = 1, CUBIC = 2, LINEAR = 3}; DEMON_RESAMPLE_* are the image resize's */
#define DEMON_LMB_RESAMPLE_NEAREST 1
#define DEMON_LMB_RESAMPLE_CUBIC 2
#define DEMON_LMB_RESAMPLE_LINEAR 3
int demon_resample_f32(const float* input, float* output, int n, int c, int in_h, int in_w, int out_h, int out_w, int antialias, int type,
                       void* stream);
int demon_resample_f64(const double* input, double* output, int n, int c, int in_h, int in_w, int out_h, int out_w, int antialias, int type,
                       void* stream);

/* ------------------------------------------------------------------------
 * DeMoN v2's training losses (python/depthmotionnet/v2/losses.py) and their gradients (csrc/losses.cu).
 * All tensor pointers are device pointers of the entry's T (float for _f32, double for _f64), NCHW and contiguous.
 * Nothing allocates or synchronises; scratch comes from the caller.
 * ---------------------------------------------------------------------- */
#define DEMON_LOSS_L2   0   /* pointwise_l2_loss: mean of sqrt(sum_c d_c^2 + eps), d = replace_nonfinite(pr - gt)       */
#define DEMON_LOSS_SIG  1   /* pointwise_l2_loss of the prediction's 5-delta SIG stack (never stored) against gt's     */
#define DEMON_LOSS_L1   2   /* l1_loss: sum of sqrt(x^2 + eps), x = pr - gt (pr alone when gt is NULL)                */
#define DEMON_LOSS_MAX_TERMS 8
typedef struct demon_loss_term {
  int kind;                 /* DEMON_LOSS_*                                                                            */
  int c;                    /* L2: channels summed per pixel; L1: elements per row; SIG: 1                             */
  int h, w;                 /* L2, SIG: plane size                                                                     */
  int gt_plane;             /* SIG: gt is a plane [n,h,w] whose SIG stack is taken on the fly (eps gt_sig_eps);
                               otherwise gt is the stack [n,10,h,w], channels (2i, 2i+1) = (x, y) of delta 2^i          */
  int accumulate;           /* backward: 0 writes grad, 1 adds to it                                                   */
  int64_t n;                /* L2: samples [n,c,h,w]; SIG: planes [n,h,w] (a flow [N,2,h,w] is 2N planes); L1: rows   */
  const void* pr;
  const void* gt;
  double eps;               /* the loss epsilon, converted to T                                                        */
  double sig_eps;           /* SIG: epsilon of the prediction's SIG (converted to T)                                   */
  double gt_sig_eps;        /* SIG with gt_plane: epsilon of the ground truth's SIG                                    */
  double weight;            /* the weight, converted to T, unless weight_dev                                           */
  const void* weight_dev;   /* device T scalar or NULL                                                                  */
  void* out;                /* device T scalar: T(mean) * weight (L1: T(sum) * weight), or NULL                         */
  void* out0;               /* device T scalar: the mean (sum) with eps 0, not weighted, or NULL                        */
  void* terms;              /* L2: the per-pixel terms [n,h,w] (eps), or NULL                                          */
  const void* grad_out;     /* backward: device T scalar, the upstream gradient of `out` (NULL: 0)                     */
  void* grad;               /* backward: d(out)/d(pr), pr's shape; NULL: no gradient for this term                    */
} demon_loss_term;
/* Scratch bytes of the forward entries (backward = 0) or the backward entries (backward = 1) for this table; -1 if invalid. */
int64_t demon_loss_workspace_bytes(const demon_loss_term* terms, int num, int elem_size, int backward);
/* Every term's `out` and `out0` in two launches.  Sums are double in an order fixed by the shapes: same bits every call. */
int demon_loss_forward_f32(const demon_loss_term* terms, int num, void* workspace, int64_t workspace_bytes, void* stream);
int demon_loss_forward_f64(const demon_loss_term* terms, int num, void* workspace, int64_t workspace_bytes, void* stream);
/* Each term's gradient into its `grad`, terms in table order (one launch per L2 / L1 term, two per SIG term).  L2:
 * g*w*d_c/(M*t), 0 where d_c is not finite; L1: g*w*x/sqrt(x^2+eps); SIG: the same per SIG channel, through each delta's
 * SIG derivative (ScaleInvariantGradientGrad's, summed over the deltas). */
int demon_loss_backward_f32(const demon_loss_term* terms, int num, void* workspace, int64_t workspace_bytes, void* stream);
int demon_loss_backward_f64(const demon_loss_term* terms, int num, void* workspace, int64_t workspace_bytes, void* stream);
/* compute_confidence_map: out = T(exp((double)(T(-scale) * |pr - gt|))), exp in double and rounded once */
int demon_confidence_map_f32(const float* pr, const float* gt, float* out, int64_t size, double scale, void* stream);
int demon_confidence_map_f64(const double* pr, const double* gt, double* out, int64_t size, double scale, void* stream);
/* prepare_ground_truth_tensors for depth [n,h,w] (inverse depth), intrinsics [n,4], rotation [n,3] (angle axis),
 * translation [n,3]: depth2 [n,h2,w2], flow0/2/5 [n,2,.,.], normal0/2 [n,3,.,.], depth0_sig / depth2_sig [n,10,.,.],
 * flow2_sig [2n,10,h2,w2] (level k has the size (s+1)/2 applied k times).  Six launches (five medians, one for the rest);
 * each output bit for bit the composition of the standalone ops.  Scratch: demon_loss_ground_truth_workspace_bytes. */
int64_t demon_loss_ground_truth_workspace_bytes(int n, int h, int w, int elem_size);
int demon_loss_ground_truth_f32(const float* depth, const float* intrinsics, const float* rotation, const float* translation, int n, int h, int w,
                                float* depth2, float* flow0, float* flow2, float* flow5, float* normal0, float* normal2, float* depth0_sig,
                                float* depth2_sig, float* flow2_sig, void* workspace, int64_t workspace_bytes, void* stream);
int demon_loss_ground_truth_f64(const double* depth, const double* intrinsics, const double* rotation, const double* translation, int n, int h,
                                int w, double* depth2, double* flow0, double* flow2, double* flow5, double* normal0, double* normal2,
                                double* depth0_sig, double* depth2_sig, double* flow2_sig, void* workspace, int64_t workspace_bytes,
                                void* stream);

/* ------------------------------------------------------------------------
 * Evaluation metrics on the device (python/depthmotionnet/evaluation/metrics.py; SURVEY.md section 8 f3).
 * One streaming pass per call; all pointers are device pointers, nothing synchronises.
 * ---------------------------------------------------------------------- */
#define DEMON_METRIC_SUMS 16
/* bytes of scratch the two *_sums entries need for n samples of hw pixels */
int64_t demon_metric_workspace_bytes(int n, int64_t hw);
/* The masked per-sample sums behind compute_errors / evaluate_depth (metrics.py:240-372) for pred, gt [n, hw]:
 *   mask        finite and > 0 in BOTH inputs (compute_valid_depth_mask, metrics.py:25-38), again after the transforms
 *   transforms  reciprocal if inverse_pred / inverse_gt (metrics.py:339-342), gt / gt_div[n] if gt_div (the translation
 *               norm, metrics.py:349-355), pred * pred_scale[n] if pred_scale (metrics.py:362)
 *   sums[n][16] 0 num_valid, 1 sum|p-g|, 2 sum|1/p-1/g|, 3 sum ld, 4 sum ld^2 (ld = log p - log g), 5 sum|p-g|/g,
 *               6 sum (p-g)^2/g, 7 sum|log10 p - log10 g|, 8 sum (p-g)^2, 9..11 count(|ld| < log t) for t = 1.25,
 *               1.5625, 1.953125, 12 sum p*p and 13 sum p*g over finite positive p*g, 14 / 15 the same for 1/p, 1/g
 *               (12..15 on the UNSCALED prediction: compute_depth_scale_factor, metrics.py:283-318)                    */
int demon_depth_error_sums_f32(const float* pred, const float* gt, int n, int64_t hw, int inverse_pred, int inverse_gt,
                               const float* gt_div, const float* pred_scale, double* sums, void* workspace, void* stream);
/* scale[n] that minimises the squared error of scale * pred against gt, from the sums above, on the device
 * (mode 0 'abs', 1 'log', 2 'inv'; metrics.py:283-318) */
int demon_depth_scale_factor(const double* sums, int n, int mode, float* scale, void* stream);
/* compute_flow_epe (metrics.py:377-387): flow1, flow2 [n,2,hw] -> sums[n][2] = {sum of the valid end point errors, count} */
int demon_flow_epe_sums_f32(const float* flow1, const float* flow2, int n, int64_t hw, double* sums, void* workspace, void* stream);

/* The two sums above with the prediction at its own size, resized to the ground truth's by nearest neighbour and cropped,
 * without materialising either (evaluate_to_xarray.py:200-211).  pred [n,ph,pw] (flow [n,2,ph,pw]), gt [n,gh,gw] (flow
 * [n,2,gh,gw]); the output window is gt rows y0..y0+oh-1, columns x0..x0+ow-1; window row r reads prediction row
 * row_idx[r], column c reads column col_idx[c] (int32 device tables, see evaluation.nearest_index); an index of -1 reads
 * 0 (skimage's cval).  gt_valid [n,gh,gw] uint8 or NULL: 0 marks a gt pixel as invalid, as a NaN there would
 * (invalidate_points_not_visible_in_second_image).  Pixel order and CTA slots are those of the entries above over oh*ow
 * pixels, so the sums equal theirs on the materialised arrays bit for bit.  Workspace: demon_metric_workspace_bytes(n, oh*ow). */
int demon_depth_error_sums_resampled_f32(const float* pred, int ph, int pw, const float* gt, const uint8_t* gt_valid, int gh, int gw,
                                         int n, int y0, int x0, int oh, int ow, const int* row_idx, const int* col_idx,
                                         int inverse_pred, int inverse_gt, const float* gt_div, const float* pred_scale,
                                         double* sums, void* workspace, void* stream);
int demon_flow_epe_sums_resampled_f32(const float* pred, int ph, int pw, const float* gt, int gh, int gw, int n, int y0, int x0,
                                      int oh, int ow, const int* row_idx, const int* col_idx, double* sums, void* workspace,
                                      void* stream);

/* compute_motion_errors (metrics.py:390-445, normalize_translations) for n samples, one thread each, in double:
 * pred_rotation / pred_translation [n,3], gt_motion [n,6] (angle axis | translation), float32 ->
 * out[n][4] = rot_err (degrees), tran_err, tran_angle_err (degrees), camera_baseline = |t_gt| (NaN if gt_motion has a NaN)
 * and gt_div[n] (float32; may be NULL): the translation norm evaluate_depth divides the gt depth by, 1 where it is
 * numpy.isclose to 1, with t_gt = (1, 0, 0) for a motion with a NaN (evaluate_to_xarray.py:290-294). */
int demon_motion_errors(const float* pred_rotation, const float* pred_translation, const float* gt_motion, int n, double* out,
                        float* gt_div, void* stream);

/* compute_visible_points_mask (dataset_tools/view_tools_cython.pyx:9-58) for n views, bit for bit: depth [n,h,w] camera z,
 * per sample K1 [3,3], R1 [3,3], t1 [3], P2 [3,4] (float32) -> mask [n,h,w] = 1 where the pixel's point projects into the
 * second image strictly inside the border (borderx, bordery) of a width2 x height2 image and in front of the camera. */
int demon_visible_points_mask_f32(const float* depth, const float* K1, const float* R1, const float* t1, const float* P2, int n, int h,
                                  int w, int width2, int height2, int borderx, int bordery, uint8_t* mask, void* stream);
/* the same on INVERSE depth: the kernel takes 1/depth in float32 first (evaluate_to_xarray.py:110) */
int demon_visible_points_mask_inverse_f32(const float* inverse_depth, const float* K1, const float* R1, const float* t1, const float* P2,
                                          int n, int h, int w, int width2, int height2, int borderx, int bordery, uint8_t* mask,
                                          void* stream);

/* ------------------------------------------------------------------------
 * Point clouds of depth maps (python/depthmotionnet/vis.py:223-401 over vis_cython.pyx:24-173).
 * ---------------------------------------------------------------------- */
/* bytes of device scratch the two point-cloud entries need for n views of h x w (0 for an empty batch) */
int64_t demon_point_cloud_scratch_bytes(int n, int h, int w);
/* compute_point_cloud_from_depthmap (vis_cython.pyx:24-173) for n views, bit for bit: depth [n,h,w] camera z; per view K [3,3],
 * R [3,3], t [3] (float32 device arrays, so a captured graph replays with new cameras).  The valid pixels (finite and > 0) in
 * row-major order give rows 0..counts[i]-1 of view i:
 *   points [n,h*w,3]   R^T ((d*((x+0.5)-cx)/fx, d*((y+0.5)-cy)/fy, d) - t), with the .pyx's float32 operations and reciprocals
 *   normals_out        R^T normal of normals [n,3,h,w] (both NULL to skip)
 *   colors_out [n,h*w,3] uint8: colors [n,3,h,w] uint8 as is, or image [n,3,h,w] float32 as ((image+0.5)*255).astype(uint8)
 *                      of vis.py:276 (numpy's x86 cast: the low byte of the truncation, 0 for NaN and out-of-range values);
 *                      at most one of colors and image, colors_out NULL with neither
 *   counts [n] int32
 * Rows at and past counts[i] are not written.  Scratch: demon_point_cloud_scratch_bytes(n, h, w) bytes.  Sides 1..8192,
 * n up to 65535.  Output rows do not depend on scheduling; nothing synchronises, so the call can be captured in a graph. */
int demon_point_cloud_f32(const float* depth, const float* K, const float* R, const float* t, const float* normals,
                          const uint8_t* colors, const float* image, int n, int h, int w, void* scratch, float* points,
                          float* normals_out, uint8_t* colors_out, int* counts, void* stream);
/* the same on INVERSE depth: the kernels take d = 1/inverse_depth in float32 first (visualize_prediction, vis.py:246) */
int demon_point_cloud_inverse_f32(const float* inverse_depth, const float* K, const float* R, const float* t, const float* normals,
                                  const uint8_t* colors, const float* image, int n, int h, int w, void* scratch, float* points,
                                  float* normals_out, uint8_t* colors_out, int* counts, void* stream);

/* ------------------------------------------------------------------------
 * Fusion of depth maps into one surface (demon_b200/sequence.py): a TSDF volume and marching cubes.
 * The volume is caller-owned, nx x ny x nz voxels with x fastest: tsdf [nz,ny,nx] and weight [nz,ny,nx] float32, color
 * [nz,ny,nx,3] float32 or NULL.  Voxel (i,j,k) is the point origin + voxel_size*(i,j,k); origin is a HOST float[3].  At least
 * 2 voxels per axis and fewer than 2^31 in all.  Every float operation is round-to-nearest in the order given here.
 * ---------------------------------------------------------------------- */
/* Adds n frames to the volume, in frame order: depth [n,h,w] camera z, K [n,3,3], R [n,3,3], t [n,3] world-to-camera (float32
 * device arrays), image [n,h,w,3] uint8 (HWC RGB) with color, or NULL without.  For every voxel and frame: X_c = R X + t,
 * u = fx x/z + cx, v = fy y/z + cy, pixel (floor(u), floor(v)); the frame is skipped when z <= 0, the pixel is outside the
 * image, d is not finite or not > 0, or sdf = d - z < -trunc; otherwise f = min(1, sdf/trunc), tsdf = (tsdf W + f)/(W + 1),
 * color likewise with the pixel's bytes, W = W + 1.  voxel_size and trunc finite and > 0; h*w < 2^24. */
int demon_tsdf_integrate_f32(float* tsdf, float* weight, float* color, int nx, int ny, int nz, const float* origin, float voxel_size,
                             float trunc, const float* depth, const float* K, const float* R, const float* t, const uint8_t* image,
                             int n, int h, int w, void* stream);
/* bytes of device scratch the marching-cubes entries need (0 for an invalid volume) */
int64_t demon_marching_cubes_scratch_bytes(int nx, int ny, int nz);
/* Marching cubes, step 1: the number of triangles into *triangles (device int64), and in scratch where each tile of cubes
 * starts.  A cube is skipped when any of its 8 corners has weight 0; corner q of the cube is inside when its tsdf < 0. */
int demon_marching_cubes_count_f32(const float* tsdf, const float* weight, int nx, int ny, int nz, void* scratch, int64_t* triangles,
                                   void* stream);
/* Step 2, on the scratch step 1 filled and the same volume: the triangle soup, in the order of the cube's linear index and
 * then the standard Lorensen-Cline table's triangle order.  For T triangles: vertices [3T,3] float32, colors [3T,3] uint8
 * (with color; NULL without), faces [T,3] int32 = 0, 1, 2, ...  A vertex on the edge from corner p0 (the lower grid
 * coordinate) to p1 is p0 + (f0/(f0 - f1))(p1 - p0), its colour c0 + (f0/(f0 - f1))(c1 - c0) rounded half to even. */
int demon_marching_cubes_f32(const float* tsdf, const float* weight, const float* color, int nx, int ny, int nz, const float* origin,
                             float voxel_size, const void* scratch, float* vertices, uint8_t* colors, int* faces, void* stream);

/* ------------------------------------------------------------------------
 * A sparse TSDF volume (demon_b200/sequence.py: SparseTsdfVolume): voxel blocks of 8x8x8 stored where depth was seen.
 * Block b = (bx, by, bz), |b| <= DEMON_SPARSE_TSDF_MAX_COORD per axis, holds voxels g = 8b + (0..7) at origin +
 * voxel_size*g, with the dense volume's arithmetic.  The caller owns the state: blocks [m,3] int32 in pool order, tsdf and
 * weight [m,8,8,8] float32 (z, y, x; x fastest), color [m,8,8,8,3] float32 or NULL; and a hash table of `capacity` slots
 * (a power of 2) from a block's key to its pool index: keys int64 [capacity] (-1 empty), values int32 [capacity] (-1 for a
 * block inserted and not yet committed), and counters int64 [4] (0: occupied slots, 1: set when the allocation found the
 * table half full, 2: the pixels the allocation skipped, 3: scratch).  The table never holds more than capacity/2 keys.
 * A call that adds frames runs allocate, reads the counters (doubling the table with rehash and allocating again when it
 * was half full), gather_new, sorts the new keys ascending, commit, and integrate.
 * ---------------------------------------------------------------------- */
#define DEMON_SPARSE_TSDF_MAX_COORD ((1 << 20) - 1)
/* a pixel whose widened cell spans more blocks than this along an axis allocates nothing */
#define DEMON_SPARSE_TSDF_MAX_SPAN 4
/* Fills keys and values with -1 and zeroes counters, then moves every entry of the old table (old_capacity <= capacity/2
 * slots; 0 and NULL for none) into it and counts them in counters[0]. */
int demon_sparse_tsdf_rehash(const int64_t* old_keys, const int* old_values, int64_t old_capacity, int64_t* keys, int* values,
                             int64_t capacity, int64_t* counters, void* stream);
/* Inserts the blocks of n frames (depth [n,h,w], K, R, t as demon_tsdf_integrate_f32 takes them) into the table.  One
 * thread per pixel with finite d > 0 takes its band cell: the pixel square [px,px+1] x [py,py+1] between camera z d - trunc
 * and d + trunc, the near face replaced by the camera centre when d - trunc <= 0.  In this float order: zf = d + trunc,
 * zn = d - trunc; for each corner (u, v), a = (u - cx)/fx and b = (v - cy)/fy, camera points (a zf, b zf, zf) and, when
 * zn > 0, (a zn, b zn, zn); (0, 0, 0) when zn <= 0; world X_i = (R_0i (x - t_0) + R_1i (y - t_1)) + R_2i (z - t_2).  Over
 * the AABB [lo, hi] of those points, blocks floor(((lo - o)/vs - 2) * 0.125) .. floor(((hi - o)/vs + 2) * 0.125) per axis
 * are inserted.  A pixel with a non-finite point, a block past +-DEMON_SPARSE_TSDF_MAX_COORD or a range wider than
 * DEMON_SPARSE_TSDF_MAX_SPAN blocks inserts nothing and is counted in counters[2].  Every block an update with
 * f < 1 of a counted-in pixel reaches, and every voxel within one voxel of it, then lies in an inserted block.  New keys
 * get value -1; when an insertion would fill more than half the table it stops and sets counters[1].  Idempotent. */
int demon_sparse_tsdf_allocate_f32(int64_t* keys, const int* values, int64_t capacity, int64_t* counters, const float* origin,
                                   float voxel_size, float trunc, const float* depth, const float* K, const float* R, const float* t,
                                   int n, int h, int w, void* stream);
/* Writes the keys with value -1 to new_keys [counters[0] - m], in no particular order. */
int demon_sparse_tsdf_gather_new(const int64_t* keys, const int* values, int64_t capacity, int64_t* counters, int64_t* new_keys,
                                 void* stream);
/* Gives sorted_keys[i] the pool index first + i and writes its block coordinates to blocks[first + i]. */
int demon_sparse_tsdf_commit(const int64_t* keys, int* values, int64_t capacity, const int64_t* sorted_keys, int count, int first,
                             int* blocks, void* stream);
/* demon_tsdf_integrate_f32 on every voxel of the m blocks: one thread per voxel, the same per-frame update and order. */
int demon_sparse_tsdf_integrate_f32(float* tsdf, float* weight, float* color, const int* blocks, int m, const float* origin, float voxel_size,
                                    float trunc, const float* depth, const float* K, const float* R, const float* t, const uint8_t* image,
                                    int n, int h, int w, void* stream);
/* bytes of device scratch the sparse marching-cubes entries need for m >= 1 blocks */
int64_t demon_sparse_tsdf_mesh_scratch_bytes(int m);
/* Marching cubes on the blocks, step 1: resolves each block's 7 positive neighbours through the table and counts the
 * triangles into *triangles (device int64).  Cube l of block b has its corner 0 at voxel 8b + l; it is skipped when a corner
 * lies in a block that is not stored or has weight 0. */
int demon_sparse_tsdf_mesh_count_f32(const float* tsdf, const float* weight, const int* blocks, int m, const int64_t* keys, const int* values,
                                     int64_t capacity, void* scratch, int64_t* triangles, void* stream);
/* Step 2, on the scratch step 1 filled: demon_marching_cubes_f32's triangle soup, in the order of the block's pool index,
 * the cube's local linear index (x fastest) and the table's triangle order. */
int demon_sparse_tsdf_mesh_f32(const float* tsdf, const float* weight, const float* color, const int* blocks, int m, const float* origin,
                               float voxel_size, const void* scratch, float* vertices, uint8_t* colors, int* faces, void* stream);

/* ------------------------------------------------------------------------
 * Ray casting a TSDF volume (demon_b200/sequence.py: TsdfVolume.raycast, SparseTsdfVolume.raycast): depth, normals and
 * colour of the surface seen from n cameras, one thread per pixel.  K [n,3,3], R [n,3,3], t [n,3] world-to-camera as
 * demon_tsdf_integrate_f32 takes them, near and far [n] float32 device arrays; outputs depth [n,h,w] float32, normals
 * [n,3,h,w] float32 (NULL: not computed), colors [n,h,w,3] uint8 (colour volumes only; NULL: not computed).  The rule for
 * pixel (x, y) of frame f, every step one round-to-nearest float32 operation in the order written:
 *   1. a = ((x + 0.5) - cx)/fx, b = ((y + 0.5) - cy)/fy; world direction D_i = (R_0i a + R_1i b) + R_2i; camera centre
 *      C_i = -((R_0i t_0 + R_1i t_1) + R_2i t_2).
 *   2. delta = (step voxel_size)/sqrt((a a + b b) + 1), so samples are `step` voxels apart in space; sample k = 0, 1, ...
 *      at camera z z_k = near + (float)k delta, X = C + z_k D.  Samples with z_k <= 0 are invalid; the march evaluates the
 *      samples with z_k <= far, at most 2^24 of them.  A frame whose near is not >= 0 renders no hit.
 *   3. g = (X - origin)/voxel_size, cube c = floor(g), w = g - c.  The sample is valid when all 8 corners of cube c are
 *      stored (inside the box; in allocated blocks for a sparse volume) with weight > 0.  Its value is trilinear: along x
 *      first (f_a + w_x (f_b - f_a)), then y, then z.
 *   4. The hit is the first k >= 1 where samples k-1 and k are valid, f_{k-1} >= 0 and f_k < 0 (marching cubes' inside
 *      when tsdf < 0, crossed from the front): depth = z_{k-1} + delta (f_{k-1}/(f_{k-1} - f_k)), X* = C + depth D.
 *   5. Normal: n_i = f(X* + voxel_size e_i) - f(X* - voxel_size e_i) (each coordinate offset by one rounded add or
 *      subtract), NaN unless all 6 samples are valid; R n, normalised by sqrt((n_0 n_0 + n_1 n_1) + n_2 n_2): the camera
 *      frame, pointing towards free space (lmbspecialops' depth_to_normals convention).
 *   6. Colour: the trilinear colour at X*, rounded half to even and clamped to [0, 255]; 0 when X*'s cube is not valid.
 *   7. No hit: depth and normal NaN, colour 0.
 * 0 < step <= 1; h*w < 2^24. */
int demon_tsdf_raycast_f32(const float* tsdf, const float* weight, const float* color, int nx, int ny, int nz, const float* origin,
                           float voxel_size, const float* K, const float* R, const float* t, const float* near, const float* far, float step,
                           int n, int h, int w, float* depth, float* normals, uint8_t* colors, void* stream);
/* bytes of device scratch demon_sparse_tsdf_raycast_f32 needs for m >= 1 blocks */
int64_t demon_sparse_tsdf_raycast_scratch_bytes(int m);
/* far [n] (device float32): for each frame the largest camera z ((R_20 X_0 + R_21 X_1) + R_22 X_2) + t_2 over the 8 corners
 * X = origin + voxel_size*(8b + (0 or 8)) of every one of the m >= 1 blocks, reduced on the device. */
int demon_sparse_tsdf_far_f32(const int* blocks, int m, const float* origin, float voxel_size, const float* R, const float* t, int n, float* far,
                              void* stream);
/* demon_tsdf_raycast_f32 on the m >= 1 blocks of a sparse volume and its table: a cube's corners are resolved through the
 * blocks' neighbour table (built in scratch), and the table is probed when a ray enters another block.  The samples of a
 * block that is not allocated are invalid, so the march jumps over them, with the same result as evaluating each. */
int demon_sparse_tsdf_raycast_f32(const float* tsdf, const float* weight, const float* color, const int* blocks, int m, const int64_t* keys,
                                  const int* values, int64_t capacity, void* scratch, const float* origin, float voxel_size, const float* K,
                                  const float* R, const float* t, const float* near, const float* far, float step, int n, int h, int w,
                                  float* depth, float* normals, uint8_t* colors, void* stream);
/* Marching cubes of the cubes of pool blocks first .. first+count-1 only (1 <= count, first + count <= m), their
 * neighbours resolved among all m blocks: demon_sparse_tsdf_mesh_count_f32 and demon_sparse_tsdf_mesh_f32 are these with
 * first = 0, count = m.  Scratch: demon_sparse_tsdf_mesh_scratch_bytes(count). */
int demon_sparse_tsdf_mesh_range_count_f32(const float* tsdf, const float* weight, const int* blocks, int m, int first, int count,
                                           const int64_t* keys, const int* values, int64_t capacity, void* scratch, int64_t* triangles,
                                           void* stream);
int demon_sparse_tsdf_mesh_range_f32(const float* tsdf, const float* weight, const float* color, const int* blocks, int m, int first,
                                     int count, const float* origin, float voxel_size, const void* scratch, float* vertices, uint8_t* colors,
                                     int* faces, void* stream);

/* ------------------------------------------------------------------------
 * The indexed mesh (TsdfVolume.indexed_mesh, SparseTsdfVolume.indexed_mesh): marching cubes' surface with one vertex per
 * edge instead of one per triangle corner.  Edge (g, a) runs from voxel g to g + e_a, a in {x, y, z}; in a sparse volume
 * it belongs to the block that holds g.
 *   1. Vertices: one for each edge that changes sign (tsdf < 0 at one end only) and lies in a cube that is not skipped
 *      (all 8 corners stored with weight > 0), keyed by the edge, not by its position.  Its position and colour are the
 *      soup's (demon_marching_cubes_f32) for that edge, bit for bit: mu = f0/(f0 - f1), p0 + mu (p1 - p0).
 *   2. Order: dense, ascending 3 (linear index of g, x fastest) + a; sparse, ascending (packed key of g's block, local
 *      linear index of g, a), whatever the pool's layout.
 *   3. Faces [T,3] int32: the soup's triangles, each corner replaced by its edge's vertex index, winding kept.  Dense: the
 *      soup's order.  Sparse: ascending block key, then the cube's local index, then the table's order.
 *   4. Normals (world frame, towards increasing tsdf): with d_i(p) = f(p + e_i) - f(p - e_i) at p = g and p = g + e_a,
 *      n_i = d_i(g) + mu (d_i(g + e_a) - d_i(g)), then n_i / sqrt((n_0 n_0 + n_1 n_1) + n_2 n_2).  NaN when any of the 10
 *      other voxels it reads is not stored or has weight 0, or when the norm is 0.
 *   5. Colour as the soup's, rounded half to even and clamped.
 * Every step is one round-to-nearest float32 operation in the order written.  Faces are int32: callers refuse 2^31
 * vertices or more (the counts are int64).  The work: every valid cube sets its edges' bits (atomicOr, so the masks do
 * not depend on scheduling), a scan of the bit counts gives each 48-word segment (512 voxels of 3 edges: a block, or 512
 * consecutive voxels of a dense box) its first vertex, and vertices and face corners find their index by popcount.
 * ---------------------------------------------------------------------- */
/* bytes of device scratch the dense indexed-mesh entries need (0 for an invalid volume) */
int64_t demon_tsdf_indexed_mesh_scratch_bytes(int nx, int ny, int nz);
/* Dense, step 1: marks the edges and counts: counts[0] = V vertices, counts[1] = T triangles (device int64 [2]). */
int demon_tsdf_indexed_mesh_count_f32(const float* tsdf, const float* weight, int nx, int ny, int nz, void* scratch, int64_t* counts,
                                      void* stream);
/* Dense, step 2, on the scratch step 1 filled and the same volume: vertices [V,3] float32, normals [V,3] float32 (NULL: not
 * computed), colors [V,3] uint8 (with color; NULL without), faces [T,3] int32. */
int demon_tsdf_indexed_mesh_f32(const float* tsdf, const float* weight, const float* color, int nx, int ny, int nz, const float* origin,
                                float voxel_size, const void* scratch, float* vertices, float* normals, uint8_t* colors, int* faces,
                                void* stream);
/* Sparse.  The caller holds, for all B blocks of the volume (on the device or not), masks uint32 [B,48] zeroed, base int32
 * [B,48], and for the pool it works on a rank map: rank[b] = the key rank (0..B-1) of pool block b.  A pool may be the
 * volume's own or a scratch pool of a chunk of blocks with their neighbours and its own table; the entries below work on
 * its blocks first .. first+count-1 and resolve their neighbours among all m.  Scratch:
 * demon_sparse_tsdf_mesh_scratch_bytes(count).
 *   mark (every chunk), then scan (once: V into *vertices), then for every chunk range_count and range (vertices of the
 *   chunk's blocks, wherever their rank puts them, and faces of its cubes).  Every triangle of a chunk's cubes uses edges
 *   of its blocks and their +x, +y, +z neighbours; normals read all 26 neighbours. */
int demon_sparse_tsdf_edge_mark_f32(const float* tsdf, const float* weight, const int* blocks, int m, int first, int count, const int64_t* keys,
                                    const int* values, int64_t capacity, const int* rank, void* scratch, uint32_t* masks, void* stream);
/* bytes of device scratch demon_sparse_tsdf_edge_scan needs for B >= 1 blocks */
int64_t demon_sparse_tsdf_edge_scan_bytes(int blocks);
/* The vertex count of the B blocks' masks into *vertices (device int64), and base: each mask word's first vertex. */
int demon_sparse_tsdf_edge_scan(const uint32_t* masks, int blocks, void* scratch, int* base, int64_t* vertices, void* stream);
/* demon_sparse_tsdf_mesh_range_count_f32 with the cubes enumerated block by block in order[0], order[1], ... (a
 * permutation of first .. first+count-1; NULL: pool order), so the range entry writes faces in that order. */
int demon_sparse_tsdf_indexed_mesh_range_count_f32(const float* tsdf, const float* weight, const int* blocks, int m, int first, int count,
                                                   const int* order, const int64_t* keys, const int* values, int64_t capacity, void* scratch,
                                                   int64_t* triangles, void* stream);
/* On the scratch range_count filled: the vertices [V,3] (normals and colors as the dense entry) of the blocks first ..
 * first+count-1 at their global indices (skipped with vertices NULL), and the faces of their cubes (skipped with faces NULL)
 * from faces[0]. */
int demon_sparse_tsdf_indexed_mesh_range_f32(const float* tsdf, const float* weight, const float* color, const int* blocks, int m, int first,
                                             int count, const int* order, const int64_t* keys, const int* values, int64_t capacity,
                                             const int* rank, const uint32_t* masks, const int* base, const float* origin, float voxel_size,
                                             const void* scratch, float* vertices, float* normals, uint8_t* colors, int* faces,
                                             void* stream);

/* ------------------------------------------------------------------------
 * Streaming a sparse volume's blocks between the device and pinned host memory (SparseTsdfVolume's max_device_blocks).
 * A table value >= 0 is a pool index, -1 a block new in the running call, and -2 - s a block kept in host slot s; every
 * entry above reads a negative value as a block that is not stored.  Host slots hold tsdf and weight [8,8,8] float32 and
 * colour [8,8,8,3] in pinned host memory the device maps (cudaHostAlloc; checked with cudaPointerGetAttributes), and the
 * slots' coordinates [3] int32 and stamps int32 on the device.
 * ---------------------------------------------------------------------- */
/* tiles [n, ceil(h/8), ceil(w/8)] float32: the largest finite depth > 0 of each 8x8 pixel tile, -inf when there is none. */
int demon_sparse_tsdf_depth_tiles_f32(const float* depth, int n, int h, int w, float* tiles, void* stream);
/* out[b] = mark for every one of the m blocks that some frame reaches; other entries are not written.  One thread per block
 * and frame.  Block B reaches frame f by this rule, every step one round-to-nearest float32 operation in the order written:
 *   1. The block's AABB widened by 3 voxels and 2 trunc: m = trunc + trunc, lo_a = (o_a + vs (float)(8 B_a - 3)) - m,
 *      hi_a = (o_a + vs (float)(8 B_a + 10)) + m.
 *   2. For its 8 corners X: z = ((R_20 X_0 + R_21 X_1) + R_22 X_2) + t_2, and x, y likewise with rows 0 and 1 and t_0, t_1;
 *      zmin and zmax = the least and largest z.  A block with zmax <= vs (not > vs) is not reached.  When a corner has
 *      z <= vs, the block is tested against every tile with zmin = 0.
 *      Otherwise u = (fx x)/z + cx and v = (fy y)/z + cy for every corner, and the pixel rectangle is
 *      floor(min u) - 1 .. floor(max u) + 1 by floor(min v) - 1 .. floor(max v) + 1; a rectangle outside the image does
 *      not reach, and one inside is clipped to it.
 *   3. The block is reached when some tile of frame f under the rectangle has tile + trunc >= zmin.
 * With demon_sparse_tsdf_depth_tiles_f32's tiles and the integration's trunc this reaches every block holding a voxel
 * demon_sparse_tsdf_integrate_f32 would change; with every tile set to a ray cast's far and trunc 0 it reaches every block
 * holding a corner of a sample, normal sample or colour lookup of demon_sparse_tsdf_raycast_f32 (DESIGN.md §3.9).
 * trunc finite and >= 0. */
int demon_sparse_tsdf_reach_f32(const int* blocks, int m, const float* origin, float voxel_size, float trunc, const float* tiles, const float* K,
                                const float* R, const float* t, int n, int h, int w, int* out, int mark, void* stream);
/* One warp per block: copies pool block src[i] (tsdf, weight, colour with color) to host slot slots[i], its coordinates and
 * stamp to host_blocks and host_stamps, and sets its table value to -2 - slots[i].  The pool is left as it was. */
int demon_sparse_tsdf_evict(const float* tsdf, const float* weight, const float* color, const int* blocks, const int* stamps, const int64_t* keys,
                            int* values, int64_t capacity, const int* src, const int* slots, int count, float* host_tsdf, float* host_weight,
                            float* host_color, int* host_blocks, int* host_stamps, void* stream);
/* One warp per block: copies host slot slots[i] to pool block dst[i] with its coordinates; with stamps, sets stamps[dst[i]]
 * = stamp; with keys (a table), sets the block's value to dst[i].  With keys NULL it copies into any pool, such as a
 * mesh chunk's. */
int demon_sparse_tsdf_restore(const float* host_tsdf, const float* host_weight, const float* host_color, const int* host_blocks, const int* slots,
                              const int* dst, int count, float* tsdf, float* weight, float* color, int* blocks, int* stamps, int stamp,
                              const int64_t* keys, int* values, int64_t capacity, void* stream);
/* Sets the value of every block first .. first+count-1 of blocks to its index, inserting keys the table lacks (count <
 * capacity; a fresh table from demon_sparse_tsdf_rehash needs capacity >= 2 count to stay half empty). */
int demon_sparse_tsdf_index(int64_t* keys, int* values, int64_t capacity, const int* blocks, int first, int count, void* stream);

/* ------------------------------------------------------------------------
 * Connected components of an indexed mesh, and the removal of the small ones (demon_b200.mesh; csrc/mesh.cu).  The mesh
 * is V vertices and faces [F,3] int32 with every index in [0, V) (the caller checks this: an index outside it is
 * undefined behaviour); degenerate faces are allowed.
 *   1. Connectivity: two vertices are connected when some face contains both, and a component is a class of that
 *      relation.  It is by index, not by position: coincident vertices stay apart.  A vertex no face uses is a component
 *      of its own with 0 triangles.
 *   2. Labels: the components are numbered 0 .. C-1 in ascending order of their smallest vertex index (so vertex 0 is in
 *      component 0); labels [V] int32 is each vertex's, and a face's is labels[faces[f,0]].  They depend on the faces
 *      alone, never on scheduling.
 *   3. Sizes: triangles [C] and vertices [C] int64 count each component's faces and vertices.
 *   4. Selection: component c is kept when triangles[c] >= min_triangles and, with a selection select [C] uint8 (NULL:
 *      every component), select[c] != 0.
 *   5. Filter: the kept vertices in ascending original index, with their vertices, normals and colours copied bit for bit,
 *      and the kept faces in their original order, each index replaced by its vertex's new index: a boolean-mask
 *      compaction.
 * The work: a lock-free union-find (one thread per face, atomicCAS hooking the larger root under the smaller, so a
 * tree's root is its smallest vertex), a tile scan of the roots for the labels, integer atomics for the sizes, and tile
 * scans of the kept vertices and faces for the filter.  All four entries take the same scratch.
 * ---------------------------------------------------------------------- */
/* bytes of device scratch the entries below need for V vertices and F faces (0 for invalid sizes) */
int64_t demon_mesh_components_scratch_bytes(int num_vertices, int64_t num_faces);
/* labels [V] int32 (rule 2) and the component count C into *components (device int64). */
int demon_mesh_components_count(const int* faces, int64_t num_faces, int num_vertices, void* scratch, int* labels, int64_t* components,
                                void* stream);
/* triangles [C] and vertices [C] int64 (rule 3) from the labels of demon_mesh_components_count and its count C. */
int demon_mesh_component_sizes(const int* faces, int64_t num_faces, const int* labels, int num_vertices, int64_t components,
                               int64_t* triangles, int64_t* vertices, void* stream);
/* The filter, step 1: counts[0] = the kept vertices, counts[1] = the kept faces (device int64 [2]), by rule 4 from the
 * labels and triangle counts above. */
int demon_mesh_filter_count(const int* faces, int64_t num_faces, const int* labels, int num_vertices, const int64_t* triangles,
                            int64_t min_triangles, const uint8_t* select, void* scratch, int64_t* counts, void* stream);
/* The filter, step 2, on the scratch step 1 filled and the same arguments: out_vertices [V',3] float32, out_normals
 * [V',3] float32 (with normals [V,3]; NULL with NULL), out_colors [V',3] uint8 (with colors [V,3]; NULL with NULL) and
 * out_faces [F',3] int32 (rule 5; NULL when F' = 0). */
int demon_mesh_filter(const int* faces, int64_t num_faces, const int* labels, int num_vertices, const int64_t* triangles,
                      int64_t min_triangles, const uint8_t* select, void* scratch, const float* vertices, const float* normals,
                      const uint8_t* colors, float* out_vertices, float* out_normals, uint8_t* out_colors, int* out_faces, void* stream);

/* ------------------------------------------------------------------------
 * Image input (examples/example.py:15-42 resizes every image with PIL.Image.resize).
 * ---------------------------------------------------------------------- */
/* resample filters, with Pillow's enum values (PIL.Image.Resampling) */
#define DEMON_RESAMPLE_NEAREST   0
#define DEMON_RESAMPLE_BILINEAR  2
#define DEMON_RESAMPLE_BICUBIC   3
/* PIL.Image.resize((ow, oh), resample) of n RGB uint8 images, bit for bit: src [n,h,w,3] with `src_sn` bytes between
 * images and `src_sy` between rows (pixel stride 3, channel stride 1) -> dst [n,oh,ow,3] contiguous.  Sides 1..8192,
 * n 0..65535.  Other filters (LANCZOS, BOX, HAMMING) are DEMON_E_INVALID. */
int demon_resize_u8(const uint8_t* src, int64_t src_sn, int64_t src_sy, int n, int h, int w, uint8_t* dst, int oh, int ow,
                    int resample, void* stream);
/* adjust_intrinsics (dataset_tools/view_tools.py:97-172) of n RGB uint8 images, the image part, bit for bit with Pillow:
 * image i of src (addressed as in demon_resize_u8) with intrinsics K[i] = (fx, fy, cx, cy) in pixels (DEVICE doubles [n,4],
 * so a captured graph replays with new values in the same buffer; the skew is ignored) is resized to
 * rw = trunc(w fx_new/fx) x rh = trunc(h fy_new/fy) with BILINEAR if fx_new/fx > 1, else LANCZOS, and cropped to
 * dst [n,oh,ow,3] from x0 = rint(cx fx_new/fx - cx_new), y0 = rint(cy fy_new/fy - cy_new), filling with 127 outside the
 * resized image.  status [n] (device): 0 ok, 1 fill was added (the reference's printed warning), 2 invalid K (non-finite or
 * non-positive focal length, non-finite principal point, rw or rh outside 1..8192, an offset beyond +-2^24): all fill.
 * The crop is the correct one where the reference's safe_crop_image is not (a box leaving the image with x0 > 0 or y0 > 0,
 * DESIGN.md section 7).  Sides 1..8192 and h <= 100 w (Pillow reorders its passes beyond), n 0..65535. */
int demon_adjust_intrinsics_u8(const uint8_t* src, int64_t src_sn, int64_t src_sy, int n, int h, int w, const double* K, double fx_new,
                               double fy_new, double cx_new, double cy_new, uint8_t* dst, int oh, int ow, uint8_t* status,
                               void* stream);

/* ------------------------------------------------------------------------
 * Dataset tools (python/depthmotionnet/dataset_tools): selecting multi-view samples from RGB-D sequences.
 * ---------------------------------------------------------------------- */
/* measure_sharpness (helpers.py:23-31) of n RGB uint8 frames, bit for bit: out[i] = np.var(laplace(grey)) as float32, with
 * grey Pillow's convert('L'), laplace scipy's (mode 'reflect') and the variance numpy's pairwise float32 sums.  images
 * [n,h,w,3] with `stride_n` bytes between frames and `stride_y` between rows (pixel stride 3, channel stride 1).
 * h*w < 2^24 (n must be exact in float32), n >= 0. */
int demon_sharpness_u8(const uint8_t* images, int64_t stride_n, int64_t stride_y, int n, int h, int w, float* out, void* stream);
/* sun3d_utils.read_depth (sun3d_utils.py:60-72) on n decoded depth PNGs, bit for bit: raw [n,h,w] uint16 ->
 * depth [n,h,w] float32 = float32(double((d >> 3) | (d << 13) in uint16) / 1000), and valid_counts [n] int64 = the number of
 * finite depths > 0 of each frame.  n up to 65535. */
int demon_sun3d_depth_u16(const uint16_t* raw, int n, int h, int w, float* depth, int64_t* valid_counts, void* stream);
/* compute_depth_ratios (view_tools_cython.pyx:107-191) of n_pairs ordered view pairs, bit for bit: depth [n_views,h,w]
 * camera z; per view K [3,3], R [3,3], t [3] and P = K [R|t] [3,4] (float32, built as the .pyx wrapper builds them);
 * pairs [n_pairs,2] int32 (i, j) -> ratios [n_pairs,h,w] = the ratio map of view i against view j.  Where the .pyx would
 * read past depth j (a lookup at flat index y2*w + x2 >= h*w) the ratio is NaN.  h*w < 2^24. */
int demon_depth_ratios_f32(const float* depth, const float* K, const float* R, const float* t, const float* P, int n_views, int h, int w,
                           const int* pairs, int n_pairs, float* ratios, void* stream);
/* the same without the maps: counts [n_pairs,2] int64 = (finite ratios, finite ratios r with lo < r < hi) of each pair,
 * what check_depth_consistency (view_tools.py:62-94) needs from a map.  Exact integer counts, independent of scheduling. */
int demon_depth_consistency_counts_f32(const float* depth, const float* K, const float* R, const float* t, const float* P, int n_views,
                                       int h, int w, const int* pairs, int n_pairs, float lo, float hi, int64_t* counts, void* stream);

/* ------------------------------------------------------------------------
 * Multi-view training reader (multivih5datareaderop/multivih5datareader.cpp): its per-pixel compute.
 * ---------------------------------------------------------------------- */
/* One view of a demon_datareader_prepare call.  image_offset / depth_offset are byte offsets into `staging`: the source
 * image uint8 [height,width,3] RGB and its depth [height,width], float32 or (depth_f16) IEEE half.  k = the intrinsics
 * normalised like prepareScene (:1393-1396) and cast to float: fx/W, skew (in pixels, not normalised), cx/W, fy/H, cy/H.
 * ray_length: the depth is the distance along the ray and is converted to camera z. */
typedef struct {
  int64_t image_offset, depth_offset, pool_index;
  int32_t width, height, depth_f16, ray_length;
  float k[5];
  int32_t pad;
} demon_datareader_view;

/* One batch item of demon_datareader_batch.  flags bit 0 = rot180, bit 1 = mirror_x.  aug = the colour draws hue, sat,
 * val, contrast, brightness, gamma.  cam[i] = view i's [fx, skew, cx, fy, cy] as in demon_datareader_view, then R
 * row-major [9] and t [3], cast to float from the unrotated double pose. */
typedef struct {
  int32_t view1, view2, flags, pad;
  double depth_scale_factor;
  float aug[6];
  float cam[2][17];
} demon_datareader_item;

/* prepareScene (:1384-1520) of n_views views into the pool at their pool_index: pool_image [*,h,w,3] uint8 and pool_depth
 * [*,h,w] float32 camera z.  The image is downscaled as cv::resize(INTER_AREA) does for width >= w and height >= h, in
 * OpenCV's three paths (2x2, other integer factors, general; DESIGN.md section 3.8), the depth by cv::resize(INTER_NEAREST);
 * both bit for bit OpenCV 4.13.0.
 * One launch.  The caller guarantees width >= w, height >= h, both <= 8192, and offsets inside staging. */
int demon_datareader_prepare(const uint8_t* staging, const demon_datareader_view* views, int n_views, int h, int w, uint8_t* pool_image,
                             float* pool_depth, void* stream);
/* The batch loop's outputs (:1585-1950) of `batch` items (a device table) from the prepared pool, in one launch:
 * image_pair [batch,6,h,w], flow [batch,2,h,w], depth and depthmasks [batch,1 or 2 (depth_pair),h,w]; a NULL output is
 * skipped.  colour applies augmentImage (:641-714) with each item's draws.  The caller guarantees view indices inside the
 * pool. */
int demon_datareader_batch(const uint8_t* pool_image, const float* pool_depth, int h, int w, const demon_datareader_item* items, int batch,
                           int colour, float range_min, float range_max, float min_depth, float max_depth, int inverse_depth, int depth_pair,
                           int border1, int border2, float* image_pair, float* flow, float* depth, float* depthmasks, void* stream);

/* ------------------------------------------------------------------------
 * Network graphs (python/depthmotionnet/networks_original.py).
 * One handle = the five blocks netFlow1, netDM1, netFlow2, netDM2, netRefine for a
 * fixed batch size at 256x192 (networks_original.py:38-42), plus a refinement block that
 * is size generic (blocks_original.py:466-475).  All device memory (packed weights,
 * activation workspace) is allocated in demon_net_create / demon_net_finalize.
 * ---------------------------------------------------------------------- */
typedef struct demon_net demon_net;

/* precision of the tensor-core convolution path */
#define DEMON_PREC_FP32_SIMT  0   /* CUDA-core fp32 FFMA for every layer                           */
#define DEMON_PREC_3XTF32     1   /* wgmma kind tf32 with error compensation (fp32-grade)         */
#define DEMON_PREC_TF32       2   /* single-pass wgmma kind tf32 (fast mode, ~1e-3 relative)      */
#define DEMON_PREC_FP16       3   /* wgmma kind f16, FP32 accumulators (fast mode, ~1e-3 relative)
 * FP16: the tensor-core layers round their weights and input activations to FP16 (round to nearest even, 2^-11 relative);
 * accumulation, bias, activations in memory and the layers without a tensor-core plan (dense, small outputs) stay fp32.
 * demon_net_finalize refuses (DEMON_E_INVALID, naming the variable) a tensor-core layer's kernel with a value FP16 cannot
 * hold: |w| > 65504 or not finite.  An input activation is converted as IEEE does: a magnitude of 65520 (65504 + half an
 * FP16 ulp) or more becomes +-inf, so an out-of-range activation shows up as non-finite outputs, not as wrong finite
 * ones. */

/* replaces BootstrapNet/IterativeNet/RefinementNet.__init__ (networks_original.py:22-57,92-152,202-234).
 * refine_h/refine_w: input size of the refinement block (192, 256 for the standard pipeline). */
int demon_net_create(demon_net** net, int batch, int refine_h, int refine_w, int precision);
void demon_net_destroy(demon_net* net);

/* replaces tf.train.Saver().restore (examples/example.py:82-83): one call per TF variable,
 * `name` e.g. "netFlow1/conv1y/kernel"; `data` is a HOST array in TensorFlow's layout
 * (conv [kh,kw,cin,cout], conv2d_transpose [kh,kw,cout,cin], dense [in,out], bias [cout]). */
int demon_net_set_weight(demon_net* net, const char* name, const float* data_host,
                         const int64_t* shape, int rank);
/* number of variables the graphs need / already set; name of the i-th variable */
int demon_net_num_variables(const demon_net* net);
const char* demon_net_variable_name(const demon_net* net, int i);
/* packs the weights for the device kernels and uploads them; required before any forward */
int demon_net_finalize(demon_net* net);

/* data_format: 0 = channels_first (NCHW), 1 = channels_last (NHWC) for every image-like tensor */

/* replaces BootstrapNet.eval (networks_original.py:60-88).
 * image_pair [B,6,192,256], image2_2 [B,3,48,64] ->
 * flow5 [B,2,6,8], flow2 [B,2,48,64], depth2 [B,1,48,64], normal2 [B,3,48,64], rotation [B,3], translation [B,3] */
int demon_bootstrap_forward(demon_net* net, const float* image_pair, const float* image2_2,
                            float* flow5, float* flow2, float* depth2, float* normal2,
                            float* rotation, float* translation, int data_format, void* stream);

/* replaces IterativeNet.eval (networks_original.py:154-198); same outputs as bootstrap. */
int demon_iterative_forward(demon_net* net, const float* image_pair, const float* image2_2,
                            const float* depth2_in, const float* normal2_in,
                            const float* rotation_in, const float* translation_in,
                            float* flow5, float* flow2, float* depth2, float* normal2,
                            float* rotation, float* translation, int data_format, void* stream);

/* replaces RefinementNet.eval (networks_original.py:236-255).
 * image1 [B,3,H,W], depth2 [B,1,H/4,W/4] -> depth0 [B,1,H,W] */
int demon_refine_forward(demon_net* net, const float* image1, const float* depth2, float* depth0,
                         int data_format, void* stream);

/* ------------------------------------------------------------------------
 * The v2 network (python/depthmotionnet/v2/networks.py, the one training/v2/training.py trains): a second plan over the
 * same kernels, with TF 'same' padding, the dense5 layer of every trunk, the motion branch of v2 and a refinement block
 * that also predicts normal0.  demon_net_set_weight / _num_variables / _variable_name / _finalize / _destroy, the fused
 * pipeline, the profile and the debug entries take either kind of handle; every stage-wise or block entry takes one kind
 * only and returns DEMON_E_INVALID for the other (the entries above are v1's, the *_v2 entries below v2's).  float32
 * device entries only.
 * ---------------------------------------------------------------------- */
int demon_net_create_v2(demon_net** net, int batch, int refine_h, int refine_w, int precision);
/* 1 for a handle of demon_net_create, 2 for one of demon_net_create_v2, 0 for NULL */
int demon_net_variant(const demon_net* net);
/* BootstrapNet.eval / IterativeNet.eval of v2 (v2/networks.py:48-75,127-172): arguments and outputs as the v1 entries */
int demon_bootstrap_forward_v2(demon_net* net, const float* image_pair, const float* image2_2,
                               float* flow5, float* flow2, float* depth2, float* normal2,
                               float* rotation, float* translation, int data_format, void* stream);
int demon_iterative_forward_v2(demon_net* net, const float* image_pair, const float* image2_2,
                               const float* depth2_in, const float* normal2_in,
                               const float* rotation_in, const float* translation_in,
                               float* flow5, float* flow2, float* depth2, float* normal2,
                               float* rotation, float* translation, int data_format, void* stream);
/* RefinementNet.eval of v2 (v2/networks.py:204-228): image1 [B,3,H,W], depth2 [B,1,H/4,W/4] -> depth0 [B,1,H,W] and
 * normal0 [B,3,H,W] (may be NULL).  normal2 is taken like the reference takes it and not read (may be NULL). */
int demon_refine_forward_v2(demon_net* net, const float* image1, const float* depth2, const float* normal2,
                            float* depth0, float* normal0, int data_format, void* stream);
/* One block of v2/blocks.py under a variable scope of training/v2/training.py, on each sample's own camera.
 * demon_flow_block_forward_v2: flow_block, scope "netFlow1" or "netFlow2" -> flowconf5 [B,4,6,8] and flowconf2 [B,4,48,64]
 * (flow x, y, confidence x, y).  netFlow2 needs image2_2 [B,3,48,64], intrinsics and the previous prediction's depth2
 * [B,1,48,64], normal2 [B,3,48,64], rotation [B,3] and translation [B,3]; netFlow1 takes none of them (image2_2 is
 * accepted and not read).
 * demon_depthmotion_block_forward_v2: depthmotion_block, scope "netDM1" or "netDM2": image_pair, image2_2, prev_flow2
 * [B,2,48,64] and prev_flowconf2 [B,4,48,64] always; netDM2 also needs prev_rotation, prev_translation and intrinsics, which
 * netDM1 refuses -> depth2, normal2, rotation, translation and scale [B,1]; any output may be NULL.
 * intrinsics: device float32 [B,4], normalised fx, fy, cx, cy of each sample (datareader INTRINSICS).  A mismatch between
 * the scope and the arguments returns DEMON_E_INVALID with the argument's name.  The blocks run on the net's buffers
 * like the stage entries above: calls on one handle must not overlap. */
int demon_flow_block_forward_v2(demon_net* net, const char* scope, const float* image_pair, const float* image2_2,
                                const float* intrinsics, const float* prev_depth2, const float* prev_normal2,
                                const float* prev_rotation, const float* prev_translation, float* flowconf5, float* flowconf2,
                                int data_format, void* stream);
int demon_depthmotion_block_forward_v2(demon_net* net, const char* scope, const float* image_pair, const float* image2_2,
                                       const float* prev_flow2, const float* prev_flowconf2, const float* prev_rotation,
                                       const float* prev_translation, const float* intrinsics, float* depth2, float* normal2,
                                       float* rotation, float* translation, float* scale, int data_format, void* stream);

/* ------------------------------------------------------------------------
 * The fused pipeline: bootstrap, `iterations` x iterative and refinement in one call that never leaves the device, the
 * whole of examples/example.py:87-99 (v2: examples/example_v2.py), on a handle of either kind; the handle says which
 * network runs.  One call is described by one demon_pipeline_args.
 * ---------------------------------------------------------------------- */
/* input kinds */
enum { DEMON_INPUT_F32 = 0, DEMON_INPUT_U8 = 1, DEMON_INPUT_RESIZE_U8 = 2, DEMON_INPUT_VIEWS_U8 = 3 };

/* One fused-pipeline call.  Every field is 64 bits wide, so the struct has no padding and equal calls are equal bytes: the
 * library keeps one CUDA graph per distinct call (the first call runs eagerly, the second captures, later ones replay),
 * keyed by these bytes.  A field the input kind does not read must be 0 / NULL, otherwise the call is refused.
 *
 * input, images, image2_2:
 *   DEMON_INPUT_F32: images float [B,6,192,256], the image pair; image2_2 float [B,3,48,64] or NULL.
 *   DEMON_INPUT_U8: images uint8 [B,2,192,256,3], image 1 then image 2 of every pair as PIL gives them (HWC RGB,
 *     examples/example.py:15-42); image2_2 uint8 [B,48,64,3] (the resized second image) or NULL.  `x/255 - 0.5` and the
 *     pair concat happen on the device in the kernel that feeds conv1y, with numpy's two float32 operations, so the outputs
 *     equal the F32 call's bit for bit; the host entry moves 4x fewer input bytes.
 *   DEMON_INPUT_RESIZE_U8: images uint8 [B,2,h,w,3] of any size with `sn`, `si`, `sy` bytes between samples, between the two
 *     images of a pair and between rows (pixel stride 3, channel stride 1, so a cropped view is read in place),
 *     1 <= h, w <= 8192.  Both images are resized to 256x192 with `resample` exactly like PIL.Image.resize
 *     (demon_resize_u8).  image2_2 NULL.  The outputs equal the U8 call on the resized bytes, bit for bit.
 *   DEMON_INPUT_VIEWS_U8: photos from any calibrated camera: images as for RESIZE_U8 with their intrinsics K [B,2,4] (fx,
 *     fy, cx, cy in pixels, DEVICE doubles).  Every image is adapted to the network's intrinsics, K_new = (0.89115971 * 256,
 *     1.18821287 * 192, 0.5 * 256, 0.5 * 192) at 256x192, exactly like demon_adjust_intrinsics_u8, with its status [B,2].
 *     image2_2 NULL.  The outputs equal the U8 call on the adapted bytes, bit for bit.  K and status are part of the
 *     CUDA-graph key: a replay reads the K buffer's current values.
 * image2_2_mode, how image2_2 is made when it is not given:
 *   0: median3x3_downsample twice of image 2 (examples/evaluation.py:170-173);
 *   1: image 2 resized to 64x48 with the call's filter (examples/example.py:22) -- RESIZE_U8 / VIEWS_U8 only;
 *   2: tf.image.resize_area of image 2's float planes to 48x64, the input training/v2/training.py:179 trains v2 on
 *      (demon_resize_area_f32 on x/255 - 0.5 for uint8 input) -- v2 handles only; image2_2 must be NULL.
 * iterations: 0..7.
 * Outputs, float32 channels_first, each may be NULL: depth0 [B,1,192,256], normal0 [B,3,192,256] (v2 handles only),
 *   rotation / translation [B,3], flow2 [B,2,48,64], depth2 [B,1,48,64], normal2 [B,3,48,64].
 * snapshots 0: the outputs after the last iteration and the refinement block.  snapshots 1: every intermediate prediction,
 *   as examples/evaluation.py:225-255 keeps them for an accuracy table.  Snapshot k = 0 is the bootstrap block's output,
 *   snapshot k = 1..iterations the output after iteration k; every output holds S = iterations + 1 snapshots [S,B,...].  The
 *   refinement block runs on every snapshot's depth2 iff depth0 is given (evaluation.py:249), and normal0 needs depth0.
 *   Snapshot k equals the stage-wise entries after k iterations bit for bit. */
typedef struct demon_pipeline_args {
  int64_t input;                       /* DEMON_INPUT_* */
  const void* images;
  const void* image2_2;
  int64_t image2_2_mode;
  int64_t sn, si, sy, h, w, resample;  /* RESIZE_U8 / VIEWS_U8 */
  const double* K;                     /* VIEWS_U8 */
  uint8_t* status;                     /* VIEWS_U8 */
  int64_t iterations;
  int64_t snapshots;
  float *depth0, *normal0, *rotation, *translation, *flow2, *depth2, *normal2;
} demon_pipeline_args;

/* The call on DEVICE pointers, asynchronous on `stream`.  Calls on one handle must not overlap.
 * DEMON_E_INVALID for an argument the struct's rules above refuse, a null images, or a net whose refinement block is not
 * 192x256; DEMON_E_STATE for a net that is not finalized, belongs to another device or has a layer trace set.  A refused
 * call launches nothing. */
int demon_pipeline_run(demon_net* net, const demon_pipeline_args* args, void* stream);
/* The same on HOST buffers in and out (pinned or pageable): F32 or U8 input, snapshots 0, depth0 required, flow2, depth2
 * and normal2 NULL.  H2D copies into the net's staging buffers, the pipeline, D2H copies of depth0, normal0, rotation and
 * translation, all inside the call.  With `synchronize` the call also synchronises the stream and returns DEMON_E_STATE if
 * a tensor-core pipeline wait timed out (demon_check_errors); this is the end-to-end path bench.py times.  Without it the
 * host outputs are valid once `stream` has been synchronised: with PINNED host buffers and two nets on two streams a caller
 * overlaps the copies of one batch with the compute of the other. */
int demon_pipeline_run_host(demon_net* net, const demon_pipeline_args* args, int synchronize, void* stream);

/* introspection for tests and bench */
int demon_net_batch(const demon_net* net);
int64_t demon_net_workspace_bytes(const demon_net* net);
/* number of kernel launches of the last fused-pipeline call without snapshots with `iterations` */
int demon_net_pipeline_launches(const demon_net* net, int iterations);
/* the same for the last call with snapshots (counted apart: snapshot calls leave the value above untouched) */
int demon_net_snapshot_launches(const demon_net* net, int iterations);
/* 1 if layer `tf_name` (e.g. "netRefine/conv1_1") runs on the tensor-core path */
int demon_net_layer_uses_tensor_cores(const demon_net* net, const char* tf_name);

/* Per-layer device timing with CUDA events recorded on the launching stream around every layer of the
 * forward calls issued between _begin and _end (synchronise the stream before _end).  Used by bench.py for
 * the roofline figure of the dominant kernel; off by default. */
int demon_net_profile_begin(demon_net* net);
int demon_net_profile_end(demon_net* net);
int demon_net_num_layers(const demon_net* net);
const char* demon_net_layer_name(const demon_net* net, int i);
/* uses_tc: kernel family of the layer -- 0 conv_simt_kernel (fp32 CUDA cores), 2 conv_tc_halo_kernel (wgmma, halo tile),
 * 3 conv_tc_halo_kernel in per-tap mode (one TMA box per filter tap) */
int demon_net_layer_profile(const demon_net* net, int i, double* ms, int64_t* calls, int* launches_per_call,
                            int* uses_tc);

/* 1 if a pipeline wait inside a tensor-core kernel has timed out on the current device since the flag was last
 * cleared (synchronises the device; does not clear). */
int demon_debug_tc_timeouts(void);
/* Synchronises the current device and returns DEMON_E_STATE if a bounded pipeline wait inside a tensor-core convolution
 * kernel timed out since the last check (such a kernel runs to completion with garbage instead of hanging the GPU),
 * DEMON_E_CUDA for a pending CUDA error, DEMON_OK otherwise.  Clears the flag.  The `_host` entry points that
 * synchronise call it themselves; callers of the asynchronous / device-pointer entry points call it after their own
 * synchronisation (replaces the `throw std::runtime_error` of _CHECK_CUDA_ERROR, lmbspecialops/src/cuda_helper.h:25-35). */
int demon_check_errors(void);
/* debug: host_out == NULL: switch the halo kernel's per-CTA wait-cycle counters on/off; otherwise copy [nblocks][16]
 * counters of the last launch to host_out. */
int demon_debug_tc_timing(int enable, int64_t* host_out, int nblocks);

/* debug: one text line per layer: its name, then its geometry as fixed key-value pairs
 *     <kind> H <h> W <w> cin <c> cin_buf <c> in_pitch <p> in_off <o> cout <c> out_pitch <p> out_off <o> kh <k> kw <k> sy <s> sx <s> leaky <0|1>
 *     scale <0|1> :
 * (kind conv / deconv / dense; H, W of the input; cin_buf = channels read, the ones past cin carry zero weights; scale 1:
 * channel 0 of the output is multiplied by a per-image scale), then the
 * kernel family and tiling plan it gets (works without a device as long as the net was created -- creation needs one;
 * see tools/describe_plan.py for the offline variant). Returns bytes written. */
int demon_debug_describe_layers(const demon_net* net, char* buf, int buflen);
/* debug, no device needed: demon_debug_describe_layers of the plan that demon_net_create (variant 1) or
 * demon_net_create_v2 (variant 2) would lay out for this batch, refinement size and precision.  A v2 conv's line carries
 * "tap0 <dy> <dx> :" after the geometry: the input offset of its first tap, minus TF's 'same' padding before. */
int demon_debug_describe_plan(int variant, int batch, int refine_h, int refine_w, int precision, char* buf, int buflen);

/* debug, a test entry like demon_conv_slice_nhwc: while set, the stage-wise entries (demon_bootstrap_forward,
 * demon_iterative_forward, demon_refine_forward) copy every layer's input slice (cin_buf channels, just before the layer
 * runs) to in[i] and its output slice (cout channels, just after) to out[i], as dense float32 [B,H,W,C] (dense layers:
 * [B,cin_buf] in the buffer's NHWC order and [B,cout]), on the launching stream; a null pointer skips that copy.  The last
 * refinement layer's output is read from the caller's depth0.  `in` and `out` are arrays of demon_net_num_layers(net)
 * device pointers in layer order (demon_net_layer_name); in == out == NULL clears the trace.  While a trace is set,
 * demon_pipeline_run and demon_pipeline_run_host return DEMON_E_STATE, so that no CUDA graph is captured with the copies
 * inside it.
 * Without a trace the forward passes are unchanged. */
int demon_debug_trace_layers(demon_net* net, float* const* in, float* const* out);

/* debug, no device needed: the kernel family and tiling plan one convolution shape would get */
int demon_debug_describe_conv(int B, int H, int W, int Cin, int in_pitch, int Cout, int out_pitch, int kh, int kw, int sy, int sx,
                              int deconv, int precision, char* buf, int buflen);

/* debug: device time (CUDA events on the launching stream) of the kernel launches of the last standalone convolution
 * call (demon_conv_slice_nhwc and the two entries below), in milliseconds (weight packing and uploads excluded); < 0 if
 * none was timed */
double demon_debug_last_conv_ms(void);

/* Standalone convolution on channel SLICES, the way the network's layers read and write their concat buffers: `in`
 * points at the first channel of a [B,H,W,*] slice of channel pitch in_pitch, `out` at the first channel of an output
 * slice of pitch out_pitch; only those Cin input and Cout output channels are read or written.  Kernel TF layout
 * [kh,kw,cin,cout] (host), or with `deconv` the k4 s2 transposed convolution (kh = kw = 4, sy = sx = 2) with kernel
 * [4,4,cout,cin].  At a tensor-core precision a shape the tensor-core path gets no plan for is refused (DEMON_E_INVALID). */
int demon_conv_slice_nhwc(const float* in, int in_pitch, float* out, int out_pitch, int B, int H, int W, int Cin, int Cout,
                          int kh, int kw, int sy, int sx, int deconv, const float* kernel_host, const float* bias_host,
                          int leaky, int precision, void* stream);

/* demon_conv_slice_nhwc (no transposed conv) with TF's 'same' padding, the padding of the v2 network's convolutions: along
 * each axis of size n with kernel k and stride s the first tap reads max((ceil(n/s) - 1) s + k - n, 0) / 2 pixels before the
 * output's first one (demon_conv_slice_nhwc uses k / 2, caffe padding). */
int demon_conv_slice_nhwc_same(const float* in, int in_pitch, float* out, int out_pitch, int B, int H, int W, int Cin, int Cout,
                               int kh, int kw, int sy, int sx, const float* kernel_host, const float* bias_host,
                               int leaky, int precision, void* stream);

/* Standalone convolution entry used by tests to compare the tensor-core path with the fp32 SIMT path on
 * the same NHWC tensors.  in [B,H,W,Cin], kernel TF layout [kh,kw,cin,cout] (host), bias [cout] (host)
 * -> out [B,ceil(H/sy),ceil(W/sx),Cout]; caffe padding (helpers.py:70-94). */
int demon_conv2d_nhwc(const float* in, float* out, int B, int H, int W, int Cin, int Cout,
                      int kh, int kw, int sy, int sx, const float* kernel_host, const float* bias_host,
                      int leaky, int precision, void* stream);
/* conv2d_transpose k4 s2 (blocks_original.py:97-110): in [B,H,W,Cin], kernel [4,4,cout,cin] (host)
 * -> out [B,2H,2W,Cout] */
int demon_deconv4x4s2_nhwc(const float* in, float* out, int B, int H, int W, int Cin, int Cout,
                           const float* kernel_host, const float* bias_host, int leaky, int precision,
                           void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DEMON_B200_H */
