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

/* The whole of examples/example.py:87-99 without leaving the device: bootstrap, `iterations` x
 * iterative, refinement.  image2_2 may be NULL: it is then computed as
 * median3x3_downsample(median3x3_downsample(image_pair[:,3:6])) (examples/evaluation.py:170-173).
 * Any output pointer may be NULL.  channels_first only. */
int demon_pipeline_forward(demon_net* net, const float* image_pair, const float* image2_2, int iterations,
                           float* depth0, float* rotation, float* translation,
                           float* flow2, float* depth2, float* normal2, void* stream);

/* ------------------------------------------------------------------------
 * The v2 network (python/depthmotionnet/v2/networks.py, the one training/v2/training.py trains): a second plan over the
 * same kernels, with TF 'same' padding, the dense5 layer of every trunk, the motion branch of v2 and a refinement block
 * that also predicts normal0.  demon_net_set_weight / _num_variables / _variable_name / _finalize / _destroy, the profile
 * and the debug entries take either kind of handle; every forward entry takes one kind only and returns DEMON_E_INVALID
 * for the other (the entries above are v1's, the *_v2 entries below v2's).  float32 device entries only.
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
/* bootstrap, `iterations` x iterative and refinement of v2 in one call, as demon_pipeline_forward (one CUDA graph per
 * distinct call, image2_2 may be NULL, any output may be NULL); normal0 [B,3,192,256].  channels_first only. */
int demon_pipeline_forward_v2(demon_net* net, const float* image_pair, const float* image2_2, int iterations,
                              float* depth0, float* normal0, float* rotation, float* translation,
                              float* flow2, float* depth2, float* normal2, void* stream);

/* The pipeline as examples/evaluation.py:225-255 runs it for an accuracy table: every intermediate prediction is kept.
 * Snapshot k = 0 is the bootstrap block's output, snapshot k = 1..iterations the output after iteration k; the arrays hold
 * S = iterations + 1 snapshots of the batch: flow2 [S,B,2,48,64], depth2 [S,B,1,48,64], normal2 [S,B,3,48,64],
 * rotation / translation [S,B,3].  depth0 [S,B,1,192,256], if not NULL, is the refinement block run on every snapshot's
 * depth2 (evaluation.py:249).  Inputs, image2_2 = NULL and the CUDA graph cache as demon_pipeline_forward; snapshot k
 * equals the stage-wise entries after k iterations bit for bit.  Any output pointer may be NULL. */
int demon_pipeline_forward_snapshots(demon_net* net, const float* image_pair, const float* image2_2, int iterations,
                                     float* flow2, float* depth2, float* normal2, float* rotation, float* translation,
                                     float* depth0, void* stream);

/* Same, HOST buffers in and out (pinned or pageable): H2D copies, the pipeline, D2H copies and a
 * stream synchronisation, all inside the call.  This is the end-to-end path bench.py times. */
int demon_pipeline_forward_host(demon_net* net, const float* image_pair_host, const float* image2_2_host,
                                int iterations, float* depth0_host, float* rotation_host,
                                float* translation_host, void* stream);
/* Same without the final synchronisation: the host outputs are valid once `stream` has been synchronised.  With PINNED
 * host buffers and two nets on two streams a caller overlaps the copies of one batch with the compute of the other. */
int demon_pipeline_forward_host_async(demon_net* net, const float* image_pair_host, const float* image2_2_host,
                                      int iterations, float* depth0_host, float* rotation_host,
                                      float* translation_host, void* stream);

/* The same pipeline on uint8 images, the form examples/example.py:15-42 starts from (PIL RGB, HWC): images [B,2,192,256,3]
 * (image 1 then image 2 of every pair), image2_2 [B,48,64,3] (the resized second image) or NULL (then it is computed with
 * median3x3_downsample twice, examples/evaluation.py:170-173).  `x/255 - 0.5` and the pair concat happen on the device in
 * the kernel that feeds conv1y, with numpy's two float32 operations, so the outputs equal the fp32 entry's bit for bit;
 * the host variants move 4x fewer input bytes. */
int demon_pipeline_forward_u8(demon_net* net, const uint8_t* images, const uint8_t* image2_2, int iterations, float* depth0,
                              float* rotation, float* translation, float* flow2, float* depth2, float* normal2, void* stream);
int demon_pipeline_forward_host_u8(demon_net* net, const uint8_t* images_host, const uint8_t* image2_2_host, int iterations,
                                   float* depth0_host, float* rotation_host, float* translation_host, void* stream);
int demon_pipeline_forward_host_u8_async(demon_net* net, const uint8_t* images_host, const uint8_t* image2_2_host, int iterations,
                                         float* depth0_host, float* rotation_host, float* translation_host, void* stream);

/* The same pipeline on image pairs of any size, resized on the device first, the whole of examples/example.py:15-42:
 * images [B,2,h,w,3] uint8 RGB with `sn`, `si`, `sy` bytes between samples, between the two images of a pair and between
 * rows (pixel stride 3, channel stride 1, so a cropped view is read in place), 1 <= h, w <= 8192.  Both images are resized
 * to 256x192 with `resample` exactly like PIL.Image.resize (demon_resize_u8), then image2_2 is
 *   image2_2_mode 0: median3x3_downsample twice of the resized second image (examples/evaluation.py:170-173), or
 *   image2_2_mode 1: the resized second image resized to 64x48 with the same filter (examples/example.py:22).
 * The outputs equal demon_pipeline_forward_u8 on the resized bytes, bit for bit. */
int demon_pipeline_forward_images_u8(demon_net* net, const uint8_t* images, int64_t sn, int64_t si, int64_t sy, int h, int w,
                                     int resample, int image2_2_mode, int iterations, float* depth0, float* rotation,
                                     float* translation, float* flow2, float* depth2, float* normal2, void* stream);

/* The same pipeline on photos from any calibrated camera: images as in demon_pipeline_forward_images_u8 with their
 * intrinsics K [B,2,4] (fx, fy, cx, cy in pixels, DEVICE doubles).  Every image is adapted to the network's intrinsics,
 * K_new = (0.89115971 * 256, 1.18821287 * 192, 0.5 * 256, 0.5 * 192) at 256x192, exactly like demon_adjust_intrinsics_u8
 * (status [B,2] as there); image2_2 is made from the adapted second image as image2_2_mode says.  The outputs equal
 * demon_pipeline_forward_u8 on the adapted bytes, bit for bit.  K and status are part of the CUDA-graph key: a replay
 * reads the K buffer's current values. */
int demon_pipeline_forward_views_u8(demon_net* net, const uint8_t* images, int64_t sn, int64_t si, int64_t sy, int h, int w,
                                    const double* K, uint8_t* status, int resample, int image2_2_mode, int iterations, float* depth0,
                                    float* rotation, float* translation, float* flow2, float* depth2, float* normal2, void* stream);

/* introspection for tests and bench */
int demon_net_batch(const demon_net* net);
int64_t demon_net_workspace_bytes(const demon_net* net);
/* number of kernel launches of one demon_pipeline_forward with `iterations` */
int demon_net_pipeline_launches(const demon_net* net, int iterations);
/* the same for the last demon_pipeline_forward_snapshots with `iterations` (counted apart: snapshot calls leave the value
 * above untouched) */
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
 * device pointers in layer order (demon_net_layer_name); in == out == NULL clears the trace.  While a trace is set, every
 * demon_pipeline_forward* entry returns DEMON_E_STATE, so that no CUDA graph is captured with the copies inside it.
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
