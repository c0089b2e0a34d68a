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

/* introspection for tests and bench */
int demon_net_batch(const demon_net* net);
int64_t demon_net_workspace_bytes(const demon_net* net);
/* number of kernel launches of one demon_pipeline_forward with `iterations` */
int demon_net_pipeline_launches(const demon_net* net, int iterations);
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
 * 3 conv_tc_halo_kernel in per-tap mode (one TMA box per filter tap); 1 is not produced by this version */
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

/* debug: one text line per layer with the kernel family and tiling plan it gets (works without a device as long as the
 * net was created -- creation needs one; see tools/describe_plan.py for the offline variant). Returns bytes written. */
int demon_debug_describe_layers(const demon_net* net, char* buf, int buflen);

/* debug, no device needed: the kernel family and tiling plan one convolution shape would get */
int demon_debug_describe_conv(int B, int H, int W, int Cin, int in_pitch, int Cout, int out_pitch, int kh, int kw, int sy, int sx,
                              int deconv, int precision, char* buf, int buflen);

/* debug: device time (CUDA events on the launching stream) of the kernel launches of the last demon_conv2d_nhwc /
 * demon_deconv4x4s2_nhwc call, in milliseconds (weight packing and uploads excluded); < 0 if none was timed */
double demon_debug_last_conv_ms(void);

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
