// Network plan of the DeMoN `networks_original` graphs: buffers, layers, glue kernels, C ABI.
//
// The five blocks (netFlow1, netDM1, netFlow2, netDM2, netRefine; networks_original.py:44,50,125,142,227)
// are laid out once, at demon_net_create, as lists of convolution problems over NHWC buffers carved
// out of one device workspace.  Skip-concats are channel slices of shared buffers (conv.cuh), the
// geometry ops between the blocks (blocks_original.py:155-187,336-366) run as two fused glue kernels
// that produce the `conv2_extra_inputs` tensor directly, and nothing on the forward path allocates,
// synchronises or touches the host.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <type_traits>
#include <vector>

#include "conv.cuh"
#include "conv_tc.cuh"
#include "geometry.cuh"
#include "images.cuh"

namespace demon {

namespace {

// ---------------------------------------------------------------------------------------------
// buffers and layers
// ---------------------------------------------------------------------------------------------
struct Buf {
  float* p = nullptr;
  int H = 0, W = 0, C = 0;  // NHWC [B,H,W,C]; C is the pixel pitch
  size_t offset = 0;        // floats from the workspace base
  size_t numel(int B) const { return (size_t)B * H * W * C; }
};

enum LayerKind { L_CONV, L_DECONV, L_DENSE };

struct Layer {
  std::string name;  // TF scope/name, e.g. "netFlow1/conv1y"
  LayerKind kind = L_CONV;
  Buf* in = nullptr;
  int in_coff = 0;
  int cin = 0;      // channels of the TF kernel
  int cin_buf = 0;  // channels read from the buffer (cin rounded up to 4; extra ones have zero weights)
  Buf* out = nullptr;
  int out_coff = 0;
  int cout = 0;
  int kh = 1, kw = 1, sy = 1, sx = 1;
  bool leaky = false;
  Buf* scale = nullptr;  // optional: channel 0 of the output is multiplied by scale[scale_coff + n*scale_stride]
  int scale_coff = 0;
  int scale_stride = 0;
  bool dense_nchw_flatten = false;  // motion_fc1: TF flattens NCHW (blocks_original.py:388-392)
  int dense_c = 0, dense_hw = 0;
  // v2 only.  tf_same: the taps of a conv sit where tf.layers.conv2d(padding='same') puts them (pad_before below) instead
  // of k/2 (caffe padding).  dense_nchw_unflatten: the output columns are reshaped to NCHW [dense_c, H, W] by TF
  // (v2/blocks.py:215), so they are permuted like the input rows.  nhwc: the dense layer reads channels [0, dense_c) of
  // every pixel of this buffer (gathered into `in` before it runs) and its output is scattered back into channels
  // [nhwc_out_coff, nhwc_out_coff + dense_c) of it (conv5_1_dense5, v2/blocks.py:198-215).
  bool tf_same = false;
  bool dense_nchw_unflatten = false;
  Buf* nhwc = nullptr;
  int nhwc_out_coff = 0;
  // expected TF variable shapes
  std::vector<int64_t> kshape;
  // device parameters
  int cout_pad = 0;
  float* w_dev[4] = {nullptr, nullptr, nullptr, nullptr};  // 1 (conv/dense) or 4 (deconv parity classes)
  float* bias_dev = nullptr;
  // tensor-core path
  TcLayer tc;
  bool use_tc() const { return tc.plan != nullptr; }
  // split-K for dense layers (SIMT path)
  int ksplit = 1;
};

// A block's layers, in the order they run: [begin, head_end) is conv1 / conv2 of the trunk (the pipeline hoists it out of
// its iteration loop), [head_end, end) the rest, which starts with the conv2_extra_inputs pair when the block has one.
// The refinement block has no head (head_end == begin).
struct Block { int begin = 0, head_end = 0, end = 0; };

// The outputs of a fused-pipeline call, in the C ABI's order; any pointer may be null (normal0: v2 nets only)
struct PipelineOutputs { float *depth0, *rotation, *translation, *flow2, *depth2, *normal2, *normal0; };

enum PipelineInput : int64_t { IN_FP32, IN_U8, IN_RESIZE, IN_VIEWS };
// NO_SNAPSHOTS: the last iteration's predictions and the refinement block; otherwise snapshot k (0 = bootstrap, k = after
// iteration k) of every output is its k-th [B, ...] slice, and SNAPSHOTS_REFINED runs the refinement block on every snapshot
// (examples/evaluation.py:225-255 refines all four)
enum SnapshotMode : int64_t { NO_SNAPSHOTS, SNAPSHOTS, SNAPSHOTS_REFINED };

// Everything one demon_pipeline_forward* call depends on, and so also the key of its CUDA graph: every field is 64 bits
// wide, so the struct has no padding and equal calls are equal bytes.  Entries value-initialise it (unused fields are 0).
struct PipelineCall {
  PipelineInput input;
  const float* image_pair;        // IN_FP32: [B,6,192,256]
  const float* image2_2;          // IN_FP32: [B,3,48,64] or null (median3x3_downsample twice)
  const uint8_t* images;          // IN_U8: [B,2,192,256,3]; IN_RESIZE / IN_VIEWS: [B,2,h,w,3] with strides sn, si, sy
  const uint8_t* image2_2_u8;     // IN_U8: [B,48,64,3] or null
  int64_t sn, si, sy, h, w, resample, image2_2_mode;
  const double* K;                // IN_VIEWS: [B,2,4], adapted to the network's intrinsics with status [B,2]
  uint8_t* status;
  int64_t iterations;
  PipelineOutputs out;
  SnapshotMode snapshots;
};
static_assert(std::has_unique_object_representations<PipelineCall>::value, "PipelineCall is compared with memcmp");

}  // namespace
}  // namespace demon

using namespace demon;

struct demon_net {
  int B = 0, RH = 0, RW = 0;
  int precision = DEMON_PREC_FP32_SIMT;
  int variant = 1;           // 1: networks_original (demon_net_create), 2: v2.networks (demon_net_create_v2); fixed at creation
  int device = 0;            // the CUDA device the handle was created on; every entry point checks it is current
  bool finalized = false;
  float* ws = nullptr;
  size_t ws_floats = 0;
  std::vector<std::unique_ptr<Buf>> bufs;
  std::vector<std::unique_ptr<Layer>> layers;
  std::map<std::string, Layer*> by_name;
  std::vector<std::string> var_names;
  std::map<std::string, std::vector<float>> host_vars;   // the weights set so far, TF layout; uploaded at finalize
  std::vector<void*> dev_allocs;
  int pipeline_launches[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  int snapshot_launches[8] = {0, 0, 0, 0, 0, 0, 0, 0};   // the same for demon_pipeline_forward_snapshots (kept apart: bench.py reads the above)
  // CUDA graphs of the fused pipeline, one per distinct call (launch-bound at small batch: ~270 launches)
  struct GraphEntry { PipelineCall call; cudaGraphExec_t exec; int launches; };
  std::vector<GraphEntry> graphs;
  cudaStream_t cap_stream = nullptr;   // capture happens on this private stream (the caller's may be the legacy default stream)
  // optional per-layer timing with CUDA events on the launching stream (bench.py's roofline leg)
  bool profiling = false;
  std::vector<cudaEvent_t> prof_events;      // pairs (start, stop)
  std::vector<int> prof_layer;               // layer index of every pair
  size_t prof_used = 0;
  std::vector<double> prof_ms;               // accumulated per layer
  std::vector<int64_t> prof_calls;
  // optional per-layer copies of every layer's input and output slice (demon_debug_trace_layers); one per layer, null skips
  bool tracing = false;
  std::vector<float*> trace_in, trace_out;

  // named buffers
  float* tc_scratch = nullptr;   // partial sums of the split-K tensor-core layers (conv_tc_halo.cu), sized at finalize
  Buf *cat2_f2, *cat2_d2;   // conv2 || conv2_extra_inputs of netFlow2 / netDM2: their conv2 half is loop invariant (see pipeline_body)
  Buf *img8, *i22, *i22_half, *c1y, *c1, *c2y, *cat2, *extra_in, *exy, *c21y, *concat2, *c3y, *c3, *c31y, *concat3, *c4y, *c4,
      *c41y, *concat4, *c5y, *c5, *c51y, *c51, *pf5a, *pf5, *p2a, *flowconf2, *dn2, *mc1, *fc1, *fc2, *motion;
  Buf *rin, *concat0, *rc1, *concat1, *rc2, *rc21, *pd0a, *rdepth0, *splitk;
  // v2 only (build_plan_v2): dense5's gathered input and its output row, the motion branch (its concat is mc1)
  Buf *d5in = nullptr, *d5out = nullptr, *mc3y = nullptr, *mc3 = nullptr, *mc4y = nullptr, *mc4 = nullptr, *mc5y = nullptr;
  // staging roles of the buffers above (see build_plan, build_plan_v2); host_normal0: v2 only
  Buf *pair_bytes, *i22_bytes, *planes2, *host_depth0, *host_motion, *host_normal0 = nullptr;
  // the five blocks' layer ranges
  Block flow1, dm1, flow2, dm2, refine;

  Buf* add_buf(int H, int W, int C) {
    bufs.emplace_back(new Buf());
    Buf* b = bufs.back().get();
    b->H = H; b->W = W; b->C = C;
    b->offset = ws_floats;
    ws_floats += (b->numel(B) + 63) / 64 * 64;  // 256-byte aligned slices
    return b;
  }
  Layer* add_layer(const std::string& name, LayerKind kind, Buf* in, int in_coff, int cin, Buf* out, int out_coff, int cout,
                   int kh, int kw, int sy, int sx, bool leaky) {
    layers.emplace_back(new Layer());
    Layer* l = layers.back().get();
    l->name = name; l->kind = kind; l->in = in; l->in_coff = in_coff; l->cin = cin; l->cin_buf = (cin + 3) / 4 * 4;
    l->out = out; l->out_coff = out_coff; l->cout = cout; l->kh = kh; l->kw = kw; l->sy = sy; l->sx = sx; l->leaky = leaky;
    l->cout_pad = (cout + 3) / 4 * 4;
    if (kind == L_CONV) l->kshape = {kh, kw, cin, cout};
    else if (kind == L_DECONV) l->kshape = {4, 4, cout, cin};
    else l->kshape = {cin, cout};
    by_name[name] = l;
    var_names.push_back(name + "/kernel");
    var_names.push_back(name + "/bias");
    return l;
  }
  // convrelu2_caffe_padding (helpers.py:105-153): y conv into `mid`, x conv into `out`; returns the y conv
  Layer* add_sep(const std::string& name, int k, int stride, Buf* in, int in_coff, int cin, Buf* mid, int cmid, Buf* out,
                 int out_coff, int cout) {
    Layer* y = add_layer(name + "y", L_CONV, in, in_coff, cin, mid, 0, cmid, k, 1, stride, 1, true);
    add_layer(name + "x", L_CONV, mid, 0, cmid, out, out_coff, cout, 1, k, 1, stride, true);
    return y;
  }
  // v2 convrelu2 (v2/helpers.py:46-91): the same pair with 'same' padding; the x conv reads its input in whole chunks of 32
  // channels, so a 24 / 48-channel y half sits in a 32 / 64-channel pixel whose other channels are never written (zero)
  // and carry zero weights, which keeps the x conv on the tensor cores
  Layer* add_sep_v2(const std::string& name, int k, int stride, Buf* in, int in_coff, int cin, Buf* mid, int cmid, Buf* out,
                    int out_coff, int cout) {
    Layer* y = add_sep(name, k, stride, in, in_coff, cin, mid, cmid, out, out_coff, cout);
    Layer* x = layers.back().get();
    y->tf_same = x->tf_same = true;
    x->cin_buf = (cmid + 31) / 32 * 32;
    return y;
  }
  // a v2 single conv (v2/helpers.py:24-43)
  Layer* add_conv_v2(const std::string& name, Buf* in, int in_coff, int cin, Buf* out, int out_coff, int cout, int k, int stride,
                     bool leaky) {
    Layer* l = add_layer(name, L_CONV, in, in_coff, cin, out, out_coff, cout, k, k, stride, stride, leaky);
    l->tf_same = true;
    return l;
  }
};

namespace demon {
namespace {

// ---------------------------------------------------------------------------------------------
// plan construction
// ---------------------------------------------------------------------------------------------
// returns the index of the first layer after conv2
int build_trunk(demon_net* n, const std::string& s, bool flow, bool iterative) {
  const int conv2_out = (flow && !iterative) ? 64 : 32;
  // conv1 and conv2 of the iterative nets depend only on the image pair (blocks_original.py:141,147 / :331,333), so the
  // pipeline computes them once per call: they get a concat buffer of their own that survives the other blocks
  Buf* cat2 = iterative ? (flow ? n->cat2_f2 : n->cat2_d2) : n->cat2;
  n->add_sep(s + "conv1", 9, 2, n->img8, 0, 6, n->c1y, 32, n->c1, 0, 32);
  n->add_sep(s + "conv2", 7, 2, n->c1, 0, 32, n->c2y, conv2_out, cat2, 0, conv2_out);
  const int head_end = (int)n->layers.size();
  if (!(flow && !iterative)) {
    const int extra = flow ? 9 : (iterative ? 8 : 7);
    Layer* ey = n->add_sep(s + "conv2_extra_inputs", 3, 1, n->extra_in, 0, extra, n->exy, 32, cat2, 32, 32);
    // the 7 / 8 / 9 real channels sit in a 32-channel (128-byte) pixel whose other channels are zero and carry zero weights:
    // one K = 32 chunk of the tensor-core halo kernel (3 steps per tile) instead of the fp32 SIMT kernel
    ey->cin_buf = 32;
  }
  n->add_sep(s + "conv2_1", 3, 1, cat2, 0, 64, n->c21y, 64, n->concat2, 64, 64);
  n->add_sep(s + "conv3", 5, 2, n->concat2, 64, 64, n->c3y, 128, n->c3, 0, 128);
  n->add_sep(s + "conv3_1", 3, 1, n->c3, 0, 128, n->c31y, 128, n->concat3, 128, 128);
  n->add_sep(s + "conv4", 5, 2, n->concat3, 128, 128, n->c4y, 256, n->c4, 0, 256);
  n->add_sep(s + "conv4_1", 3, 1, n->c4, 0, 256, n->c41y, 256, n->concat4, 256, 256);
  n->add_sep(s + "conv5", flow ? 5 : 3, 2, n->concat4, 256, 256, n->c5y, 512, n->c5, 0, 512);
  n->add_sep(s + "conv5_1", 3, 1, n->c5, 0, 512, n->c51y, 512, n->c51, 0, 512);
  return head_end;
}

Block build_flow_block(demon_net* n, const std::string& scope, bool iterative) {
  const std::string s = scope + "/";
  const int begin = (int)n->layers.size();
  const int head_end = build_trunk(n, s, true, iterative);
  n->add_layer(s + "predict_flow5/conv1", L_CONV, n->c51, 0, 512, n->pf5a, 0, 24, 3, 3, 1, 1, true);
  n->add_layer(s + "predict_flow5/conv2", L_CONV, n->pf5a, 0, 24, n->pf5, 0, 4, 3, 3, 1, 1, false);
  // _upsample_prediction: no activation (blocks_original.py:70); lands in concat4[512:514]
  n->add_layer(s + "upsample_flow5to4/upconv", L_DECONV, n->pf5, 0, 4, n->concat4, 512, 2, 4, 4, 2, 2, false);
  n->add_layer(s + "refine4/upconv", L_DECONV, n->c51, 0, 512, n->concat4, 0, 256, 4, 4, 2, 2, true);
  Layer* r3 = n->add_layer(s + "refine3/upconv", L_DECONV, n->concat4, 0, 514, n->concat3, 0, 128, 4, 4, 2, 2, true);
  r3->cin_buf = 576;   // channels 514..575 of concat4 are never written (zero) and carry zero weights; 18 chunks (not 17) so that the K loop can be split
  n->add_layer(s + "refine2/upconv", L_DECONV, n->concat3, 0, 256, n->concat2, 0, 64, 4, 4, 2, 2, true);
  n->add_layer(s + "predict_flow2/conv1", L_CONV, n->concat2, 0, 128, n->p2a, 0, 24, 3, 3, 1, 1, true);
  n->add_layer(s + "predict_flow2/conv2", L_CONV, n->p2a, 0, 24, n->flowconf2, 0, 4, 3, 3, 1, 1, false);
  return {begin, head_end, (int)n->layers.size()};
}

Block build_dm_block(demon_net* n, const std::string& scope, bool iterative) {
  const std::string s = scope + "/";
  const int begin = (int)n->layers.size();
  const int head_end = build_trunk(n, s, false, iterative);
  n->add_layer(s + "motion_conv1", L_CONV, n->c51, 0, 512, n->mc1, 0, 128, 3, 3, 1, 1, true);
  Layer* f1 = n->add_layer(s + "motion_fc1", L_DENSE, n->mc1, 0, 6144, n->fc1, 0, 1024, 1, 1, 1, 1, true);
  f1->dense_nchw_flatten = true; f1->dense_c = 128; f1->dense_hw = 48;
  f1->ksplit = 24;   // 16 column tiles x 24 K slices = 384 CTAs instead of 16
  Layer* f2 = n->add_layer(s + "motion_fc2", L_DENSE, n->fc1, 0, 1024, n->fc2, 0, 128, 1, 1, 1, 1, true);
  f2->ksplit = 16;
  n->add_layer(s + "motion_fc3", L_DENSE, n->fc2, 0, 128, n->motion, 0, 7, 1, 1, 1, 1, false);
  n->add_layer(s + "refine4/upconv", L_DECONV, n->c51, 0, 512, n->concat4, 0, 256, 4, 4, 2, 2, true);
  n->add_layer(s + "refine3/upconv", L_DECONV, n->concat4, 0, 512, n->concat3, 0, 128, 4, 4, 2, 2, true);
  n->add_layer(s + "refine2/upconv", L_DECONV, n->concat3, 0, 256, n->concat2, 0, 64, 4, 4, 2, 2, true);
  n->add_layer(s + "predict_depthnormal2/conv1", L_CONV, n->concat2, 0, 128, n->p2a, 0, 24, 3, 3, 1, 1, true);
  Layer* dn = n->add_layer(s + "predict_depthnormal2/conv2", L_CONV, n->p2a, 0, 24, n->dn2, 0, 4, 3, 3, 1, 1, false);
  dn->scale = n->motion; dn->scale_coff = 6; dn->scale_stride = 8;   // depth = motion[:,6] (the scale) * channel 0
  return {begin, head_end, (int)n->layers.size()};
}

Block build_refine_block(demon_net* n, const std::string& scope) {
  const std::string s = scope + "/";
  const int begin = (int)n->layers.size();
  Layer* c0 = n->add_layer(s + "conv0", L_CONV, n->rin, 0, 4, n->concat0, 32, 32, 3, 3, 1, 1, true);
  c0->cin_buf = 8;
  n->add_layer(s + "conv1", L_CONV, n->concat0, 32, 32, n->rc1, 0, 64, 3, 3, 2, 2, true);
  n->add_layer(s + "conv1_1", L_CONV, n->rc1, 0, 64, n->concat1, 64, 64, 3, 3, 1, 1, true);
  n->add_layer(s + "conv2", L_CONV, n->concat1, 64, 64, n->rc2, 0, 128, 3, 3, 2, 2, true);
  n->add_layer(s + "conv2_1", L_CONV, n->rc2, 0, 128, n->rc21, 0, 128, 3, 3, 1, 1, true);
  n->add_layer(s + "refine1/upconv", L_DECONV, n->rc21, 0, 128, n->concat1, 0, 64, 4, 4, 2, 2, true);
  n->add_layer(s + "refine0/upconv", L_DECONV, n->concat1, 0, 128, n->concat0, 0, 32, 4, 4, 2, 2, true);
  n->add_layer(s + "predict_depth0/conv1", L_CONV, n->concat0, 0, 64, n->pd0a, 0, 16, 3, 3, 1, 1, true);
  n->add_layer(s + "predict_depth0/conv2", L_CONV, n->pd0a, 0, 16, n->rdepth0, 0, 1, 3, 3, 1, 1, false);
  return {begin, begin, (int)n->layers.size()};
}

void build_plan(demon_net* n) {
  const int H = 192, W = 256;
  n->img8 = n->add_buf(H, W, 8);
  n->i22_half = n->add_buf(3, 96, 128);  // NCHW [B,3,96,128] scratch of the first median pass
  n->i22 = n->add_buf(3, 48, 64);        // NCHW [B,3,48,64]
  n->c1y = n->add_buf(96, 256, 32);
  n->c1 = n->add_buf(96, 128, 32);
  n->c2y = n->add_buf(48, 128, 64);
  n->cat2 = n->add_buf(48, 64, 64);
  n->cat2_f2 = n->add_buf(48, 64, 64);
  n->cat2_d2 = n->add_buf(48, 64, 64);
  n->extra_in = n->add_buf(48, 64, 32);   // 12 channels written at most (flow_extra_kernel), the rest stays zero
  n->exy = n->add_buf(48, 64, 32);
  n->c21y = n->add_buf(48, 64, 64);
  n->concat2 = n->add_buf(48, 64, 128);
  n->c3y = n->add_buf(24, 64, 128);
  n->c3 = n->add_buf(24, 32, 128);
  n->c31y = n->add_buf(24, 32, 128);
  n->concat3 = n->add_buf(24, 32, 256);
  n->c4y = n->add_buf(12, 32, 256);
  n->c4 = n->add_buf(12, 16, 256);
  n->c41y = n->add_buf(12, 16, 256);
  n->concat4 = n->add_buf(12, 16, 576);   // 512 + 2 (upsampled flow) padded to 18 chunks of 32 channels for the tensor-core path (18 = 2 x 3 x 3: split-K)
  n->c5y = n->add_buf(6, 16, 512);
  n->c5 = n->add_buf(6, 8, 512);
  n->c51y = n->add_buf(6, 8, 512);
  n->c51 = n->add_buf(6, 8, 512);
  n->pf5a = n->add_buf(6, 8, 24);
  n->pf5 = n->add_buf(6, 8, 4);
  n->p2a = n->add_buf(48, 64, 24);
  n->flowconf2 = n->add_buf(48, 64, 4);
  n->dn2 = n->add_buf(48, 64, 4);
  n->mc1 = n->add_buf(6, 8, 128);
  n->fc1 = n->add_buf(1, 1, 1024);
  n->fc2 = n->add_buf(1, 1, 128);
  n->motion = n->add_buf(1, 1, 8);
  n->splitk = n->add_buf(1, 24, 1024);   // split-K partial sums [24][B][1024]
  const int RH = n->RH, RW = n->RW;
  n->rin = n->add_buf(RH, RW, 8);   // [image1(3), depth upsampled(1), 0, 0, 0, 0]: 8 channels for the tensor-core 8-channel mode
  n->concat0 = n->add_buf(RH, RW, 64);
  n->rc1 = n->add_buf(RH / 2, RW / 2, 64);
  n->concat1 = n->add_buf(RH / 2, RW / 2, 128);
  n->rc2 = n->add_buf(RH / 4, RW / 4, 128);
  n->rc21 = n->add_buf(RH / 4, RW / 4, 128);
  n->pd0a = n->add_buf(RH, RW, 16);
  n->rdepth0 = n->add_buf(RH, RW, 1);
  // The fused pipeline stages its inputs and the host entries' outputs in buffers that hold nothing live at the time:
  n->pair_bytes = n->concat0;    // the image pair as uint8 [B,2,192,256,3] (resized / adapted), or a host entry's image pair
  n->i22_bytes = n->pd0a;        // image2_2 as uint8 [B,48,64,3] (resized), or a host entry's image2_2
  n->planes2 = n->c1y;           // image 2 as NCHW fp32 planes, input of the median pair of a uint8 call without image2_2
  n->host_depth0 = n->rdepth0;   // a host entry's depth0 before its copy to the host
  n->host_motion = n->fc1;       // a host entry's rotation and translation ([B,3] each) before their copy to the host
  // The first three are consumed into img8 / i22 before the first block runs; then c1y is next written by conv1y, and
  // concat0 and pd0a only by the refinement block.  That block shares no buffer with the iteration state, so it may also
  // run between two iterations (snapshots): it writes rin, concat0, rc1, concat1, rc2, rc21, pd0a, rdepth0 (or the
  // caller's depth0) and the split-K scratch, which holds partial sums only inside one layer; the iterations carry dn2,
  // flowconf2, motion, i22, img8, cat2_f2, cat2_d2 and extra_in from one block to the next, and the refinement block only
  // reads img8 (image 1, whatever the input kind) and dn2.  rdepth0 is that block's own output, and fc1 is free after the
  // last DM block, which a host entry's one export follows.

  n->flow1 = build_flow_block(n, "netFlow1", false);
  n->dm1 = build_dm_block(n, "netDM1", false);
  n->flow2 = build_flow_block(n, "netFlow2", true);
  n->dm2 = build_dm_block(n, "netDM2", true);
  n->refine = build_refine_block(n, "netRefine");
}

// ---- v2 (python/depthmotionnet/v2/blocks.py): the same kernels over a second plan ----------------------------------------
// returns the index of the first layer after conv2 (as build_trunk)
int build_trunk_v2(demon_net* n, const std::string& s, bool flow, bool iterative) {
  const bool wide2 = flow && !iterative;   // the bootstrap flow block's conv2 is (48, 64) and has no extra inputs
  Buf* cat2 = iterative ? (flow ? n->cat2_f2 : n->cat2_d2) : n->cat2;
  n->add_sep_v2(s + "conv1", 9, 2, n->img8, 0, 6, n->c1y, 24, n->c1, 0, 32);
  n->add_sep_v2(s + "conv2", 7, 2, n->c1, 0, 32, n->c2y, wide2 ? 48 : 32, cat2, 0, wide2 ? 64 : 32);
  const int head_end = (int)n->layers.size();
  if (!wide2) {
    const int extra = flow ? 9 : (iterative ? 8 : 7);
    Layer* ey = n->add_sep_v2(s + "conv2_extra_inputs", 3, 1, n->extra_in, 0, extra, n->exy, 32, cat2, 32, 32);
    ey->cin_buf = 32;   // as in build_trunk
  }
  n->add_sep_v2(s + "conv2_1", 3, 1, cat2, 0, 64, n->c21y, 64, n->concat2, 64, 64);
  n->add_sep_v2(s + "conv3", 5, 2, n->concat2, 64, 64, n->c3y, 96, n->c3, 0, 128);
  n->add_sep_v2(s + "conv3_1", 3, 1, n->c3, 0, 128, n->c31y, 128, n->concat3, 128, 128);
  n->add_sep_v2(s + "conv4", 5, 2, n->concat3, 128, 128, n->c4y, 192, n->c4, 0, 256);
  n->add_sep_v2(s + "conv4_1", 3, 1, n->c4, 0, 256, n->c41y, 256, n->concat4, 256, 256);
  n->add_sep_v2(s + "conv5", flow ? 5 : 3, 2, n->concat4, 256, 256, n->c5y, 384, n->c5, 0, 384);
  n->add_sep_v2(s + "conv5_1", 3, 1, n->c5, 0, 384, n->c51y, 384, n->c51, 0, 384);
  // dense5 over conv5_1[:, 0:96] flattened NCHW, reshaped [96,6,8] and concatenated after conv5_1: channels 384..479 of
  // c51 (conv5_1_dense5)
  Layer* d5 = n->add_layer(s + "dense5", L_DENSE, n->d5in, 0, 4608, n->d5out, 0, 4608, 1, 1, 1, 1, true);
  d5->dense_nchw_flatten = d5->dense_nchw_unflatten = true; d5->dense_c = 96; d5->dense_hw = 48;
  d5->nhwc = n->c51; d5->nhwc_out_coff = 384;
  // 72 column tiles x 16 K slices of 288 rows: at batch 1 the layer is a read of its 85 MB weight, and 1152 CTAs keep enough
  // loads in flight for it (4 slices, 288 CTAs, reached a fifth of HBM bandwidth); build_plan_v2 sizes the split-K buffer
  d5->ksplit = 16;
  return head_end;
}

Block build_flow_block_v2(demon_net* n, const std::string& scope, bool iterative) {
  const std::string s = scope + "/";
  const int begin = (int)n->layers.size();
  const int head_end = build_trunk_v2(n, s, true, iterative);
  n->add_conv_v2(s + "predict_flow5/conv1", n->c51, 0, 480, n->pf5a, 0, 24, 3, 1, true);
  n->add_conv_v2(s + "predict_flow5/conv2", n->pf5a, 0, 24, n->pf5, 0, 4, 3, 1, false);
  n->add_layer(s + "upsample_flow5to4/upconv", L_DECONV, n->pf5, 0, 4, n->concat4, 512, 2, 4, 4, 2, 2, false);
  n->add_layer(s + "refine4/upconv", L_DECONV, n->c51, 0, 480, n->concat4, 0, 256, 4, 4, 2, 2, true);
  Layer* r3 = n->add_layer(s + "refine3/upconv", L_DECONV, n->concat4, 0, 514, n->concat3, 0, 128, 4, 4, 2, 2, true);
  r3->cin_buf = 576;   // as in build_flow_block
  n->add_layer(s + "refine2/upconv", L_DECONV, n->concat3, 0, 256, n->concat2, 0, 64, 4, 4, 2, 2, true);
  n->add_conv_v2(s + "predict_flow2/conv1", n->concat2, 0, 128, n->p2a, 0, 24, 3, 1, true);
  n->add_conv_v2(s + "predict_flow2/conv2", n->p2a, 0, 24, n->flowconf2, 0, 4, 3, 1, false);
  return {begin, head_end, (int)n->layers.size()};
}

Block build_dm_block_v2(demon_net* n, const std::string& scope, bool iterative) {
  const std::string s = scope + "/";
  const int begin = (int)n->layers.size();
  const int head_end = build_trunk_v2(n, s, false, iterative);
  // motion branch (v2/blocks.py:417-429): three separable stride-2 pairs on conv2_1 and a 3x3 conv on conv5_1_dense5, each
  // into one half of the 128-channel concat that motion_fc1 flattens NCHW
  n->add_sep_v2(s + "motion_conv3", 5, 2, n->concat2, 64, 64, n->mc3y, 64, n->mc3, 0, 64);
  n->add_sep_v2(s + "motion_conv4", 5, 2, n->mc3, 0, 64, n->mc4y, 64, n->mc4, 0, 64);
  n->add_sep_v2(s + "motion_conv5a", 3, 2, n->mc4, 0, 64, n->mc5y, 64, n->mc1, 0, 64);
  n->add_conv_v2(s + "motion_conv5b", n->c51, 0, 480, n->mc1, 64, 64, 3, 1, true);
  Layer* f1 = n->add_layer(s + "motion_fc1", L_DENSE, n->mc1, 0, 6144, n->fc1, 0, 1024, 1, 1, 1, 1, true);
  f1->dense_nchw_flatten = true; f1->dense_c = 128; f1->dense_hw = 48;
  f1->ksplit = 24;
  Layer* f2 = n->add_layer(s + "motion_fc2", L_DENSE, n->fc1, 0, 1024, n->fc2, 0, 128, 1, 1, 1, 1, true);
  f2->ksplit = 16;
  n->add_layer(s + "motion_fc3", L_DENSE, n->fc2, 0, 128, n->motion, 0, 7, 1, 1, 1, 1, false);
  n->add_layer(s + "refine4/upconv", L_DECONV, n->c51, 0, 384, n->concat4, 0, 256, 4, 4, 2, 2, true);   // conv5_1 alone
  n->add_layer(s + "refine3/upconv", L_DECONV, n->concat4, 0, 512, n->concat3, 0, 128, 4, 4, 2, 2, true);
  n->add_layer(s + "refine2/upconv", L_DECONV, n->concat3, 0, 256, n->concat2, 0, 64, 4, 4, 2, 2, true);
  n->add_conv_v2(s + "predict_depthnormal2/conv1", n->concat2, 0, 128, n->p2a, 0, 24, 3, 1, true);
  Layer* dn = n->add_conv_v2(s + "predict_depthnormal2/conv2", n->p2a, 0, 24, n->dn2, 0, 4, 3, 1, false);
  dn->scale = n->motion; dn->scale_coff = 6; dn->scale_stride = 8;
  return {begin, head_end, (int)n->layers.size()};
}

// v2/blocks.py:499-560: as build_refine_block, with 'same' padding and depth0 + normal0 out of predict_depth0/conv2
Block build_refine_block_v2(demon_net* n, const std::string& scope) {
  const std::string s = scope + "/";
  const int begin = (int)n->layers.size();
  Layer* c0 = n->add_conv_v2(s + "conv0", n->rin, 0, 4, n->concat0, 32, 32, 3, 1, true);
  c0->cin_buf = 8;
  n->add_conv_v2(s + "conv1", n->concat0, 32, 32, n->rc1, 0, 64, 3, 2, true);
  n->add_conv_v2(s + "conv1_1", n->rc1, 0, 64, n->concat1, 64, 64, 3, 1, true);
  n->add_conv_v2(s + "conv2", n->concat1, 64, 64, n->rc2, 0, 128, 3, 2, true);
  n->add_conv_v2(s + "conv2_1", n->rc2, 0, 128, n->rc21, 0, 128, 3, 1, true);
  n->add_layer(s + "refine1/upconv", L_DECONV, n->rc21, 0, 128, n->concat1, 0, 64, 4, 4, 2, 2, true);
  n->add_layer(s + "refine0/upconv", L_DECONV, n->concat1, 0, 128, n->concat0, 0, 32, 4, 4, 2, 2, true);
  n->add_conv_v2(s + "predict_depth0/conv1", n->concat0, 0, 64, n->pd0a, 0, 16, 3, 1, true);
  n->add_conv_v2(s + "predict_depth0/conv2", n->pd0a, 0, 16, n->rdepth0, 0, 4, 3, 1, false);
  return {begin, begin, (int)n->layers.size()};
}

void build_plan_v2(demon_net* n) {
  const int H = 192, W = 256;
  n->img8 = n->add_buf(H, W, 8);
  n->i22_half = n->add_buf(3, 96, 128);
  n->i22 = n->add_buf(3, 48, 64);
  n->c1y = n->add_buf(96, 256, 32);      // 24 channels written
  n->c1 = n->add_buf(96, 128, 32);
  n->c2y = n->add_buf(48, 128, 64);      // 48 (bootstrap flow block) or 32 channels written
  n->cat2 = n->add_buf(48, 64, 64);
  n->cat2_f2 = n->add_buf(48, 64, 64);
  n->cat2_d2 = n->add_buf(48, 64, 64);
  n->extra_in = n->add_buf(48, 64, 32);
  n->exy = n->add_buf(48, 64, 32);
  n->c21y = n->add_buf(48, 64, 64);
  n->concat2 = n->add_buf(48, 64, 128);
  n->c3y = n->add_buf(24, 64, 96);
  n->c3 = n->add_buf(24, 32, 128);
  n->c31y = n->add_buf(24, 32, 128);
  n->concat3 = n->add_buf(24, 32, 256);
  n->c4y = n->add_buf(12, 32, 192);
  n->c4 = n->add_buf(12, 16, 256);
  n->c41y = n->add_buf(12, 16, 256);
  n->concat4 = n->add_buf(12, 16, 576);
  n->c5y = n->add_buf(6, 16, 384);
  n->c5 = n->add_buf(6, 8, 384);
  n->c51y = n->add_buf(6, 8, 384);
  n->c51 = n->add_buf(6, 8, 480);        // conv5_1_dense5: conv5_1 (384) ++ dense5 reshaped (96)
  n->d5in = n->add_buf(1, 1, 4608);
  n->d5out = n->add_buf(1, 1, 4608);
  n->pf5a = n->add_buf(6, 8, 24);
  n->pf5 = n->add_buf(6, 8, 4);
  n->p2a = n->add_buf(48, 64, 24);
  n->flowconf2 = n->add_buf(48, 64, 4);
  n->dn2 = n->add_buf(48, 64, 4);
  n->mc3y = n->add_buf(24, 64, 64);
  n->mc3 = n->add_buf(24, 32, 64);
  n->mc4y = n->add_buf(12, 32, 64);
  n->mc4 = n->add_buf(12, 16, 64);
  n->mc5y = n->add_buf(6, 16, 64);
  n->mc1 = n->add_buf(6, 8, 128);        // motion_conv5a ++ motion_conv5b
  n->fc1 = n->add_buf(1, 1, 1024);
  n->fc2 = n->add_buf(1, 1, 128);
  n->motion = n->add_buf(1, 1, 8);
  n->splitk = n->add_buf(1, 16, 4608);   // split-K partial sums: dense5 [16][B][4608], motion_fc1 [24][B][1024]
  const int RH = n->RH, RW = n->RW;
  n->rin = n->add_buf(RH, RW, 8);
  n->concat0 = n->add_buf(RH, RW, 64);
  n->rc1 = n->add_buf(RH / 2, RW / 2, 64);
  n->concat1 = n->add_buf(RH / 2, RW / 2, 128);
  n->rc2 = n->add_buf(RH / 4, RW / 4, 128);
  n->rc21 = n->add_buf(RH / 4, RW / 4, 128);
  n->pd0a = n->add_buf(RH, RW, 16);
  n->rdepth0 = n->add_buf(RH, RW, 4);    // depth0 ++ normal0
  // Staging roles as in build_plan, for the same reasons: pair_bytes, i22_bytes and planes2 are consumed into img8 / i22
  // before the first block, c1y is next written by conv1y, concat0 and pd0a only by the refinement block, which reads img8
  // and dn2 alone; fc1 is free after the last DM block.  Unlike v1's, rdepth0 is not free for a host entry's depth0: it
  // holds depth0 ++ normal0 (predict_depth0/conv2), which export_outputs reads.  The host outputs are exported after the
  // refinement block's last layer instead, into buffers whose last reader that block has already run: pd0a (read by
  // predict_depth0/conv2) takes depth0 and concat0 (read by predict_depth0/conv1) takes normal0.  A host entry takes no
  // snapshots, so the block runs once, and nothing runs after the export but the copies to the host.
  n->pair_bytes = n->concat0;    // the image pair as uint8 [B,2,192,256,3] (resized / adapted), or a host entry's image pair
  n->i22_bytes = n->pd0a;        // image2_2 as uint8 [B,48,64,3] (resized), or a host entry's image2_2
  n->planes2 = n->c1y;           // image 2 as NCHW fp32 planes, input of the median or area downsampling of a uint8 call
  n->host_depth0 = n->pd0a;      // a host entry's depth0 [B,1,192,256] before its copy to the host
  n->host_normal0 = n->concat0;  // a host entry's normal0 [B,3,192,256] before its copy to the host
  n->host_motion = n->fc1;       // a host entry's rotation and translation ([B,3] each) before their copy to the host

  n->flow1 = build_flow_block_v2(n, "netFlow1", false);
  n->dm1 = build_dm_block_v2(n, "netDM1", false);
  n->flow2 = build_flow_block_v2(n, "netFlow2", true);
  n->dm2 = build_dm_block_v2(n, "netDM2", true);
  n->refine = build_refine_block_v2(n, "netRefine");
}

// ---------------------------------------------------------------------------------------------
// weight packing: TF layout -> [tap][cin_buf][cout_pad]
// ---------------------------------------------------------------------------------------------
// transposed conv k4 s2, "VALID then slice 1" == "same" (blocks_original.py:64-74,97-110):
//   out[2y+py, 2x+px] = sum over the two kernel rows/cols of matching parity
//   py = 0: (ky=1, dy=0), (ky=3, dy=-1);   py = 1: (ky=0, dy=+1), (ky=2, dy=0)
const int kDeconvK[2][2] = {{1, 3}, {0, 2}};
const int kDeconvD[2][2] = {{0, -1}, {1, 0}};

void pack_conv(const Layer& l, const float* k, std::vector<float>& out) {
  const int taps = l.kh * l.kw;
  out.assign((size_t)taps * l.cin_buf * l.cout_pad, 0.f);
  for (int t = 0; t < taps; ++t)
    for (int ci = 0; ci < l.cin; ++ci)
      for (int co = 0; co < l.cout; ++co)
        out[((size_t)t * l.cin_buf + ci) * l.cout_pad + co] = k[((size_t)t * l.cin + ci) * l.cout + co];
}

void pack_deconv_class(const Layer& l, const float* k, int py, int px, std::vector<float>& out) {
  out.assign((size_t)4 * l.cin_buf * l.cout_pad, 0.f);
  for (int a = 0; a < 2; ++a)
    for (int b = 0; b < 2; ++b) {
      const int ky = kDeconvK[py][a], kx = kDeconvK[px][b];
      const int t = a * 2 + b;
      for (int ci = 0; ci < l.cin; ++ci)
        for (int co = 0; co < l.cout; ++co)
          out[((size_t)t * l.cin_buf + ci) * l.cout_pad + co] = k[(((size_t)ky * 4 + kx) * l.cout + co) * l.cin + ci];
    }
}

// dense5 (v2): buffer column j = hw*C + c holds TF column c*HW + hw (TF reshapes the output to NCHW [C, H, W])
int dense_unflatten_src(const Layer& l, int j) { return (j % l.dense_c) * l.dense_hw + j / l.dense_c; }

void pack_dense(const Layer& l, const float* k, std::vector<float>& out) {
  out.assign((size_t)l.cin_buf * l.cout_pad, 0.f);
  for (int i = 0; i < l.cin; ++i) {
    int src = i;
    if (l.dense_nchw_flatten) {  // buffer index i = hw*C + c  <->  TF row c*HW + hw
      const int hw = i / l.dense_c, c = i % l.dense_c;
      src = c * l.dense_hw + hw;
    }
    if (!l.dense_nchw_unflatten) {
      for (int co = 0; co < l.cout; ++co) out[(size_t)i * l.cout_pad + co] = k[(size_t)src * l.cout + co];
      continue;
    }
    for (int co = 0; co < l.cout; ++co) out[(size_t)i * l.cout_pad + co] = k[(size_t)src * l.cout + dense_unflatten_src(l, co)];
  }
}

int upload(std::vector<void*>& allocs, const std::vector<float>& host, float** dev) {
  void* p = nullptr;
  DEMON_CHECK_CUDA(cudaMalloc(&p, host.size() * sizeof(float) + 256));
  allocs.push_back(p);
  DEMON_CHECK_CUDA(cudaMemcpy(p, host.data(), host.size() * sizeof(float), cudaMemcpyHostToDevice));
  *dev = (float*)p;
  return DEMON_OK;
}

// ---------------------------------------------------------------------------------------------
// layer execution
// ---------------------------------------------------------------------------------------------
// tf.nn.conv2d(padding='SAME') along one axis: out = ceil(in / s), pad_total = max((out - 1) * s + k - in, 0), and the
// smaller half goes before.  Equal to k / 2 (caffe padding) for s = 1 and odd k, and for s = 2 on an odd input; one less
// for s = 2 on an even input.
int tf_same_pad_before(int in, int k, int s) {
  const int out = ceil_div(in, s);
  return std::max((out - 1) * s + k - in, 0) / 2;
}

// The convolution problem(s) of a layer: 1 for conv / dense, 4 sub-pixel classes for a transposed conv.
// `dst`, if given, replaces the base of the layer's output buffer (same shape and channel pitch).
int build_problems(const Layer& l, int B, ConvProblem* out, float* dst = nullptr) {
  ConvProblem p;
  memset(&p, 0, sizeof(p));
  p.in = l.in->p + l.in_coff;
  p.in_pitch = l.in->C;
  p.B = B;
  p.Cin = l.cin_buf;
  p.out = (dst ? dst : l.out->p) + l.out_coff;
  p.out_pitch = l.out->C;
  p.Cout = l.cout;
  p.Cout_pad = l.cout_pad;
  p.bias = l.bias_dev;
  p.leaky = l.leaky ? 1 : 0;
  p.scale = l.scale ? l.scale->p + l.scale_coff : nullptr;
  p.scale_stride = l.scale_stride;
  p.osy = p.osx = 1;
  if (l.kind == L_DENSE) {
    p.Hi = p.Wi = p.Ho = p.Wo = p.Hfull = p.Wfull = 1;
    p.in_pitch = l.cin_buf;
    p.sy = p.sx = 1;
    p.ntaps = 1;
    p.w = l.w_dev[0];
    out[0] = p;
    return 1;
  }
  p.Hi = l.in->H; p.Wi = l.in->W;
  if (l.kind == L_CONV) {
    p.sy = l.sy; p.sx = l.sx;
    p.Ho = ceil_div(p.Hi, l.sy); p.Wo = ceil_div(p.Wi, l.sx);
    p.Hfull = p.Ho; p.Wfull = p.Wo;
    p.ntaps = l.kh * l.kw;
    const int py = l.tf_same ? tf_same_pad_before(p.Hi, l.kh, l.sy) : l.kh / 2;
    const int px = l.tf_same ? tf_same_pad_before(p.Wi, l.kw, l.sx) : l.kw / 2;
    for (int ky = 0; ky < l.kh; ++ky)
      for (int kx = 0; kx < l.kw; ++kx) { p.dy[ky * l.kw + kx] = ky - py; p.dx[ky * l.kw + kx] = kx - px; }
    p.w = l.w_dev[0];
    out[0] = p;
    return 1;
  }
  // transposed conv: four sub-pixel 2x2 convolutions
  p.sy = p.sx = 1;
  p.Ho = p.Hi; p.Wo = p.Wi;
  p.Hfull = 2 * p.Hi; p.Wfull = 2 * p.Wi;
  p.osy = p.osx = 2;
  p.ntaps = 4;
  for (int py = 0; py < 2; ++py)
    for (int px = 0; px < 2; ++px) {
      p.ooy = py; p.oox = px;
      for (int a = 0; a < 2; ++a)
        for (int b = 0; b < 2; ++b) { p.dy[a * 2 + b] = kDeconvD[py][a]; p.dx[a * 2 + b] = kDeconvD[px][b]; }
      p.w = l.w_dev[py * 2 + px];
      out[py * 2 + px] = p;
    }
  return 4;
}

int run_layer(const Layer& l, int B, cudaStream_t stream, float* splitk_ws, float* tc_ws, float* dst = nullptr) {
  ConvProblem probs[4];
  const int nclass = build_problems(l, B, probs, dst);
  if (l.use_tc()) {
    probs[0].partial = tc_ws;   // scratch of the split-K tensor-core layers (the net's, so two nets in flight do not share it)
    return conv_tc_launch(l.tc, probs, stream);
  }
  for (int c = 0; c < nclass; ++c) {
    if (l.kind == L_DENSE && l.ksplit > 1 && splitk_ws) { probs[c].partial = splitk_ws; probs[c].ksplit = l.ksplit; }
    int rc = conv_simt_launch(probs[c], stream);
    if (rc != DEMON_OK) return rc;
  }
  return DEMON_OK;
}

// Uploads a layer's bias and its kernel (TF layout) packed for the path that runs it: at a tensor-core precision the planner
// (tc_prepare) may take a conv / transposed conv and pack the kernel for the tensor cores; any other layer gets the SIMT
// packing [tap][cin_buf][cout_pad].  Device allocations other than the plan's (tc_layer_free) are appended to `allocs`.
int upload_layer(Layer& l, const float* k, const float* bias_host, int B, int precision, std::vector<void*>& allocs) {
  std::vector<float> bias(l.cout_pad, 0.f);
  std::copy(bias_host, bias_host + l.cout, bias.begin());
  if (l.dense_nchw_unflatten)
    for (int j = 0; j < l.cout; ++j) bias[j] = bias_host[dense_unflatten_src(l, j)];
  int rc;
  if ((rc = upload(allocs, bias, &l.bias_dev))) return rc;
  std::vector<float> w[4];
  const float* w_hosts[4] = {nullptr, nullptr, nullptr, nullptr};
  const int nw = (l.kind == L_DECONV) ? 4 : 1;
  for (int c = 0; c < nw; ++c) {
    if (l.kind == L_CONV) pack_conv(l, k, w[c]);
    else if (l.kind == L_DENSE) pack_dense(l, k, w[c]);
    else pack_deconv_class(l, k, c / 2, c % 2, w[c]);
    w_hosts[c] = w[c].data();
  }
  if (precision != DEMON_PREC_FP32_SIMT && l.kind != L_DENSE) {
    ConvProblem probs[4];
    const int nclass = build_problems(l, B, probs);
    rc = tc_prepare(l.tc, probs, w_hosts, nclass, precision);
    if (rc == kTcWeightRange)
      return fail(DEMON_E_INVALID, "variable %s/kernel: a value is not finite or above 65504 in magnitude, which FP16 cannot hold",
                  l.name.c_str());
    if (rc != kTcNoPlan) return rc;   // on the tensor cores, or an error
  }
  for (int c = 0; c < nw; ++c)
    if ((rc = upload(allocs, w[c], &l.w_dev[c]))) return rc;
  return DEMON_OK;
}

// The plan line of a layer: the tensor-core planner's, or "simt" for a layer it does not take.
int describe_layer(const Layer& l, int B, int precision, char* buf, int buflen) {
  if (l.kind == L_DENSE) return snprintf(buf, buflen, "dense simt ksplit %d", l.ksplit);
  ConvProblem probs[4];
  const int nclass = build_problems(l, B, probs);
  const int len = (precision != DEMON_PREC_FP32_SIMT) ? tc_describe(probs, nclass, precision, buf, buflen) : 0;
  return (len > 0) ? len : snprintf(buf, buflen, "simt");
}

// A layer outside any net (the standalone entries): a convolution, or with `deconv` a k4 s2 transposed convolution, of
// an NHWC [B,H,W,in_pitch] input into an NHWC output of channel pitch out_pitch.
struct StandaloneLayer {
  Buf in, out;
  Layer layer;
  StandaloneLayer(const float* in_p, float* out_p, int H, int W, int Cin, int in_pitch, int Cout, int out_pitch, int kh, int kw, int sy,
                  int sx, bool deconv, bool leaky) {
    in.p = const_cast<float*>(in_p); in.H = H; in.W = W; in.C = in_pitch;
    out.p = out_p; out.C = out_pitch;
    if (deconv) { out.H = 2 * H; out.W = 2 * W; } else { out.H = ceil_div(H, sy); out.W = ceil_div(W, sx); }
    Layer& l = layer;
    l.name = "standalone"; l.kind = deconv ? L_DECONV : L_CONV; l.in = &in; l.cin = Cin; l.cin_buf = (Cin + 3) / 4 * 4; l.out = &out;
    l.cout = Cout; l.cout_pad = (Cout + 3) / 4 * 4; l.kh = kh; l.kw = kw; l.sy = sy; l.sx = sx; l.leaky = leaky;
  }
  StandaloneLayer(const StandaloneLayer&) = delete;             // `layer` points at `in` and `out`
  StandaloneLayer& operator=(const StandaloneLayer&) = delete;
};

// `dst`: see build_problems
int run_layer_timed(demon_net* n, int idx, cudaStream_t stream, float* dst) {
  const Layer& l = *n->layers[idx];
  static const bool sync_layers = getenv("DEMON_SYNC_LAYERS") && atoi(getenv("DEMON_SYNC_LAYERS")) != 0;   // debugging aid
  if (sync_layers) {
    int rc = run_layer(l, n->B, stream, n->splitk->p, n->tc_scratch, dst);
    cudaError_t e = cudaStreamSynchronize(stream);
    if (rc == DEMON_OK && e != cudaSuccess) return fail(DEMON_E_CUDA, "layer %s: %s", l.name.c_str(), cudaGetErrorString(e));
    return rc;
  }
  if (!n->profiling) return run_layer(l, n->B, stream, n->splitk->p, n->tc_scratch, dst);
  if (n->prof_used + 2 > n->prof_events.size()) {
    const size_t old = n->prof_events.size();
    n->prof_events.resize(old + 1024);
    for (size_t i = old; i < n->prof_events.size(); ++i) DEMON_CHECK_CUDA(cudaEventCreate(&n->prof_events[i]));
  }
  DEMON_CHECK_CUDA(cudaEventRecord(n->prof_events[n->prof_used], stream));
  int rc = run_layer(l, n->B, stream, n->splitk->p, n->tc_scratch, dst);
  DEMON_CHECK_CUDA(cudaEventRecord(n->prof_events[n->prof_used + 1], stream));
  n->prof_layer.push_back(idx);
  n->prof_used += 2;
  return rc;
}

// A dense copy of layer l's input slice (cin_buf channels) or output slice (cout channels) to `to`: float32 [B,H,W,C], or
// [B,C] for a dense layer, which reads rows of cin_buf floats (build_problems) and writes one pixel per image.
int trace_copy(const demon_net* n, const Layer& l, bool input, float* dst, float* to, cudaStream_t stream) {
  const Buf* b = input ? l.in : l.out;
  const float* src = input ? l.in->p + l.in_coff : (dst ? dst : l.out->p) + l.out_coff;
  const size_t width = (input ? l.cin_buf : l.cout) * sizeof(float);
  const size_t pitch = (input && l.kind == L_DENSE ? l.cin_buf : b->C) * sizeof(float);
  const size_t rows = (size_t)n->B * (l.kind == L_DENSE ? 1 : b->H * b->W);
  DEMON_CHECK_CUDA(cudaMemcpy2DAsync(to, width, src, pitch, width, rows, cudaMemcpyDeviceToDevice, stream));
  return DEMON_OK;
}

int dense_nhwc_copy(const demon_net* n, const Layer& l, bool gather, cudaStream_t s);

// `dst`: see build_problems.  With a trace set (demon_debug_trace_layers), the layer's input slice is copied out before it
// runs and its output slice after.
int run_layer_traced(demon_net* n, int idx, cudaStream_t stream, float* dst) {
  if (!n->tracing) return run_layer_timed(n, idx, stream, dst);
  const Layer& l = *n->layers[idx];
  int rc = n->trace_in[idx] ? trace_copy(n, l, true, dst, n->trace_in[idx], stream) : DEMON_OK;
  if (rc == DEMON_OK) rc = run_layer_timed(n, idx, stream, dst);
  if (rc == DEMON_OK && n->trace_out[idx]) rc = trace_copy(n, l, false, dst, n->trace_out[idx], stream);
  return rc;
}

// A dense layer over pixels (v2's dense5) gathers its input row before it runs and scatters its output after
int run_layer_profiled(demon_net* n, int idx, cudaStream_t stream, float* dst = nullptr) {
  const Layer& l = *n->layers[idx];
  if (!l.nhwc) return run_layer_traced(n, idx, stream, dst);
  int rc = dense_nhwc_copy(n, l, true, stream);
  if (rc == DEMON_OK) rc = run_layer_traced(n, idx, stream, dst);
  if (rc == DEMON_OK) rc = dense_nhwc_copy(n, l, false, stream);
  return rc;
}

// layers [begin, end) in order
int run_layers(demon_net* n, int begin, int end, cudaStream_t stream) {
  for (int i = begin; i < end; ++i) {
    int rc = run_layer_profiled(n, i, stream);
    if (rc != DEMON_OK) return rc;
  }
  return DEMON_OK;
}

// ---------------------------------------------------------------------------------------------
// glue kernels
// ---------------------------------------------------------------------------------------------
// strided element copy: dst[n*dn + p*dp + c*dc] = src[n*sn + p*sp + c*sc], c fastest
__global__ void __launch_bounds__(256) strided_copy_kernel(const float* __restrict__ src, float* __restrict__ dst, int N, int P, int C,
                                                          long sn, long sp, long sc, long dn, long dp, long dc) {
  pdl_launch_dependents();   // common.cuh: programmatic dependent launch
  pdl_wait();
  const long total = (long)N * P * C;
  for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long)gridDim.x * 256) {
    const int c = (int)(i % C);
    const long r = i / C;
    const int p = (int)(r % P);
    const int n = (int)(r / P);
    dst[n * dn + p * dp + c * dc] = __ldg(src + n * sn + p * sp + c * sc);
  }
}

// strides in floats between samples, pixels and channels
struct Strides { long n, p, c; };

// an API tensor of C channels over P pixels: [B,C,H,W] (data_format 0) or [B,H,W,C] (data_format 1)
Strides api_strides(int data_format, long P, int C) {
  return data_format == 0 ? Strides{C * P, 1, P} : Strides{C * P, C, 1};
}

// a workspace buffer (NHWC)
Strides buf_strides(const Buf* b) { return Strides{(long)b->H * b->W * b->C, b->C, 1}; }

int strided_copy(const float* src, float* dst, int N, int P, int C, Strides s, Strides d, cudaStream_t stream) {
  const long total = (long)N * P * C;
  if (total == 0) return DEMON_OK;
  long blocks = (total + 255) / 256;
  if (blocks > 132 * 32) blocks = 132 * 32;
  (void)launch_pdl(strided_copy_kernel, dim3((int)blocks), dim3(256), 0, stream, src, dst, N, P, C, s.n, s.p, s.c, d.n, d.p, d.c);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

// dense5's two copies (Layer::nhwc): gather channels [0, dense_c) of every pixel into the row [B, HW*C] the dense kernel
// reads, or scatter its output row into channels [nhwc_out_coff, +dense_c).  Two small copies of B x 18 KB rather than a
// pixel pitch inside the dense kernel and its split-K reduction, which v1's layers share.
int dense_nhwc_copy(const demon_net* n, const Layer& l, bool gather, cudaStream_t s) {
  const Buf* b = l.nhwc;
  const Strides row{(long)l.dense_hw * l.dense_c, l.dense_c, 1};
  if (gather) return strided_copy(b->p, l.in->p, n->B, l.dense_hw, l.dense_c, buf_strides(b), row, s);
  return strided_copy(l.out->p, b->p + l.nhwc_out_coff, n->B, l.dense_hw, l.dense_c, row, buf_strides(b), s);
}

// median3x3_downsample over planes with a batch stride (image_pair[:,3:6] -> image2_2,
// examples/evaluation.py:170-173)
__global__ void __launch_bounds__(128) median_planes_kernel(const float* __restrict__ in, float* __restrict__ out, int C, int H, int W,
                                                           int Ho, int Wo, long in_sn, long out_sn) {
  pdl_launch_dependents();   // common.cuh: programmatic dependent launch
  pdl_wait();
  const int xo = blockIdx.x * 128 + threadIdx.x;
  const int yo = blockIdx.y;
  const int n = blockIdx.z / C, c = blockIdx.z % C;
  if (xo >= Wo) return;
  const float* p = in + n * in_sn + (long)c * H * W;
  float v[9];
  int idx = 0;
#pragma unroll
  for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
    for (int dx = -1; dx <= 1; ++dx) v[idx++] = __ldg(p + (size_t)clampi(2 * yo + dy, H) * W + clampi(2 * xo + dx, W));
  out[n * out_sn + (long)c * Ho * Wo + (size_t)yo * Wo + xo] = median9_reference_order(v);
}

// tf.image.resize_area (align_corners=False) by integer factors fy = H / Ho, fx = W / Wo, over NCHW planes with a batch stride
// (training/v2/training.py:179 makes image2_2 with it).  Every weight of TF's area kernel is 1 for an integer factor, and
// this project defines the result, in float32, as: each source row's fx pixels summed left to right from +0, the fy row sums
// summed top to bottom from +0, times `scale` = float32(1 / (fy fx)) (DESIGN.md §3.6).  Rounded adds and one rounded
// multiply, so no contraction can change the bits.  One output per thread; grid-stride over N*C*Ho*Wo.
__global__ void __launch_bounds__(256) area_planes_kernel(const float* __restrict__ in, float* __restrict__ out, int N, int C, int H, int W,
                                                         int Ho, int Wo, long in_sn, float scale) {
  pdl_launch_dependents();   // common.cuh: programmatic dependent launch
  pdl_wait();
  const int fy = H / Ho, fx = W / Wo;
  const long total = (long)N * C * Ho * Wo;
  for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long)gridDim.x * 256) {
    const int xo = (int)(i % Wo);
    long r = i / Wo;
    const int yo = (int)(r % Ho);
    r /= Ho;
    const int c = (int)(r % C);
    const long n = r / C;
    const float* p = in + n * in_sn + ((long)c * H + (long)yo * fy) * W + (long)xo * fx;
    float sum = 0.f;
    for (int y = 0; y < fy; ++y) {
      float row = 0.f;
      for (int x = 0; x < fx; ++x) row = fadd(row, __ldg(p + (long)y * W + x));
      sum = fadd(sum, row);
    }
    out[i] = fmul(sum, scale);
  }
}

// Argument checks of area_launch
int area_check(int N, int C, int H, int W, int Ho, int Wo, long in_sn, const char* who) {
  DEMON_REQUIRE(N >= 0 && C >= 0 && H >= 1 && W >= 1 && Ho >= 1 && Wo >= 1, "%s: size %dx%dx%dx%d -> %dx%d", who, N, C, H, W, Ho, Wo);
  DEMON_REQUIRE(H % Ho == 0 && W % Wo == 0, "%s: %dx%d -> %dx%d is not a downsampling by integer factors", who, H, W, Ho, Wo);
  DEMON_REQUIRE(in_sn >= (long)C * H * W, "%s: batch stride %ld below one sample's %ld floats", who, in_sn, (long)C * H * W);
  return DEMON_OK;
}

// [N,C,H,W] planes `in_sn` floats apart -> packed [N,C,Ho,Wo]; the factors must be integers (area_check)
int area_launch(const float* in, float* out, int N, int C, int H, int W, int Ho, int Wo, long in_sn, cudaStream_t s) {
  const long total = (long)N * C * Ho * Wo;
  if (total == 0) return DEMON_OK;
  long blocks = (total + 255) / 256;
  if (blocks > 132 * 32) blocks = 132 * 32;
  const float scale = 1.0f / (float)((H / Ho) * (W / Wo));   // float32(1 / (fy fx)): one correctly rounded division
  (void)launch_pdl(area_planes_kernel, dim3((int)blocks), dim3(256), 0, s, in, out, N, C, H, W, Ho, Wo, in_sn, scale);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

// Flow2 extra inputs (blocks_original.py:155-183): depth_to_flow(inverse_depth, normalize_flow) ->
// zero where |flow| >= 1 or NaN -> warp2d(image2_2, normalized, 'value') -> NHWC12
// [warped(3), flow(2), depth(1), normal(3), 0, 0, 0].  dn2 = [depth, normal] NHWC4, motion [B,8] = rot|trans|scale.
// intrinsics: [B,4] normalised (fx, fy, cx, cy) of each sample (v2/blocks.py:154-161), or null for the constant the
// networks use (networks_original.py:108, v2/networks.py:90)
__global__ void __launch_bounds__(256) flow_extra_kernel(const float* __restrict__ dn2, const float* __restrict__ motion,
                                                        const float* __restrict__ image2_2, float* __restrict__ extra, int H, int W,
                                                        int extra_pitch, const float* __restrict__ intrinsics) {
  pdl_launch_dependents();   // common.cuh: programmatic dependent launch
  pdl_wait();
  __shared__ D2FCamera<float> cam;
  const int n = blockIdx.y;
  if (threadIdx.x == 0) {
    const float K[4] = {0.89115971f, 1.18821287f, 0.5f, 0.5f};  // networks_original.py:108
    d2f_camera(cam, intrinsics ? intrinsics + 4 * n : K, motion + 8 * n, motion + 8 * n + 3, DEMON_ROT_ANGLEAXIS3, W, H);
  }
  __syncthreads();
  const int hw = H * W;
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= hw) return;
  const int y = i / W, x = i - y * W;
  const float4 d = __ldg(reinterpret_cast<const float4*>(dn2) + (size_t)n * hw + i);
  float fx, fy;
  d2f_pixel(fx, fy, d.x, x, y, cam, true, true);
  const float norm = sqrtf(fadd(fmul(fx, fx), fmul(fy, fy)));
  if (!(norm < 1.0f)) { fx = 0.f; fy = 0.f; }
  const WarpTap<float> t = warp2d_tap<float>(x, y, fx, fy, W, H, true);
  const bool valid = warp2d_valid(t.x0, t.y0, W, H);
  float wv[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float r = 0.f;
    if (valid) {
      const float* p = image2_2 + ((size_t)n * 3 + c) * hw + (size_t)t.y0 * W + t.x0;
      r = warp2d_blend(__ldg(p), __ldg(p + 1), __ldg(p + W), __ldg(p + W + 1), t);
    }
    wv[c] = r;
  }
  float4* o = reinterpret_cast<float4*>(extra + ((size_t)n * hw + i) * extra_pitch);
  o[0] = make_float4(wv[0], wv[1], wv[2], fx);
  o[1] = make_float4(fy, d.x, d.y, d.z);
  o[2] = make_float4(d.w, 0.f, 0.f, 0.f);
}

// tf.clip_by_value(x, 0, 50) of TF 1.4 (v2/blocks.py:379): minimum(x, 50) then maximum(., 0) with the compare order of
// std::min / std::max, so +inf -> 50, -inf -> 0 and NaN stays NaN (neither less than 0 nor greater than 50)
__device__ __forceinline__ float clip_0_50(float x) {
  const float t = (50.f < x) ? 50.f : x;
  return (t < 0.f) ? 0.f : t;
}

// DM extra inputs (blocks_original.py:336-364): warp2d(image2_2, flow2) ++ flowconf2 (++ flow_to_depth) -> NHWC8.
// kClip (v2): the depth from flow is clipped to [0, 50] (v2/blocks.py:379).  intrinsics as in flow_extra_kernel.
// flow2: the flow that is warped with and turned into depth, NHWC with `flow2_pitch` floats per pixel, or null for the
// first two channels of flowconf2 (the networks' case: prev_flow2 is a slice of prev_flowconf2)
template <bool kClip>
__global__ void __launch_bounds__(128) dm_extra_kernel(const float* __restrict__ flowconf2, const float* __restrict__ motion_prev,
                                                      const float* __restrict__ image2_2, float* __restrict__ extra, int H, int W,
                                                      int extra_pitch, bool with_depth, const float* __restrict__ intrinsics,
                                                      const float* __restrict__ flow2, int flow2_pitch) {
  pdl_launch_dependents();   // common.cuh: programmatic dependent launch
  pdl_wait();
  __shared__ F2DCamera cam;
  const int n = blockIdx.y;
  if (with_depth && threadIdx.x == 0) {
    const float K[4] = {0.89115971f, 1.18821287f, 0.5f, 0.5f};
    f2d_camera(cam, intrinsics ? intrinsics + 4 * n : K, motion_prev + 8 * n, motion_prev + 8 * n + 3, DEMON_ROT_ANGLEAXIS3, W, H);
  }
  __syncthreads();
  const int hw = H * W;
  const int i = blockIdx.x * 128 + threadIdx.x;
  if (i >= hw) return;
  const int y = i / W, x = i - y * W;
  const float4 fc = __ldg(reinterpret_cast<const float4*>(flowconf2) + (size_t)n * hw + i);
  float fx = fc.x, fy = fc.y;
  if (flow2) {
    const float* f = flow2 + ((size_t)n * hw + i) * flow2_pitch;
    fx = __ldg(f); fy = __ldg(f + 1);
  }
  const WarpTap<float> t = warp2d_tap<float>(x, y, fx, fy, W, H, true);
  const bool valid = warp2d_valid(t.x0, t.y0, W, H);
  float wv[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float r = 0.f;
    if (valid) {
      const float* p = image2_2 + ((size_t)n * 3 + c) * hw + (size_t)t.y0 * W + t.x0;
      r = warp2d_blend(__ldg(p), __ldg(p + 1), __ldg(p + W), __ldg(p + W + 1), t);
    }
    wv[c] = r;
  }
  float dff = with_depth ? f2d_pixel(fx, fy, x, y, cam, true, true) : 0.f;
  if (kClip) dff = clip_0_50(dff);
  float* o = extra + ((size_t)n * hw + i) * extra_pitch;
  *reinterpret_cast<float4*>(o) = make_float4(wv[0], wv[1], wv[2], fc.x);
  *reinterpret_cast<float4*>(o + 4) = make_float4(fc.y, fc.z, fc.w, dff);
  // channels 8..11 belong to the Flow block's record (normal z, 0, 0, 0): clear them, a stale NaN there would survive its
  // zero weight (the buffer is shared by the two blocks; channels 12.. are never written by anybody)
  if (extra_pitch >= 12) *reinterpret_cast<float4*>(o + 8) = make_float4(0.f, 0.f, 0.f, 0.f);
}

// refinement input (blocks_original.py:466-482): concat(image1, nearest-neighbour upsampled depth2) -> NHWC4
// image1 is read with strides so it can alias image_pair[:, 0:3]; depth with (sample, pixel) strides.
__global__ void __launch_bounds__(256) refine_input_kernel(const float* __restrict__ image1, long img_sn, long img_sp, long img_sc,
                                                          const float* __restrict__ depth, long d_sn, long d_sp, float* __restrict__ rin,
                                                          int N, int H, int W, int h, int w) {
  pdl_launch_dependents();   // common.cuh: programmatic dependent launch
  pdl_wait();
  const long total = (long)N * H * W;
  for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long)gridDim.x * 256) {
    const int x = (int)(i % W);
    const long r = i / W;
    const int y = (int)(r % H);
    const int n = (int)(r / H);
    const long p = (long)y * W + x;
    const float* im = image1 + n * img_sn + p * img_sp;
    // tf.image.resize_nearest_neighbor, align_corners=False: src = floor(dst * in / out)
    const int sy = (int)(((long)y * h) / H), sx = (int)(((long)x * w) / W);
    const float dv = __ldg(depth + n * d_sn + ((long)sy * w + sx) * d_sp);
    reinterpret_cast<float4*>(rin)[2 * i] = make_float4(__ldg(im), __ldg(im + img_sc), __ldg(im + 2 * img_sc), dv);
    reinterpret_cast<float4*>(rin)[2 * i + 1] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// uint8 input (examples/example.py:15-42: PIL RGB images, `np.array(img).astype(np.float32)/255 - 0.5`, pair concat):
// images [B,2,H,W,3] uint8 -> img8 [B,H,W,8] fp32 = [image1 rgb, image2 rgb, 0, 0] (the conv1y input) and the NCHW
// fp32 planes of image 2 (input of the median3x3 pair that makes image2_2, examples/evaluation.py:170-173).
// Same two IEEE operations as numpy's float32 expression, so the result equals the fp32 entry bit for bit.
__global__ void __launch_bounds__(256) u8_import_kernel(const unsigned char* __restrict__ images, float* __restrict__ img8,
                                                       float* __restrict__ planes2, int B, int P) {
  pdl_launch_dependents();   // common.cuh: programmatic dependent launch
  pdl_wait();
  const long total = (long)B * P;
  for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long)gridDim.x * 256) {
    const int n = (int)(i / P), p = (int)(i - (long)n * P);
    const unsigned char* a = images + ((long)n * 2 * P + p) * 3;
    const unsigned char* b = a + (long)P * 3;
    float v[6];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      v[c] = fsub(fdiv((float)a[c], 255.0f), 0.5f);
      v[3 + c] = fsub(fdiv((float)b[c], 255.0f), 0.5f);
    }
    reinterpret_cast<float4*>(img8)[2 * i] = make_float4(v[0], v[1], v[2], v[3]);
    reinterpret_cast<float4*>(img8)[2 * i + 1] = make_float4(v[4], v[5], 0.f, 0.f);
    if (planes2) {
      float* q = planes2 + (long)n * 3 * P + p;
      q[0] = v[3]; q[P] = v[4]; q[2L * P] = v[5];
    }
  }
}

// image2_2 given as uint8 [B,h,w,3] (examples/example.py:22: the PIL-resized second image) -> NCHW fp32 planes
__global__ void __launch_bounds__(256) u8_planes_kernel(const unsigned char* __restrict__ img, float* __restrict__ planes, int B, int P) {
  pdl_launch_dependents();   // common.cuh: programmatic dependent launch
  pdl_wait();
  const long total = (long)B * P;
  for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long)gridDim.x * 256) {
    const int n = (int)(i / P), p = (int)(i - (long)n * P);
    const unsigned char* a = img + i * 3;
    float* q = planes + (long)n * 3 * P + p;
#pragma unroll
    for (int c = 0; c < 3; ++c) q[(long)c * P] = fsub(fdiv((float)a[c], 255.0f), 0.5f);
  }
}

// ---------------------------------------------------------------------------------------------
// forward passes
// ---------------------------------------------------------------------------------------------
int import_image_pair(demon_net* n, const float* image_pair, int data_format, cudaStream_t s) {
  const int P = 192 * 256;
  return strided_copy(image_pair, n->img8->p, n->B, P, 6, api_strides(data_format, P, 6), buf_strides(n->img8), s);
}

// i22 holds NCHW planes: an NCHW image2_2 is a plain copy
int import_image2_2(demon_net* n, const float* image2_2, int data_format, cudaStream_t s) {
  const int P = 48 * 64;
  if (data_format == 0) {
    DEMON_CHECK_CUDA(cudaMemcpyAsync(n->i22->p, image2_2, (size_t)n->B * 3 * P * sizeof(float), cudaMemcpyDeviceToDevice, s));
    return DEMON_OK;
  }
  return strided_copy(image2_2, n->i22->p, n->B, P, 3, api_strides(data_format, P, 3), api_strides(0, P, 3), s);
}

// planes: image 2 as NCHW fp32 planes, `sn` floats between samples (6*P inside an image pair, 3*P for a packed copy)
int median_image2_2(demon_net* n, const float* planes, long sn, cudaStream_t s) {
  const int B = n->B;
  (void)launch_pdl(median_planes_kernel, dim3(dim3(1, 96, B * 3)), dim3(128), 0, s, planes, n->i22_half->p, 3, 192, 256, 96, 128, sn, 3L * 96 * 128);
  DEMON_LAUNCH_CHECK();
  (void)launch_pdl(median_planes_kernel, dim3(dim3(1, 48, B * 3)), dim3(128), 0, s, n->i22_half->p, n->i22->p, 3, 96, 128, 48, 64, 3L * 96 * 128, 3L * 48 * 64);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

// image2_2 made from image 2's planes when the call brings none: image2_2_mode 2 is resize_area to 48x64
// (training/v2/training.py:179), any other the median pair
int downsample_image2_2(demon_net* n, const float* planes, long sn, int64_t image2_2_mode, cudaStream_t s) {
  if (image2_2_mode == 2) return area_launch(planes, n->i22->p, n->B, 3, 192, 256, 48, 64, sn, s);
  return median_image2_2(n, planes, sn, s);
}

// export one NHWC channel slice to the API layout
int export_slice(demon_net* n, const Buf* b, int coff, int C, float* dst, int data_format, cudaStream_t s) {
  if (!dst) return DEMON_OK;
  const int P = b->H * b->W;
  return strided_copy(b->p + coff, dst, n->B, P, C, buf_strides(b), api_strides(data_format, P, C), s);
}

int export_predictions(demon_net* n, float* flow5, float* flow2, float* depth2, float* normal2, float* rotation, float* translation,
                       int data_format, cudaStream_t s) {
  int rc;
  if ((rc = export_slice(n, n->pf5, 0, 2, flow5, data_format, s))) return rc;
  if ((rc = export_slice(n, n->flowconf2, 0, 2, flow2, data_format, s))) return rc;
  if ((rc = export_slice(n, n->dn2, 0, 1, depth2, data_format, s))) return rc;
  if ((rc = export_slice(n, n->dn2, 1, 3, normal2, data_format, s))) return rc;
  if (rotation && (rc = strided_copy(n->motion->p, rotation, n->B, 1, 3, {8, 0, 1}, {3, 0, 1}, s))) return rc;
  if (translation && (rc = strided_copy(n->motion->p + 3, translation, n->B, 1, 3, {8, 0, 1}, {3, 0, 1}, s))) return rc;
  return DEMON_OK;
}

// flow block (blocks_original.py:190-235); `head`: run conv1 / conv2 (false when the pipeline has hoisted them out of the
// iteration loop); `intrinsics`: the cameras of the samples [B,4] on the device, or null for the networks' constant
int run_flow_block(demon_net* n, const Block& b, bool iterative, cudaStream_t s, bool head = true, const float* intrinsics = nullptr) {
  int rc;
  if (head && (rc = run_layers(n, b.begin, b.head_end, s))) return rc;
  if (iterative) {
    (void)launch_pdl(flow_extra_kernel, dim3(dim3(ceil_div(48 * 64, 256), n->B)), dim3(256), 0, s, n->dn2->p, n->motion->p, n->i22->p, n->extra_in->p, 48, 64, n->extra_in->C,
                     intrinsics);
    DEMON_LAUNCH_CHECK();
  }
  return run_layers(n, b.head_end, b.end, s);
}

// `flow2`: the flow the extra inputs warp with (NHWC, `flow2_pitch` floats per pixel), or null for flowconf2's first two
// channels; `intrinsics` as in run_flow_block
int run_dm_block(demon_net* n, const Block& b, bool iterative, cudaStream_t s, bool head = true, const float* intrinsics = nullptr,
                 const float* flow2 = nullptr, int flow2_pitch = 0) {
  int rc;
  if (head && (rc = run_layers(n, b.begin, b.head_end, s))) return rc;
  // the previous motion is still in n->motion here: this block's motion_fc3 overwrites it later
  (void)launch_pdl(n->variant == 2 ? dm_extra_kernel<true> : dm_extra_kernel<false>, dim3(dim3(ceil_div(48 * 64, 128), n->B)), dim3(128), 0, s,
                   n->flowconf2->p, n->motion->p, n->i22->p, n->extra_in->p, 48, 64, n->extra_in->C, iterative, intrinsics, flow2, flow2_pitch);
  DEMON_LAUNCH_CHECK();
  return run_layers(n, b.head_end, b.end, s);
}

// `depth`: channel 0 of (sample, pixel) strided depth planes; `depth0`: the output, or null for rdepth0
int run_refine_block(demon_net* n, const float* image1, Strides img, const float* depth, Strides dep, int dh, int dw, float* depth0,
                     cudaStream_t s) {
  const long total = (long)n->B * n->RH * n->RW;
  long blocks = (total + 255) / 256;
  if (blocks > 132 * 32) blocks = 132 * 32;
  (void)launch_pdl(refine_input_kernel, dim3((int)blocks), dim3(256), 0, s, image1, img.n, img.p, img.c, depth, dep.n, dep.p, n->rin->p, n->B, n->RH, n->RW, dh, dw);
  DEMON_LAUNCH_CHECK();
  const Block& b = n->refine;
  int rc;
  if ((rc = run_layers(n, b.begin, b.end - 1, s))) return rc;
  // the last layer writes straight into the caller's output (C = 1: NHWC == NCHW)
  return run_layer_profiled(n, b.end - 1, s, depth0);
}

// v2: predict_depth0/conv2 writes depth0 ++ normal0 into rdepth0, from where the two are exported in `data_format`
int run_refine_block_v2(demon_net* n, const float* image1, Strides img, const float* depth, Strides dep, int dh, int dw, float* depth0,
                        float* normal0, int data_format, cudaStream_t s) {
  int rc = run_refine_block(n, image1, img, depth, dep, dh, dw, nullptr, s);
  if (rc || (rc = export_slice(n, n->rdepth0, 0, 1, depth0, data_format, s))) return rc;
  return export_slice(n, n->rdepth0, 1, 3, normal0, data_format, s);
}

}  // namespace
}  // namespace demon

// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------
extern "C" {

static int net_create(demon_net** out, int batch, int refine_h, int refine_w, int precision, int variant) {
  DEMON_REQUIRE(out, "demon_net_create: null out");
  DEMON_REQUIRE(batch >= 1 && batch <= 4096, "demon_net_create: batch %d", batch);
  DEMON_REQUIRE(refine_h >= 4 && refine_w >= 4 && refine_h % 4 == 0 && refine_w % 4 == 0, "demon_net_create: refine size %dx%d must be a multiple of 4", refine_h, refine_w);
  DEMON_REQUIRE(precision >= 0 && precision <= DEMON_PREC_FP16, "demon_net_create: precision %d", precision);
  std::unique_ptr<demon_net> n(new demon_net());
  n->B = batch; n->RH = refine_h; n->RW = refine_w; n->precision = precision; n->variant = variant;
  DEMON_CHECK_CUDA(cudaGetDevice(&n->device));
  if (variant == 2) build_plan_v2(n.get());
  else build_plan(n.get());
  void* p = nullptr;
  DEMON_CHECK_CUDA(cudaMalloc(&p, n->ws_floats * sizeof(float)));
  n->ws = (float*)p;
  DEMON_CHECK_CUDA(cudaMemset(p, 0, n->ws_floats * sizeof(float)));
  for (auto& b : n->bufs) b->p = n->ws + b->offset;
  *out = n.release();
  return DEMON_OK;
}

int demon_net_create(demon_net** out, int batch, int refine_h, int refine_w, int precision) {
  return net_create(out, batch, refine_h, refine_w, precision, 1);
}

int demon_net_create_v2(demon_net** out, int batch, int refine_h, int refine_w, int precision) {
  return net_create(out, batch, refine_h, refine_w, precision, 2);
}

int demon_net_variant(const demon_net* n) { return n ? n->variant : 0; }

void demon_net_destroy(demon_net* n) {
  if (!n) return;
  for (void* p : n->dev_allocs) cudaFree(p);
  for (cudaEvent_t e : n->prof_events) cudaEventDestroy(e);
  for (auto& g : n->graphs) if (g.exec) cudaGraphExecDestroy(g.exec);
  if (n->cap_stream) cudaStreamDestroy(n->cap_stream);
  for (auto& l : n->layers) tc_layer_free(l->tc);
  cudaFree(n->ws);
  delete n;
}

int demon_net_num_variables(const demon_net* n) { return n ? (int)n->var_names.size() : 0; }
const char* demon_net_variable_name(const demon_net* n, int i) {
  if (!n || i < 0 || i >= (int)n->var_names.size()) return nullptr;
  return n->var_names[i].c_str();
}

int demon_net_set_weight(demon_net* n, const char* name, const float* data, const int64_t* shape, int rank) {
  DEMON_REQUIRE(n && name && data && shape, "demon_net_set_weight: null argument");
  if (n->finalized) return fail(DEMON_E_STATE, "demon_net_set_weight after finalize");
  std::string nm(name);
  const size_t slash = nm.rfind('/');
  DEMON_REQUIRE(slash != std::string::npos, "demon_net_set_weight: bad name %s", name);
  const std::string lname = nm.substr(0, slash), leaf = nm.substr(slash + 1);
  auto it = n->by_name.find(lname);
  if (it == n->by_name.end() || (leaf != "kernel" && leaf != "bias")) return fail(DEMON_E_NOTFOUND, "unknown variable %s", name);
  const Layer& l = *it->second;
  std::vector<int64_t> want = l.kshape;
  if (leaf == "bias") want = {l.cout};
  bool ok = (int)want.size() == rank;
  for (int i = 0; ok && i < rank; ++i) ok = want[i] == shape[i];
  if (!ok) {
    std::string w, g;
    for (auto v : want) w += std::to_string(v) + ",";
    for (int i = 0; i < rank; ++i) g += std::to_string(shape[i]) + ",";
    return fail(DEMON_E_INVALID, "variable %s: expected shape [%s] got [%s]", name, w.c_str(), g.c_str());
  }
  int64_t numel = 1;
  for (int i = 0; i < rank; ++i) numel *= shape[i];
  n->host_vars[nm].assign(data, data + numel);
  return DEMON_OK;
}

int demon_net_finalize(demon_net* n) {
  DEMON_REQUIRE(n, "demon_net_finalize: null net");
  if (n->finalized) return DEMON_OK;
  for (auto& nm : n->var_names)
    if (!n->host_vars.count(nm)) return fail(DEMON_E_STATE, "demon_net_finalize: variable %s was not set", nm.c_str());
  for (auto& lp : n->layers) {
    Layer& l = *lp;
    const int rc = upload_layer(l, n->host_vars[l.name + "/kernel"].data(), n->host_vars[l.name + "/bias"].data(), n->B, n->precision,
                                n->dev_allocs);
    if (rc) return rc;
  }
  // scratch of the split-K tensor-core layers: the largest need, owned by the net
  size_t need = 0;
  for (auto& lp : n->layers) need = std::max(need, lp->tc.splitk_bytes);
  if (need) {
    void* q = nullptr;
    DEMON_CHECK_CUDA(cudaMalloc(&q, need));
    n->dev_allocs.push_back(q);
    n->tc_scratch = static_cast<float*>(q);
  }
  n->host_vars.clear();
  n->finalized = true;
  return DEMON_OK;
}

int demon_debug_tc_timeouts(void) { return tc_read_error_flag(false); }
int demon_check_errors(void) {
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) return fail(DEMON_E_CUDA, "demon_check_errors: %s", cudaGetErrorString(e));
  if (tc_read_error_flag(true))
    return fail(DEMON_E_STATE, "a pipeline wait inside a tensor-core convolution kernel timed out: results since the last check are invalid");
  return DEMON_OK;
}
int demon_debug_tc_timing(int enable, int64_t* host_out, int nblocks) {
  if (host_out) return tc_halo_read_timing(reinterpret_cast<long long*>(host_out), nblocks);
  tc_halo_enable_timing(enable != 0);
  return 0;
}

int demon_net_batch(const demon_net* n) { return n ? n->B : 0; }
int64_t demon_net_workspace_bytes(const demon_net* n) { return n ? (int64_t)(n->ws_floats * sizeof(float)) : 0; }
int demon_net_pipeline_launches(const demon_net* n, int iterations) {
  if (!n || iterations < 0 || iterations > 7) return 0;
  return n->pipeline_launches[iterations];
}
int demon_net_snapshot_launches(const demon_net* n, int iterations) {
  if (!n || iterations < 0 || iterations > 7) return 0;
  return n->snapshot_launches[iterations];
}
int demon_net_layer_uses_tensor_cores(const demon_net* n, const char* name) {
  if (!n || !name) return 0;
  auto it = n->by_name.find(name);
  return (it != n->by_name.end() && it->second->use_tc()) ? 1 : 0;
}

int demon_net_profile_begin(demon_net* n) {
  DEMON_REQUIRE(n, "null net");
  n->profiling = true;
  n->prof_used = 0;
  n->prof_layer.clear();
  n->prof_ms.assign(n->layers.size(), 0.0);
  n->prof_calls.assign(n->layers.size(), 0);
  return DEMON_OK;
}

// Call after the stream has been synchronised.  Stops profiling and folds the event pairs into per-layer sums.
int demon_net_profile_end(demon_net* n) {
  DEMON_REQUIRE(n, "null net");
  n->profiling = false;
  for (size_t i = 0; i < n->prof_layer.size(); ++i) {
    float ms = 0.f;
    DEMON_CHECK_CUDA(cudaEventElapsedTime(&ms, n->prof_events[2 * i], n->prof_events[2 * i + 1]));
    n->prof_ms[n->prof_layer[i]] += ms;
    n->prof_calls[n->prof_layer[i]] += 1;
  }
  n->prof_layer.clear();
  n->prof_used = 0;
  return DEMON_OK;
}

int demon_net_num_layers(const demon_net* n) { return n ? (int)n->layers.size() : 0; }
const char* demon_net_layer_name(const demon_net* n, int i) {
  if (!n || i < 0 || i >= (int)n->layers.size()) return nullptr;
  return n->layers[i]->name.c_str();
}
// accumulated device time (ms) and number of calls of layer i since demon_net_profile_begin; kernel launches per call
int demon_net_layer_profile(const demon_net* n, int i, double* ms, int64_t* calls, int* launches_per_call, int* uses_tc) {
  DEMON_REQUIRE(n && i >= 0 && i < (int)n->layers.size(), "layer index");
  if (ms) *ms = i < (int)n->prof_ms.size() ? n->prof_ms[i] : 0.0;
  if (calls) *calls = i < (int)n->prof_calls.size() ? n->prof_calls[i] : 0;
  const Layer& l = *n->layers[i];
  if (launches_per_call) *launches_per_call = (l.use_tc() ? 1 : (l.kind == L_DECONV ? 4 : (l.ksplit > 1 ? 2 : 1))) + (l.nhwc ? 2 : 0);
  // kernel family: 0 conv_simt_kernel, 2 conv_tc_halo_kernel (halo), 3 conv_tc_halo_kernel (per tap)
  if (uses_tc) *uses_tc = !l.use_tc() ? 0 : (l.tc.per_tap ? 3 : 2);
  return DEMON_OK;
}

// A forward entry of network variant v (1: the demon_* entries, 2: the demon_*_v2 entries) takes only a net of that variant
#define REQUIRE_READY_AS(n, v)                                                   \
  do {                                                                           \
    DEMON_REQUIRE(n, "null net");                                                \
    DEMON_REQUIRE((n)->variant == (v), "a v%d net handle was passed to a v%d entry", (n)->variant, (v)); \
    if (!(n)->finalized) return fail(DEMON_E_STATE, "forward before demon_net_finalize"); \
    int _dev = -1;                                                               \
    cudaGetDevice(&_dev);                                                        \
    if (_dev != (n)->device)                                                     \
      return fail(DEMON_E_STATE, "net handle belongs to CUDA device %d but device %d is current", (n)->device, _dev); \
  } while (0)
#define REQUIRE_READY(n) REQUIRE_READY_AS(n, 1)

static int bootstrap_impl(demon_net* n, const float* image_pair, const float* image2_2, float* flow5, float* flow2, float* depth2,
                          float* normal2, float* rotation, float* translation, int data_format, void* stream) {
  DEMON_REQUIRE(image_pair && image2_2, "bootstrap: null input");
  DEMON_REQUIRE(data_format == 0 || data_format == 1, "bootstrap: data_format %d", data_format);
  cudaStream_t s = (cudaStream_t)stream;
  int rc;
  if ((rc = import_image_pair(n, image_pair, data_format, s))) return rc;
  if ((rc = import_image2_2(n, image2_2, data_format, s))) return rc;
  if ((rc = run_flow_block(n, n->flow1, false, s))) return rc;
  if ((rc = run_dm_block(n, n->dm1, false, s))) return rc;
  return export_predictions(n, flow5, flow2, depth2, normal2, rotation, translation, data_format, s);
}

int demon_bootstrap_forward(demon_net* n, const float* image_pair, const float* image2_2, float* flow5, float* flow2, float* depth2,
                            float* normal2, float* rotation, float* translation, int data_format, void* stream) {
  REQUIRE_READY(n);
  return bootstrap_impl(n, image_pair, image2_2, flow5, flow2, depth2, normal2, rotation, translation, data_format, stream);
}

int demon_bootstrap_forward_v2(demon_net* n, const float* image_pair, const float* image2_2, float* flow5, float* flow2, float* depth2,
                               float* normal2, float* rotation, float* translation, int data_format, void* stream) {
  REQUIRE_READY_AS(n, 2);
  return bootstrap_impl(n, image_pair, image2_2, flow5, flow2, depth2, normal2, rotation, translation, data_format, stream);
}

// previous predictions -> dn2 (NHWC4) and motion [B,8], where the flow and DM blocks' extra inputs read them
static int import_prev_depth_normal(demon_net* n, const float* depth2, const float* normal2, int data_format, cudaStream_t s) {
  const int P = 48 * 64;
  int rc;
  if ((rc = strided_copy(depth2, n->dn2->p, n->B, P, 1, api_strides(data_format, P, 1), buf_strides(n->dn2), s))) return rc;
  return strided_copy(normal2, n->dn2->p + 1, n->B, P, 3, api_strides(data_format, P, 3), buf_strides(n->dn2), s);
}

static int import_prev_motion(demon_net* n, const float* rotation, const float* translation, cudaStream_t s) {
  int rc;
  if ((rc = strided_copy(rotation, n->motion->p, n->B, 1, 3, {3, 0, 1}, {8, 0, 1}, s))) return rc;
  return strided_copy(translation, n->motion->p + 3, n->B, 1, 3, {3, 0, 1}, {8, 0, 1}, s);
}

static int iterative_impl(demon_net* n, const float* image_pair, const float* image2_2, const float* depth2_in, const float* normal2_in,
                          const float* rotation_in, const float* translation_in, float* flow5, float* flow2, float* depth2,
                          float* normal2, float* rotation, float* translation, int data_format, void* stream) {
  DEMON_REQUIRE(image_pair && image2_2 && depth2_in && normal2_in && rotation_in && translation_in, "iterative: null input");
  DEMON_REQUIRE(data_format == 0 || data_format == 1, "iterative: data_format %d", data_format);
  cudaStream_t s = (cudaStream_t)stream;
  int rc;
  if ((rc = import_image_pair(n, image_pair, data_format, s))) return rc;
  if ((rc = import_image2_2(n, image2_2, data_format, s))) return rc;
  if ((rc = import_prev_depth_normal(n, depth2_in, normal2_in, data_format, s))) return rc;
  if ((rc = import_prev_motion(n, rotation_in, translation_in, s))) return rc;
  if ((rc = run_flow_block(n, n->flow2, true, s))) return rc;
  if ((rc = run_dm_block(n, n->dm2, true, s))) return rc;
  return export_predictions(n, flow5, flow2, depth2, normal2, rotation, translation, data_format, s);
}

int demon_iterative_forward(demon_net* n, const float* image_pair, const float* image2_2, const float* depth2_in, const float* normal2_in,
                            const float* rotation_in, const float* translation_in, float* flow5, float* flow2, float* depth2,
                            float* normal2, float* rotation, float* translation, int data_format, void* stream) {
  REQUIRE_READY(n);
  return iterative_impl(n, image_pair, image2_2, depth2_in, normal2_in, rotation_in, translation_in, flow5, flow2, depth2, normal2,
                        rotation, translation, data_format, stream);
}

int demon_iterative_forward_v2(demon_net* n, const float* image_pair, const float* image2_2, const float* depth2_in, const float* normal2_in,
                               const float* rotation_in, const float* translation_in, float* flow5, float* flow2, float* depth2,
                               float* normal2, float* rotation, float* translation, int data_format, void* stream) {
  REQUIRE_READY_AS(n, 2);
  return iterative_impl(n, image_pair, image2_2, depth2_in, normal2_in, rotation_in, translation_in, flow5, flow2, depth2, normal2,
                        rotation, translation, data_format, stream);
}

int demon_refine_forward(demon_net* n, const float* image1, const float* depth2, float* depth0, int data_format, void* stream) {
  REQUIRE_READY(n);
  DEMON_REQUIRE(image1 && depth2 && depth0, "refine: null pointer");
  DEMON_REQUIRE(data_format == 0 || data_format == 1, "refine: data_format %d", data_format);
  const long P = (long)n->RH * n->RW;
  const int dh = n->RH / 4, dw = n->RW / 4;
  return run_refine_block(n, image1, api_strides(data_format, P, 3), depth2, api_strides(data_format, (long)dh * dw, 1), dh, dw, depth0,
                          (cudaStream_t)stream);
}

// normal2 is accepted and not read, as by the reference's RefinementNet.eval (v2/networks.py:204-228)
int demon_refine_forward_v2(demon_net* n, const float* image1, const float* depth2, const float* normal2, float* depth0, float* normal0,
                            int data_format, void* stream) {
  REQUIRE_READY_AS(n, 2);
  (void)normal2;
  DEMON_REQUIRE(image1 && depth2 && depth0, "refine_v2: null pointer");
  DEMON_REQUIRE(data_format == 0 || data_format == 1, "refine_v2: data_format %d", data_format);
  const long P = (long)n->RH * n->RW;
  const int dh = n->RH / 4, dw = n->RW / 4;
  return run_refine_block_v2(n, image1, api_strides(data_format, P, 3), depth2, api_strides(data_format, (long)dh * dw, 1), dh, dw, depth0,
                             normal0, data_format, (cudaStream_t)stream);
}

// The scope of a block entry: `second` is set for the iterative block's scope (netFlow2 / netDM2), whose weights include
// conv2_extra_inputs over the previous predictions.  Each argument in `args` must be given for that scope and absent for
// the bootstrap one (netFlow1 / netDM1).
struct BlockArg { const char* name; const void* p; };
static int check_block_args(const char* entry, const char* scope, const char* first, const char* second_name, bool* second,
                            const BlockArg* args, int nargs) {
  DEMON_REQUIRE(scope, "%s: null scope", entry);
  *second = strcmp(scope, second_name) == 0;
  DEMON_REQUIRE(*second || strcmp(scope, first) == 0, "%s: scope must be %s or %s, got '%s'", entry, first, second_name, scope);
  for (int k = 0; k < nargs; ++k) {
    if (*second) DEMON_REQUIRE(args[k].p, "%s: scope %s needs %s", entry, scope, args[k].name);
    else DEMON_REQUIRE(!args[k].p, "%s: scope %s takes no %s (its weights have no input for it)", entry, scope, args[k].name);
  }
  return DEMON_OK;
}

int demon_flow_block_forward_v2(demon_net* n, const char* scope, const float* image_pair, const float* image2_2, const float* intrinsics,
                                const float* prev_depth2, const float* prev_normal2, const float* prev_rotation,
                                const float* prev_translation, float* flowconf5, float* flowconf2, int data_format, void* stream) {
  REQUIRE_READY_AS(n, 2);
  bool iterative = false;
  const BlockArg args[] = {{"intrinsics", intrinsics}, {"prev_predictions['predict_depth2']", prev_depth2},
                           {"prev_predictions['predict_normal2']", prev_normal2},
                           {"prev_predictions['predict_rotation']", prev_rotation},
                           {"prev_predictions['predict_translation']", prev_translation}};
  int rc;
  if ((rc = check_block_args("flow_block", scope, "netFlow1", "netFlow2", &iterative, args, 5))) return rc;
  // netFlow1 does not read image2_2 (v2/blocks.py:142-144), so there it may come or not
  if (iterative) DEMON_REQUIRE(image2_2, "flow_block: scope %s needs image2_2", scope);
  DEMON_REQUIRE(image_pair, "flow_block: null image_pair");
  DEMON_REQUIRE(data_format == 0 || data_format == 1, "flow_block: data_format %d", data_format);
  cudaStream_t s = (cudaStream_t)stream;
  if ((rc = import_image_pair(n, image_pair, data_format, s))) return rc;
  if (iterative) {
    if ((rc = import_image2_2(n, image2_2, data_format, s))) return rc;
    if ((rc = import_prev_depth_normal(n, prev_depth2, prev_normal2, data_format, s))) return rc;
    if ((rc = import_prev_motion(n, prev_rotation, prev_translation, s))) return rc;
  }
  if ((rc = run_flow_block(n, iterative ? n->flow2 : n->flow1, iterative, s, true, intrinsics))) return rc;
  if ((rc = export_slice(n, n->pf5, 0, 4, flowconf5, data_format, s))) return rc;
  return export_slice(n, n->flowconf2, 0, 4, flowconf2, data_format, s);
}

int demon_depthmotion_block_forward_v2(demon_net* n, const char* scope, const float* image_pair, const float* image2_2,
                                       const float* prev_flow2, const float* prev_flowconf2, const float* prev_rotation,
                                       const float* prev_translation, const float* intrinsics, float* depth2, float* normal2,
                                       float* rotation, float* translation, float* scale, int data_format, void* stream) {
  REQUIRE_READY_AS(n, 2);
  bool iterative = false;
  const BlockArg args[] = {{"prev_rotation", prev_rotation}, {"prev_translation", prev_translation}, {"intrinsics", intrinsics}};
  int rc;
  if ((rc = check_block_args("depthmotion_block", scope, "netDM1", "netDM2", &iterative, args, 3))) return rc;
  DEMON_REQUIRE(image_pair, "depthmotion_block: null image_pair");
  DEMON_REQUIRE(image2_2, "depthmotion_block: null image2_2");
  DEMON_REQUIRE(prev_flow2, "depthmotion_block: null prev_flow2");
  DEMON_REQUIRE(prev_flowconf2, "depthmotion_block: null prev_flowconf2");
  DEMON_REQUIRE(data_format == 0 || data_format == 1, "depthmotion_block: data_format %d", data_format);
  cudaStream_t s = (cudaStream_t)stream;
  const int P = 48 * 64;
  if ((rc = import_image_pair(n, image_pair, data_format, s))) return rc;
  if ((rc = import_image2_2(n, image2_2, data_format, s))) return rc;
  // prev_flowconf2 -> flowconf2 (NHWC4), prev_flow2 -> p2a's first two channels: p2a is next written by
  // predict_depthnormal2/conv1, after the extra inputs have read it
  if ((rc = strided_copy(prev_flowconf2, n->flowconf2->p, n->B, P, 4, api_strides(data_format, P, 4), buf_strides(n->flowconf2), s)))
    return rc;
  if ((rc = strided_copy(prev_flow2, n->p2a->p, n->B, P, 2, api_strides(data_format, P, 2), buf_strides(n->p2a), s))) return rc;
  if (iterative && (rc = import_prev_motion(n, prev_rotation, prev_translation, s))) return rc;
  if ((rc = run_dm_block(n, iterative ? n->dm2 : n->dm1, iterative, s, true, intrinsics, n->p2a->p, n->p2a->C))) return rc;
  if ((rc = export_predictions(n, nullptr, nullptr, depth2, normal2, rotation, translation, data_format, s))) return rc;
  return scale ? strided_copy(n->motion->p + 6, scale, n->B, 1, 1, {8, 0, 1}, {1, 0, 1}, s) : DEMON_OK;
}

// The intrinsics DeMoN was trained for (examples/example.py:51-61), in pixels of the 256x192 input
static const double kNetIntrinsics[4] = {0.89115971 * 256, 1.18821287 * 192, 0.5 * 256, 0.5 * 192};

// The predictions at snapshot point k (0 = bootstrap, k = after iteration k) into the call's outputs, at slice k with
// snapshots, then the refinement block on them unless the call takes snapshots without it
static int export_outputs(demon_net* n, const PipelineCall& c, int k, cudaStream_t s) {
  const long B = n->B, P2 = 48L * 64, P0 = 192L * 256;
  const long slice = c.snapshots == NO_SNAPSHOTS ? 0 : k;
  const auto at = [slice](float* p, long per_snapshot) { return p ? p + slice * per_snapshot : nullptr; };
  const PipelineOutputs& o = c.out;
  int rc = export_predictions(n, nullptr, at(o.flow2, B * 2 * P2), at(o.depth2, B * P2), at(o.normal2, B * 3 * P2), at(o.rotation, B * 3),
                              at(o.translation, B * 3), 0, s);
  if (rc || c.snapshots == SNAPSHOTS) return rc;
  if (n->variant == 2)
    return run_refine_block_v2(n, n->img8->p, buf_strides(n->img8), n->dn2->p, buf_strides(n->dn2), 48, 64, at(o.depth0, B * P0),
                               at(o.normal0, B * 3 * P0), 0, s);
  // image1 is read back from img8 (NHWC8: the first three channels), whatever the input kind; no depth0: into rdepth0
  return run_refine_block(n, n->img8->p, buf_strides(n->img8), n->dn2->p, buf_strides(n->dn2), 48, 64, at(o.depth0, B * P0), s);
}

static int pipeline_body(demon_net* n, const PipelineCall& c, cudaStream_t s) {
  int rc;
  const long P = 192L * 256;
  const uint8_t* images = c.images;
  const uint8_t* image2_2_u8 = c.image2_2_u8;
  if (c.input == IN_RESIZE || c.input == IN_VIEWS) {
    uint8_t* pair = reinterpret_cast<uint8_t*>(n->pair_bytes->p);
    if (c.input == IN_VIEWS)
      rc = adjust_intrinsics_launch(c.images, c.sn, c.si, 2, c.sy, 2 * n->B, (int)c.h, (int)c.w, c.K, kNetIntrinsics, pair, 192, 256,
                                    c.status, s);
    else
      rc = resize_u8_launch(c.images, c.sn, c.si, 2, c.sy, 2 * n->B, (int)c.h, (int)c.w, pair, 192, 256, (int)c.resample, s);
    if (rc) return rc;
    images = pair;
    if (c.image2_2_mode == 1) {
      uint8_t* i22 = reinterpret_cast<uint8_t*>(n->i22_bytes->p);
      if ((rc = resize_u8_launch(pair + P * 3, 2 * P * 3, 0, 1, 256 * 3, n->B, 192, 256, i22, 48, 64, (int)c.resample, s))) return rc;
      image2_2_u8 = i22;
    }
  }
  if (c.input != IN_FP32) {
    // img8 straight from the bytes; without image2_2, image 2's planes for the median pair
    float* planes2 = image2_2_u8 ? nullptr : n->planes2->p;
    long blocks = ((long)n->B * P + 255) / 256;
    if (blocks > 132 * 32) blocks = 132 * 32;
    (void)launch_pdl(u8_import_kernel, dim3((int)blocks), dim3(256), 0, s, images, n->img8->p, planes2, n->B, (int)P);
    DEMON_LAUNCH_CHECK();
    if (image2_2_u8) {
      long b2 = ((long)n->B * 48 * 64 + 255) / 256;
      (void)launch_pdl(u8_planes_kernel, dim3((int)b2), dim3(256), 0, s, image2_2_u8, n->i22->p, n->B, 48 * 64);
      DEMON_LAUNCH_CHECK();
    } else if ((rc = downsample_image2_2(n, planes2, 3 * P, c.image2_2_mode, s))) {
      return rc;
    }
  } else {
    if ((rc = import_image_pair(n, c.image_pair, 0, s))) return rc;
    if (c.image2_2) {
      if ((rc = import_image2_2(n, c.image2_2, 0, s))) return rc;
    } else {
      if ((rc = downsample_image2_2(n, c.image_pair + 3 * P, 6 * P, c.image2_2_mode, s))) return rc;
    }
  }
  // k = 0: the bootstrap blocks; k > 0: iteration k
  for (int k = 0; k <= c.iterations; ++k) {
    if ((rc = run_flow_block(n, k ? n->flow2 : n->flow1, k > 0, s, k == 0))) return rc;
    if ((rc = run_dm_block(n, k ? n->dm2 : n->dm1, k > 0, s, k == 0))) return rc;
    if ((c.snapshots != NO_SNAPSHOTS || k == c.iterations) && (rc = export_outputs(n, c, k, s))) return rc;
    // conv1 / conv2 of netFlow2 and netDM2 read only the image pair and fixed weights: once per call instead of once per
    // iteration (bit identical; 2 x 2 x 221.7 MMAC per pair less to execute at three iterations)
    if (k == 0 && c.iterations > 0) {
      if ((rc = run_layers(n, n->flow2.begin, n->flow2.head_end, s))) return rc;
      if ((rc = run_layers(n, n->dm2.begin, n->dm2.head_end, s))) return rc;
    }
  }
  return DEMON_OK;
}

// The fused pipeline is not traced: a graph captured with the trace's copies inside would replay them after it is cleared
static int refuse_while_tracing(const demon_net* n) {
  if (n->tracing) return fail(DEMON_E_STATE, "pipeline: a layer trace is set (demon_debug_trace_layers); only the stage-wise entries are traced");
  return DEMON_OK;
}

static int pipeline_forward_impl(demon_net* n, const PipelineCall& c, void* stream) {
  if (int rc = refuse_while_tracing(n)) return rc;
  DEMON_REQUIRE(c.iterations >= 0 && c.iterations <= 7, "pipeline: iterations %d", (int)c.iterations);
  int* launch_record = c.snapshots != NO_SNAPSHOTS ? n->snapshot_launches : n->pipeline_launches;
  DEMON_REQUIRE(n->RH == 192 && n->RW == 256, "pipeline: net was created with a %dx%d refinement block", n->RH, n->RW);
  cudaStream_t s = (cudaStream_t)stream;
  // The call is one CUDA graph per distinct PipelineCall (DEMON_GRAPH=0 disables): the first call with a new one runs
  // eagerly, the second captures, later ones replay.  Not used while per-layer profiling is on or when the caller is itself
  // capturing this stream.
  static const bool graphs_on = []() { const char* e = getenv("DEMON_GRAPH"); return !(e && e[0] == '0'); }();
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(s, &cap);
  if (graphs_on && !n->profiling && cap == cudaStreamCaptureStatusNone) {
    for (auto& g : n->graphs)
      if (memcmp(&g.call, &c, sizeof(c)) == 0) {
        if (g.exec == nullptr) {   // second call: capture
          cudaGraph_t graph = nullptr;
          const int64_t l0 = g_launch_count.load();
          if (!n->cap_stream) DEMON_CHECK_CUDA(cudaStreamCreateWithFlags(&n->cap_stream, cudaStreamNonBlocking));
          DEMON_CHECK_CUDA(cudaStreamBeginCapture(n->cap_stream, cudaStreamCaptureModeThreadLocal));
          int rc = pipeline_body(n, c, n->cap_stream);
          cudaError_t e = cudaStreamEndCapture(n->cap_stream, &graph);
          if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
          if (e != cudaSuccess) return fail(DEMON_E_CUDA, "pipeline: stream capture failed: %s", cudaGetErrorString(e));
          g.launches = (int)(g_launch_count.load() - l0);
          g_launch_count.fetch_sub(g.launches);   // counted again by the launch below
          e = cudaGraphInstantiate(&g.exec, graph, 0);
          cudaGraphDestroy(graph);
          if (e != cudaSuccess) { g.exec = nullptr; return fail(DEMON_E_CUDA, "pipeline: graph instantiate failed: %s", cudaGetErrorString(e)); }
        }
        DEMON_CHECK_CUDA(cudaGraphLaunch(g.exec, s));
        g_launch_count.fetch_add(g.launches);
        launch_record[c.iterations] = g.launches;
        return DEMON_OK;
      }
    if (n->graphs.size() >= 32) {   // evict the oldest entry
      if (n->graphs.front().exec) cudaGraphExecDestroy(n->graphs.front().exec);
      n->graphs.erase(n->graphs.begin());
    }
    n->graphs.push_back({c, nullptr, 0});
  }
  const int64_t launches0 = g_launch_count.load();
  int rc = pipeline_body(n, c, s);
  if (rc) return rc;
  launch_record[c.iterations] = (int)(g_launch_count.load() - launches0);
  return DEMON_OK;
}

int demon_pipeline_forward(demon_net* n, const float* image_pair, const float* image2_2, int iterations, float* depth0, float* rotation,
                           float* translation, float* flow2, float* depth2, float* normal2, void* stream) {
  REQUIRE_READY(n);
  DEMON_REQUIRE(image_pair, "pipeline: null image_pair");
  PipelineCall c{};
  c.input = IN_FP32; c.image_pair = image_pair; c.image2_2 = image2_2; c.iterations = iterations;
  c.out = {depth0, rotation, translation, flow2, depth2, normal2};
  return pipeline_forward_impl(n, c, stream);
}

int demon_pipeline_forward_v2(demon_net* n, const float* image_pair, const float* image2_2, int iterations, float* depth0, float* normal0,
                              float* rotation, float* translation, float* flow2, float* depth2, float* normal2, void* stream) {
  REQUIRE_READY_AS(n, 2);
  DEMON_REQUIRE(image_pair, "pipeline_v2: null image_pair");
  PipelineCall c{};
  c.input = IN_FP32; c.image_pair = image_pair; c.image2_2 = image2_2; c.iterations = iterations;
  c.out = {depth0, rotation, translation, flow2, depth2, normal2, normal0};
  return pipeline_forward_impl(n, c, stream);
}

// The image2_2 source of a v2 entry that takes pairs at the network's size (uint8 or float32): 0 (the given image2_2, or
// the median pair without one) or 2 (resize_area of image 2; then there is no given image2_2)
static int check_pair_mode(int image2_2_mode, const void* image2_2, const char* who) {
  DEMON_REQUIRE(image2_2_mode == 0 || image2_2_mode == 2, "%s: image2_2_mode %d is not 0 (median) or 2 (area)", who, image2_2_mode);
  DEMON_REQUIRE(image2_2_mode == 0 || !image2_2, "%s: image2_2_mode 2 (area) computes image2_2, which must then be NULL", who);
  return DEMON_OK;
}

// snapshot k of every output at slice k; the refinement block runs on every snapshot iff depth0 is given
static int snapshots_impl(demon_net* n, const float* image_pair, const float* image2_2, int image2_2_mode, int iterations,
                          const PipelineOutputs& o, void* stream) {
  DEMON_REQUIRE(image_pair, "pipeline_snapshots: null image_pair");
  DEMON_REQUIRE(o.depth0 || !o.normal0, "pipeline_snapshots: normal0 without depth0 (normal0 comes out of the refinement block)");
  PipelineCall c{};
  c.input = IN_FP32; c.image_pair = image_pair; c.image2_2 = image2_2; c.image2_2_mode = image2_2_mode; c.iterations = iterations;
  c.out = o;
  c.snapshots = o.depth0 ? SNAPSHOTS_REFINED : SNAPSHOTS;
  return pipeline_forward_impl(n, c, stream);
}

int demon_pipeline_forward_snapshots(demon_net* n, const float* image_pair, const float* image2_2, int iterations, float* flow2,
                                     float* depth2, float* normal2, float* rotation, float* translation, float* depth0, void* stream) {
  REQUIRE_READY(n);
  return snapshots_impl(n, image_pair, image2_2, 0, iterations, {depth0, rotation, translation, flow2, depth2, normal2}, stream);
}

int demon_pipeline_forward_snapshots_v2(demon_net* n, const float* image_pair, const float* image2_2, int image2_2_mode, int iterations,
                                        float* depth0, float* normal0, float* rotation, float* translation, float* flow2, float* depth2,
                                        float* normal2, void* stream) {
  REQUIRE_READY_AS(n, 2);
  if (int rc = check_pair_mode(image2_2_mode, image2_2, "pipeline_snapshots_v2")) return rc;
  return snapshots_impl(n, image_pair, image2_2, image2_2_mode, iterations, {depth0, rotation, translation, flow2, depth2, normal2, normal0},
                        stream);
}

static int u8_impl(demon_net* n, const uint8_t* images, const uint8_t* image2_2, int image2_2_mode, int iterations, const PipelineOutputs& o,
                   void* stream) {
  DEMON_REQUIRE(images, "pipeline_u8: null images");
  PipelineCall c{};
  c.input = IN_U8; c.images = images; c.image2_2_u8 = image2_2; c.image2_2_mode = image2_2_mode; c.iterations = iterations;
  c.out = o;
  return pipeline_forward_impl(n, c, stream);
}

int demon_pipeline_forward_u8(demon_net* n, const uint8_t* images, const uint8_t* image2_2, int iterations, float* depth0, float* rotation,
                              float* translation, float* flow2, float* depth2, float* normal2, void* stream) {
  REQUIRE_READY(n);
  return u8_impl(n, images, image2_2, 0, iterations, {depth0, rotation, translation, flow2, depth2, normal2}, stream);
}

int demon_pipeline_forward_u8_v2(demon_net* n, const uint8_t* images, const uint8_t* image2_2, int image2_2_mode, int iterations,
                                 float* depth0, float* normal0, float* rotation, float* translation, float* flow2, float* depth2,
                                 float* normal2, void* stream) {
  REQUIRE_READY_AS(n, 2);
  if (int rc = check_pair_mode(image2_2_mode, image2_2, "pipeline_u8_v2")) return rc;
  return u8_impl(n, images, image2_2, image2_2_mode, iterations, {depth0, rotation, translation, flow2, depth2, normal2, normal0}, stream);
}

// The argument checks shared by the entries that take uint8 pairs of any size, which then fill the source fields of `c`.
// image2_2_mode 2 (area) is v2's only: it is the input training/v2/training.py feeds v2, and v1 never saw it
static int set_source(const demon_net* n, PipelineCall& c, PipelineInput input, const uint8_t* images, int64_t sn, int64_t si, int64_t sy,
                      int h, int w, int resample, int image2_2_mode, const char* who) {
  DEMON_REQUIRE(sn >= 0 && si >= 0 && sy >= 0, "%s: negative stride", who);
  if (n->variant == 2)
    DEMON_REQUIRE(image2_2_mode >= 0 && image2_2_mode <= 2, "%s: image2_2_mode %d is not 0 (median), 1 (resize) or 2 (area)", who,
                  image2_2_mode);
  else
    DEMON_REQUIRE(image2_2_mode == 0 || image2_2_mode == 1, "%s: image2_2_mode %d is not 0 (median) or 1 (resize)", who, image2_2_mode);
  c.input = input; c.images = images; c.sn = sn; c.si = si; c.sy = sy; c.h = h; c.w = w; c.resample = resample;
  c.image2_2_mode = image2_2_mode;
  return DEMON_OK;
}

static int images_impl(demon_net* n, const uint8_t* images, int64_t sn, int64_t si, int64_t sy, int h, int w, int resample,
                       int image2_2_mode, int iterations, const PipelineOutputs& o, void* stream) {
  DEMON_REQUIRE(images, "pipeline_images_u8: null images");
  PipelineCall c{};
  int rc = set_source(n, c, IN_RESIZE, images, sn, si, sy, h, w, resample, image2_2_mode, "pipeline_images_u8");
  if (rc || (rc = resize_u8_check(h, w, 192, 256, resample, "pipeline_images_u8"))) return rc;
  c.iterations = iterations;
  c.out = o;
  return pipeline_forward_impl(n, c, stream);
}

int demon_pipeline_forward_images_u8(demon_net* n, const uint8_t* images, int64_t sn, int64_t si, int64_t sy, int h, int w, int resample,
                                     int image2_2_mode, int iterations, float* depth0, float* rotation, float* translation, float* flow2,
                                     float* depth2, float* normal2, void* stream) {
  REQUIRE_READY(n);
  return images_impl(n, images, sn, si, sy, h, w, resample, image2_2_mode, iterations, {depth0, rotation, translation, flow2, depth2, normal2},
                     stream);
}

int demon_pipeline_forward_images_u8_v2(demon_net* n, const uint8_t* images, int64_t sn, int64_t si, int64_t sy, int h, int w, int resample,
                                        int image2_2_mode, int iterations, float* depth0, float* normal0, float* rotation, float* translation,
                                        float* flow2, float* depth2, float* normal2, void* stream) {
  REQUIRE_READY_AS(n, 2);
  return images_impl(n, images, sn, si, sy, h, w, resample, image2_2_mode, iterations,
                     {depth0, rotation, translation, flow2, depth2, normal2, normal0}, stream);
}

static int views_impl(demon_net* n, const uint8_t* images, int64_t sn, int64_t si, int64_t sy, int h, int w, const double* K, uint8_t* status,
                      int resample, int image2_2_mode, int iterations, const PipelineOutputs& o, void* stream) {
  DEMON_REQUIRE(images && K && status, "pipeline_views_u8: null images, K or status");
  PipelineCall c{};
  int rc = set_source(n, c, IN_VIEWS, images, sn, si, sy, h, w, resample, image2_2_mode, "pipeline_views_u8");
  if (rc || (rc = adjust_intrinsics_check(h, w, kNetIntrinsics, 192, 256, "pipeline_views_u8"))) return rc;
  if ((rc = resize_u8_check(192, 256, 48, 64, resample, "pipeline_views_u8"))) return rc;
  c.K = K; c.status = status; c.iterations = iterations;
  c.out = o;
  return pipeline_forward_impl(n, c, stream);
}

int demon_pipeline_forward_views_u8(demon_net* n, const uint8_t* images, int64_t sn, int64_t si, int64_t sy, int h, int w, const double* K,
                                    uint8_t* status, int resample, int image2_2_mode, int iterations, float* depth0, float* rotation,
                                    float* translation, float* flow2, float* depth2, float* normal2, void* stream) {
  REQUIRE_READY(n);
  return views_impl(n, images, sn, si, sy, h, w, K, status, resample, image2_2_mode, iterations,
                    {depth0, rotation, translation, flow2, depth2, normal2}, stream);
}

int demon_pipeline_forward_views_u8_v2(demon_net* n, const uint8_t* images, int64_t sn, int64_t si, int64_t sy, int h, int w, const double* K,
                                       uint8_t* status, int resample, int image2_2_mode, int iterations, float* depth0, float* normal0,
                                       float* rotation, float* translation, float* flow2, float* depth2, float* normal2, void* stream) {
  REQUIRE_READY_AS(n, 2);
  return views_impl(n, images, sn, si, sy, h, w, K, status, resample, image2_2_mode, iterations,
                    {depth0, rotation, translation, flow2, depth2, normal2, normal0}, stream);
}

// H2D of the inputs into the staging buffers (build_plan, build_plan_v2), the pipeline of network `variant`, D2H of depth0 /
// normal0 (v2) / rotation / translation
static int pipeline_host(demon_net* n, int variant, const void* images_host, const void* image2_2_host, bool u8, int image2_2_mode,
                         int iterations, float* depth0_host, float* normal0_host, float* rotation_host, float* translation_host, void* stream,
                         bool sync) {
  REQUIRE_READY_AS(n, variant);
  if (int rc = refuse_while_tracing(n)) return rc;
  DEMON_REQUIRE(images_host && depth0_host, "pipeline_host: null pointer");
  if (variant == 2)
    if (int rc = check_pair_mode(image2_2_mode, image2_2_host, "pipeline_host_v2")) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  const size_t px = (size_t)n->B * 192 * 256;
  const size_t ip_bytes = u8 ? px * 6 : px * 6 * sizeof(float);
  const size_t i22_bytes = (size_t)n->B * 3 * 48 * 64 * (u8 ? 1 : sizeof(float));
  void* ip_dev = n->pair_bytes->p;
  void* i22_dev = image2_2_host ? n->i22_bytes->p : nullptr;
  DEMON_CHECK_CUDA(cudaMemcpyAsync(ip_dev, images_host, ip_bytes, cudaMemcpyHostToDevice, s));
  if (i22_dev) DEMON_CHECK_CUDA(cudaMemcpyAsync(i22_dev, image2_2_host, i22_bytes, cudaMemcpyHostToDevice, s));
  float* rt_dev = n->host_motion->p;
  PipelineCall c{};
  if (u8) { c.input = IN_U8; c.images = static_cast<const uint8_t*>(ip_dev); c.image2_2_u8 = static_cast<const uint8_t*>(i22_dev); }
  else { c.input = IN_FP32; c.image_pair = static_cast<const float*>(ip_dev); c.image2_2 = static_cast<const float*>(i22_dev); }
  c.image2_2_mode = image2_2_mode;
  c.iterations = iterations;
  c.out.depth0 = n->host_depth0->p;
  c.out.normal0 = normal0_host ? n->host_normal0->p : nullptr;
  c.out.rotation = rotation_host ? rt_dev : nullptr;
  c.out.translation = translation_host ? rt_dev + 3 * n->B : nullptr;
  int rc = pipeline_forward_impl(n, c, stream);
  if (rc) return rc;
  DEMON_CHECK_CUDA(cudaMemcpyAsync(depth0_host, c.out.depth0, px * sizeof(float), cudaMemcpyDeviceToHost, s));
  if (normal0_host) DEMON_CHECK_CUDA(cudaMemcpyAsync(normal0_host, c.out.normal0, px * 3 * sizeof(float), cudaMemcpyDeviceToHost, s));
  if (rotation_host) DEMON_CHECK_CUDA(cudaMemcpyAsync(rotation_host, rt_dev, (size_t)n->B * 3 * sizeof(float), cudaMemcpyDeviceToHost, s));
  if (translation_host)
    DEMON_CHECK_CUDA(cudaMemcpyAsync(translation_host, rt_dev + 3 * n->B, (size_t)n->B * 3 * sizeof(float), cudaMemcpyDeviceToHost, s));
  if (sync) {
    DEMON_CHECK_CUDA(cudaStreamSynchronize(s));
    if (tc_read_error_flag(true))
      return fail(DEMON_E_STATE, "a pipeline wait inside a tensor-core convolution kernel timed out: the outputs are invalid");
  }
  return DEMON_OK;
}

int demon_pipeline_forward_host(demon_net* n, const float* image_pair_host, const float* image2_2_host, int iterations, float* depth0_host,
                                float* rotation_host, float* translation_host, void* stream) {
  return pipeline_host(n, 1, image_pair_host, image2_2_host, false, 0, iterations, depth0_host, nullptr, rotation_host, translation_host,
                       stream, true);
}

int demon_pipeline_forward_host_async(demon_net* n, const float* image_pair_host, const float* image2_2_host, int iterations,
                                      float* depth0_host, float* rotation_host, float* translation_host, void* stream) {
  return pipeline_host(n, 1, image_pair_host, image2_2_host, false, 0, iterations, depth0_host, nullptr, rotation_host, translation_host,
                       stream, false);
}

int demon_pipeline_forward_host_u8(demon_net* n, const uint8_t* images_host, const uint8_t* image2_2_host, int iterations, float* depth0_host,
                                   float* rotation_host, float* translation_host, void* stream) {
  return pipeline_host(n, 1, images_host, image2_2_host, true, 0, iterations, depth0_host, nullptr, rotation_host, translation_host, stream,
                       true);
}

int demon_pipeline_forward_host_u8_async(demon_net* n, const uint8_t* images_host, const uint8_t* image2_2_host, int iterations,
                                         float* depth0_host, float* rotation_host, float* translation_host, void* stream) {
  return pipeline_host(n, 1, images_host, image2_2_host, true, 0, iterations, depth0_host, nullptr, rotation_host, translation_host, stream,
                       false);
}

int demon_pipeline_forward_host_v2(demon_net* n, const float* image_pair_host, const float* image2_2_host, int image2_2_mode, int iterations,
                                   float* depth0_host, float* normal0_host, float* rotation_host, float* translation_host, void* stream) {
  return pipeline_host(n, 2, image_pair_host, image2_2_host, false, image2_2_mode, iterations, depth0_host, normal0_host, rotation_host,
                       translation_host, stream, true);
}

int demon_pipeline_forward_host_async_v2(demon_net* n, const float* image_pair_host, const float* image2_2_host, int image2_2_mode,
                                         int iterations, float* depth0_host, float* normal0_host, float* rotation_host,
                                         float* translation_host, void* stream) {
  return pipeline_host(n, 2, image_pair_host, image2_2_host, false, image2_2_mode, iterations, depth0_host, normal0_host, rotation_host,
                       translation_host, stream, false);
}

int demon_pipeline_forward_host_u8_v2(demon_net* n, const uint8_t* images_host, const uint8_t* image2_2_host, int image2_2_mode, int iterations,
                                      float* depth0_host, float* normal0_host, float* rotation_host, float* translation_host, void* stream) {
  return pipeline_host(n, 2, images_host, image2_2_host, true, image2_2_mode, iterations, depth0_host, normal0_host, rotation_host,
                       translation_host, stream, true);
}

int demon_pipeline_forward_host_u8_async_v2(demon_net* n, const uint8_t* images_host, const uint8_t* image2_2_host, int image2_2_mode,
                                            int iterations, float* depth0_host, float* normal0_host, float* rotation_host,
                                            float* translation_host, void* stream) {
  return pipeline_host(n, 2, images_host, image2_2_host, true, image2_2_mode, iterations, depth0_host, normal0_host, rotation_host,
                       translation_host, stream, false);
}

// resize_area over NCHW planes (area_planes_kernel): input [N,C,h,w] with `in_sn` floats between samples -> packed
// [N,C,oh,ow]; h / oh and w / ow must be integers
int demon_resize_area_f32(const float* input, int64_t in_sn, float* output, int n, int c, int h, int w, int oh, int ow, void* stream) {
  if (int rc = area_check(n, c, h, w, oh, ow, (long)in_sn, "resize_area")) return rc;
  if ((int64_t)n * c == 0) return DEMON_OK;
  DEMON_REQUIRE(input && output, "resize_area: null pointer");
  return area_launch(input, output, n, c, h, w, oh, ow, (long)in_sn, (cudaStream_t)stream);
}

// debug: the geometry of every layer of the net and which kernel family / plan it got (one line per layer).  A v2 conv's
// line also gives its first tap (dy, dx): minus the 'same' padding before the first row / column.
int demon_debug_describe_layers(const demon_net* n, char* buf, int buflen) {
  DEMON_REQUIRE(n && buf && buflen > 0, "describe: null");
  static const char* const kKind[] = {"conv", "deconv", "dense"};
  int off = 0;
  for (auto& lp : n->layers) {
    if (off >= buflen - 512) break;
    const Layer& l = *lp;
    off += snprintf(buf + off, buflen - off,
                    "%-40s %s H %d W %d cin %d cin_buf %d in_pitch %d in_off %d cout %d out_pitch %d out_off %d kh %d kw %d sy %d sx %d leaky %d scale %d : ",
                    l.name.c_str(), kKind[l.kind], l.in->H, l.in->W, l.cin, l.cin_buf, l.in->C, l.in_coff, l.cout, l.out->C, l.out_coff,
                    l.kh, l.kw, l.sy, l.sx, l.leaky ? 1 : 0, l.scale ? 1 : 0);
    if (l.tf_same) {
      ConvProblem p;
      build_problems(l, n->B, &p);
      off += snprintf(buf + off, buflen - off, "tap0 %d %d : ", p.dy[0], p.dx[0]);
    }
    off += describe_layer(l, n->B, n->precision, buf + off, buflen - off);
    off += snprintf(buf + off, buflen - off, "\n");
  }
  return off;
}

// debug, no device needed: demon_debug_describe_layers of the plan a net of this variant (1 or 2), batch, refinement size
// and precision gets, without creating it
int demon_debug_describe_plan(int variant, int batch, int refine_h, int refine_w, int precision, char* buf, int buflen) {
  DEMON_REQUIRE(variant == 1 || variant == 2, "describe_plan: variant %d", variant);
  DEMON_REQUIRE(batch >= 1 && refine_h >= 4 && refine_w >= 4 && refine_h % 4 == 0 && refine_w % 4 == 0, "describe_plan: shape");
  DEMON_REQUIRE(precision >= 0 && precision <= DEMON_PREC_FP16, "describe_plan: precision %d", precision);
  std::unique_ptr<demon_net> n(new demon_net());
  n->B = batch; n->RH = refine_h; n->RW = refine_w; n->precision = precision; n->variant = variant;
  if (variant == 2) build_plan_v2(n.get());
  else build_plan(n.get());
  // the buffers at their workspace offsets from a 256-byte aligned base that is never dereferenced (the planner looks at
  // alignment only)
  float* base = reinterpret_cast<float*>(uintptr_t(1) << 32);
  for (auto& b : n->bufs) b->p = base + b->offset;
  return demon_debug_describe_layers(n.get(), buf, buflen);
}

// debug: per-layer input / output copies of the stage-wise entries (run_layer_profiled)
int demon_debug_trace_layers(demon_net* n, float* const* in, float* const* out) {
  DEMON_REQUIRE(n, "trace: null net");
  const size_t L = n->layers.size();
  n->trace_in.assign(L, nullptr);
  n->trace_out.assign(L, nullptr);
  if (in) std::copy(in, in + L, n->trace_in.begin());
  if (out) std::copy(out, out + L, n->trace_out.begin());
  n->tracing = in || out;
  return DEMON_OK;
}

// debug, no device needed: the plan of one convolution shape ([B,H,W,Cin] NHWC, channel pitches given)
int demon_debug_describe_conv(int B, int H, int W, int Cin, int in_pitch, int Cout, int out_pitch, int kh, int kw, int sy, int sx, int deconv,
                              int precision, char* buf, int buflen) {
  DEMON_REQUIRE(buf && buflen > 0, "describe: null");
  DEMON_REQUIRE(precision >= 0 && precision <= DEMON_PREC_FP16, "describe: precision %d", precision);
  StandaloneLayer s(nullptr, nullptr, H, W, Cin, in_pitch, Cout, out_pitch, kh, kw, sy, sx, deconv != 0, false);
  return describe_layer(s.layer, B, precision, buf, buflen);
}

// ---- standalone convolution entries (tests) ---------------------------------------------------
static double g_last_conv_ms = -1.0;
double demon_debug_last_conv_ms(void) { return g_last_conv_ms; }

static int standalone_conv(const float* in, int in_pitch, float* out, int out_pitch, int B, int H, int W, int Cin, int Cout, int kh, int kw,
                           int sy, int sx, const float* kernel_host, const float* bias_host, int leaky, int precision, bool deconv, void* stream,
                           bool tf_same = false) {
  DEMON_REQUIRE(in && out && kernel_host && bias_host, "conv: null pointer");
  DEMON_REQUIRE(Cin % 4 == 0, "conv test entry: Cin must be a multiple of 4");
  DEMON_REQUIRE(B >= 1 && H >= 1 && W >= 1 && Cout >= 1 && in_pitch >= Cin && out_pitch >= Cout, "conv test entry: shape or pitch");
  if (deconv) DEMON_REQUIRE(kh == 4 && kw == 4 && sy == 2 && sx == 2, "deconv: only k4 s2");
  else DEMON_REQUIRE(kh >= 1 && kw >= 1 && kh * kw <= kMaxTaps && (kh & 1) && (kw & 1), "conv: kernel %dx%d", kh, kw);
  DEMON_REQUIRE(sy >= 1 && sx >= 1, "conv: stride");
  DEMON_REQUIRE(precision >= 0 && precision <= DEMON_PREC_FP16, "conv: precision %d", precision);
  std::vector<void*> allocs;
  StandaloneLayer s(in, out, H, W, Cin, in_pitch, Cout, out_pitch, kh, kw, sy, sx, deconv, leaky != 0);
  Layer& l = s.layer;
  l.tf_same = tf_same;
  int rc = upload_layer(l, kernel_host, bias_host, B, precision, allocs);
  if (rc == DEMON_OK && precision != DEMON_PREC_FP32_SIMT && !l.use_tc())
    rc = fail(DEMON_E_INVALID, "conv test entry: shape not supported by the tensor-core path");
  float* tc_ws = nullptr;
  if (rc == DEMON_OK && l.tc.splitk_bytes) {
    void* q = nullptr;
    if (cudaMalloc(&q, l.tc.splitk_bytes) == cudaSuccess) {
      allocs.push_back(q);
      tc_ws = static_cast<float*>(q);
    } else {
      rc = fail(DEMON_E_CUDA, "conv test entry: scratch allocation failed");
    }
  }
  cudaError_t e = cudaSuccess;
  if (rc == DEMON_OK) {
    cudaEvent_t ev0, ev1;
    cudaEventCreate(&ev0); cudaEventCreate(&ev1);
    cudaEventRecord(ev0, (cudaStream_t)stream);
    rc = run_layer(l, B, (cudaStream_t)stream, nullptr, tc_ws);
    cudaEventRecord(ev1, (cudaStream_t)stream);
    e = cudaStreamSynchronize((cudaStream_t)stream);
    float ms = -1.f;
    if (e == cudaSuccess && cudaEventElapsedTime(&ms, ev0, ev1) == cudaSuccess) g_last_conv_ms = ms;
    cudaEventDestroy(ev0); cudaEventDestroy(ev1);
  }
  for (void* q : allocs) cudaFree(q);
  tc_layer_free(l.tc);
  if (rc) return rc;
  if (e != cudaSuccess) return fail(DEMON_E_CUDA, "conv test entry: %s", cudaGetErrorString(e));
  return DEMON_OK;
}

int demon_conv_slice_nhwc(const float* in, int in_pitch, float* out, int out_pitch, int B, int H, int W, int Cin, int Cout, int kh, int kw,
                          int sy, int sx, int deconv, const float* kernel_host, const float* bias_host, int leaky, int precision, void* stream) {
  return standalone_conv(in, in_pitch, out, out_pitch, B, H, W, Cin, Cout, kh, kw, sy, sx, kernel_host, bias_host, leaky, precision,
                         deconv != 0, stream);
}

// demon_conv_slice_nhwc of a convolution with the taps of tf.layers.conv2d(padding='same') (the v2 network's layers):
// along each axis the first tap reads pad_before = max((ceil(n/s) - 1) s + k - n, 0) / 2 before the output's first pixel
int demon_conv_slice_nhwc_same(const float* in, int in_pitch, float* out, int out_pitch, int B, int H, int W, int Cin, int Cout, int kh,
                               int kw, int sy, int sx, const float* kernel_host, const float* bias_host, int leaky, int precision, void* stream) {
  return standalone_conv(in, in_pitch, out, out_pitch, B, H, W, Cin, Cout, kh, kw, sy, sx, kernel_host, bias_host, leaky, precision, false,
                         stream, true);
}

int demon_conv2d_nhwc(const float* in, float* out, int B, int H, int W, int Cin, int Cout, int kh, int kw, int sy, int sx,
                      const float* kernel_host, const float* bias_host, int leaky, int precision, void* stream) {
  return demon_conv_slice_nhwc(in, Cin, out, Cout, B, H, W, Cin, Cout, kh, kw, sy, sx, 0, kernel_host, bias_host, leaky, precision, stream);
}

int demon_deconv4x4s2_nhwc(const float* in, float* out, int B, int H, int W, int Cin, int Cout, const float* kernel_host,
                           const float* bias_host, int leaky, int precision, void* stream) {
  return demon_conv_slice_nhwc(in, Cin, out, Cout, B, H, W, Cin, Cout, 4, 4, 2, 2, 1, kernel_host, bias_host, leaky, precision, stream);
}

}  // extern "C"
