// Network plan of the DeMoN `networks_original` graphs: buffers, layers, glue kernels, C ABI.
//
// The five blocks (netFlow1, netDM1, netFlow2, netDM2, netRefine; networks_original.py:44,50,125,142,227)
// are laid out once, at demon_net_create, as lists of convolution problems over NHWC buffers carved
// out of one device workspace.  Skip-concats are channel slices of shared buffers (conv.cuh), the
// geometry ops between the blocks (blocks_original.py:155-187,336-366) run as two fused glue kernels
// that produce the `conv2_extra_inputs` tensor directly, and nothing on the forward path allocates,
// synchronises or touches the host.
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "conv.cuh"
#include "conv_tc.cuh"
#include "geometry.cuh"

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
  const float* scale = nullptr;
  int scale_stride = 0;
  bool dense_nchw_flatten = false;  // motion_fc1: TF flattens NCHW (blocks_original.py:388-392)
  int dense_c = 0, dense_hw = 0;
  // expected TF variable shapes
  std::vector<int64_t> kshape;
  // device parameters
  int cout_pad = 0;
  float* w_dev[4] = {nullptr, nullptr, nullptr, nullptr};  // 1 (conv/dense) or 4 (deconv parity classes)
  float* bias_dev = nullptr;
  // tensor-core path
  bool use_tc = false;
  TcLayer tc;
  // split-K for dense layers (SIMT path)
  int ksplit = 1;
};

struct HostVar {
  std::vector<float> data;
  std::vector<int64_t> shape;
};

}  // namespace
}  // namespace demon

using namespace demon;

struct demon_net {
  int B = 0, RH = 0, RW = 0;
  int precision = DEMON_PREC_FP32_SIMT;
  int device = 0;            // the CUDA device the handle was created on; every entry point checks it is current
  bool finalized = false;
  float* ws = nullptr;
  size_t ws_floats = 0;
  std::vector<std::unique_ptr<Buf>> bufs;
  std::vector<std::unique_ptr<Layer>> layers;
  std::map<std::string, Layer*> by_name;
  std::vector<std::string> var_names;
  std::map<std::string, HostVar> host_vars;
  std::vector<void*> dev_allocs;
  int pipeline_launches[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  // CUDA graphs of demon_pipeline_forward, keyed by the pointer arguments (launch-bound at small batch: ~270 launches)
  struct GraphEntry { std::vector<const void*> key; cudaGraphExec_t exec; int launches; };
  std::vector<GraphEntry> graphs;
  cudaStream_t cap_stream = nullptr;   // capture happens on this private stream (the caller's may be the legacy default stream)
  // optional per-layer timing with CUDA events on the launching stream (bench.py's roofline leg)
  bool profiling = false;
  std::vector<cudaEvent_t> prof_events;      // pairs (start, stop)
  std::vector<int> prof_layer;               // layer index of every pair
  size_t prof_used = 0;
  std::vector<double> prof_ms;               // accumulated per layer
  std::vector<int64_t> prof_calls;

  // named buffers
  float* tc_scratch = nullptr;   // partial sums of the split-K tensor-core layers (conv_tc_halo.cu), sized at finalize
  Buf *cat2_f2, *cat2_d2;   // conv2 || conv2_extra_inputs of netFlow2 / netDM2: their conv2 half is loop invariant (see pipeline_body)
  Buf *img8, *i22, *i22_half, *c1y, *c1, *c2y, *cat2, *extra_in, *exy, *c21y, *concat2, *c3y, *c3, *c31y, *concat3, *c4y, *c4,
      *c41y, *concat4, *c5y, *c5, *c51y, *c51, *pf5a, *pf5, *p2a, *flowconf2, *dn2, *mc1, *fc1, *fc2, *motion;
  Buf *rin, *concat0, *rc1, *concat1, *rc2, *rc21, *pd0a, *rdepth0, *splitk;

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
  // convrelu2_caffe_padding (helpers.py:105-153): y conv into `mid`, x conv into `out`
  void add_sep(const std::string& name, int k, int stride, Buf* in, int in_coff, int cin, Buf* mid, int cmid, Buf* out,
               int out_coff, int cout) {
    add_layer(name + "y", L_CONV, in, in_coff, cin, mid, 0, cmid, k, 1, stride, 1, true);
    add_layer(name + "x", L_CONV, mid, 0, cmid, out, out_coff, cout, 1, k, 1, stride, true);
  }
};

namespace demon {
namespace {

// ---------------------------------------------------------------------------------------------
// plan construction
// ---------------------------------------------------------------------------------------------
void build_trunk(demon_net* n, const std::string& s, bool flow, bool iterative) {
  const int conv2_out = (flow && !iterative) ? 64 : 32;
  // conv1 and conv2 of the iterative nets depend only on the image pair (blocks_original.py:141,147 / :331,333), so the
  // pipeline computes them once per call: they get a concat buffer of their own that survives the other blocks
  Buf* cat2 = iterative ? (flow ? n->cat2_f2 : n->cat2_d2) : n->cat2;
  n->add_sep(s + "conv1", 9, 2, n->img8, 0, 6, n->c1y, 32, n->c1, 0, 32);
  n->add_sep(s + "conv2", 7, 2, n->c1, 0, 32, n->c2y, conv2_out, cat2, 0, conv2_out);
  if (!(flow && !iterative)) {
    const int extra = flow ? 9 : (iterative ? 8 : 7);
    n->add_sep(s + "conv2_extra_inputs", 3, 1, n->extra_in, 0, extra, n->exy, 32, cat2, 32, 32);
    // the 7 / 8 / 9 real channels sit in a 32-channel (128-byte) pixel whose other channels are zero and carry zero weights:
    // one K = 32 chunk of the tensor-core halo kernel (3 steps per tile) instead of the fp32 SIMT kernel
    n->by_name[s + "conv2_extra_inputsy"]->cin_buf = 32;
  }
  n->add_sep(s + "conv2_1", 3, 1, cat2, 0, 64, n->c21y, 64, n->concat2, 64, 64);
  n->add_sep(s + "conv3", 5, 2, n->concat2, 64, 64, n->c3y, 128, n->c3, 0, 128);
  n->add_sep(s + "conv3_1", 3, 1, n->c3, 0, 128, n->c31y, 128, n->concat3, 128, 128);
  n->add_sep(s + "conv4", 5, 2, n->concat3, 128, 128, n->c4y, 256, n->c4, 0, 256);
  n->add_sep(s + "conv4_1", 3, 1, n->c4, 0, 256, n->c41y, 256, n->concat4, 256, 256);
  n->add_sep(s + "conv5", flow ? 5 : 3, 2, n->concat4, 256, 256, n->c5y, 512, n->c5, 0, 512);
  n->add_sep(s + "conv5_1", 3, 1, n->c5, 0, 512, n->c51y, 512, n->c51, 0, 512);
}

void build_flow_block(demon_net* n, const std::string& scope, bool iterative) {
  const std::string s = scope + "/";
  build_trunk(n, s, true, iterative);
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
}

void build_dm_block(demon_net* n, const std::string& scope, bool iterative) {
  const std::string s = scope + "/";
  build_trunk(n, s, false, iterative);
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
  dn->scale = nullptr;  // bound to motion[:,6] at finalize (buffer addresses are not known yet)
  dn->scale_stride = 8;
}

void build_refine_block(demon_net* n, const std::string& scope) {
  const std::string s = scope + "/";
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

  build_flow_block(n, "netFlow1", false);
  build_dm_block(n, "netDM1", false);
  build_flow_block(n, "netFlow2", true);
  build_dm_block(n, "netDM2", true);
  build_refine_block(n, "netRefine");
}

// ---------------------------------------------------------------------------------------------
// weight packing: TF layout -> [tap][cin_buf][cout_pad]
// ---------------------------------------------------------------------------------------------
// transposed conv k4 s2, "VALID then slice 1" == "same" (blocks_original.py:64-74,97-110):
//   out[2y+py, 2x+px] = sum over the two kernel rows/cols of matching parity
//   py = 0: (ky=1, dy=0), (ky=3, dy=-1);   py = 1: (ky=0, dy=+1), (ky=2, dy=0)
const int kDeconvK[2][2] = {{1, 3}, {0, 2}};
const int kDeconvD[2][2] = {{0, -1}, {1, 0}};

void pack_conv(const Layer& l, const HostVar& k, std::vector<float>& out) {
  const int taps = l.kh * l.kw;
  out.assign((size_t)taps * l.cin_buf * l.cout_pad, 0.f);
  for (int t = 0; t < taps; ++t)
    for (int ci = 0; ci < l.cin; ++ci)
      for (int co = 0; co < l.cout; ++co)
        out[((size_t)t * l.cin_buf + ci) * l.cout_pad + co] = k.data[((size_t)t * l.cin + ci) * l.cout + co];
}

void pack_deconv_class(const Layer& l, const HostVar& k, int py, int px, std::vector<float>& out) {
  out.assign((size_t)4 * l.cin_buf * l.cout_pad, 0.f);
  for (int a = 0; a < 2; ++a)
    for (int b = 0; b < 2; ++b) {
      const int ky = kDeconvK[py][a], kx = kDeconvK[px][b];
      const int t = a * 2 + b;
      for (int ci = 0; ci < l.cin; ++ci)
        for (int co = 0; co < l.cout; ++co)
          out[((size_t)t * l.cin_buf + ci) * l.cout_pad + co] = k.data[(((size_t)ky * 4 + kx) * l.cout + co) * l.cin + ci];
    }
}

void pack_dense(const Layer& l, const HostVar& k, std::vector<float>& out) {
  out.assign((size_t)l.cin_buf * l.cout_pad, 0.f);
  for (int i = 0; i < l.cin; ++i) {
    int src = i;
    if (l.dense_nchw_flatten) {  // buffer index i = hw*C + c  <->  TF row c*HW + hw
      const int hw = i / l.dense_c, c = i % l.dense_c;
      src = c * l.dense_hw + hw;
    }
    for (int co = 0; co < l.cout; ++co) out[(size_t)i * l.cout_pad + co] = k.data[(size_t)src * l.cout + co];
  }
}

int upload(demon_net* n, const std::vector<float>& host, float** dev) {
  void* p = nullptr;
  DEMON_CHECK_CUDA(cudaMalloc(&p, host.size() * sizeof(float) + 256));
  n->dev_allocs.push_back(p);
  DEMON_CHECK_CUDA(cudaMemcpy(p, host.data(), host.size() * sizeof(float), cudaMemcpyHostToDevice));
  *dev = (float*)p;
  return DEMON_OK;
}

// ---------------------------------------------------------------------------------------------
// layer execution
// ---------------------------------------------------------------------------------------------
void fill_problem(const Layer& l, int B, ConvProblem& p) {
  memset(&p, 0, sizeof(p));
  p.in = l.in->p + l.in_coff;
  p.in_pitch = l.in->C;
  p.B = B;
  p.Cin = l.cin_buf;
  p.out = l.out->p + l.out_coff;
  p.out_pitch = l.out->C;
  p.Cout = l.cout;
  p.Cout_pad = l.cout_pad;
  p.bias = l.bias_dev;
  p.leaky = l.leaky ? 1 : 0;
  p.scale = l.scale;
  p.scale_stride = l.scale_stride;
  p.osy = p.osx = 1;
}

// DEMON_TC_HALO=0 keeps every tensor-core layer on the per-tap kernel (A/B measurements)
bool use_halo_kernel() {
  const char* e = getenv("DEMON_TC_HALO");
  return !(e && e[0] == '0');
}

// The convolution problem(s) of a layer: 1 for conv / dense, 4 sub-pixel classes for a transposed conv.
int build_problems(const Layer& l, int B, ConvProblem* out) {
  ConvProblem p;
  fill_problem(l, B, p);
  if (l.kind == L_DENSE) {
    p.Hi = p.Wi = p.Ho = p.Wo = p.Hfull = p.Wfull = 1;
    p.in_pitch = l.cin_buf;
    p.out_pitch = l.out->C;
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
    for (int ky = 0; ky < l.kh; ++ky)
      for (int kx = 0; kx < l.kw; ++kx) { p.dy[ky * l.kw + kx] = ky - l.kh / 2; p.dx[ky * l.kw + kx] = kx - l.kw / 2; }
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

int run_layer(const Layer& l, int B, cudaStream_t stream, float* splitk_ws = nullptr, float* tc_ws = nullptr) {
  ConvProblem probs[4];
  const int nclass = build_problems(l, B, probs);
  if (l.use_tc) {
    probs[0].partial = tc_ws;   // scratch of the split-K tensor-core layers (the net's, so two nets in flight do not share it)
    return l.tc.halo_plan ? conv_tc_halo_launch(l.tc, probs, stream) : conv_tc_launch(l.tc, probs, stream);
  }
  for (int c = 0; c < nclass; ++c) {
    if (l.kind == L_DENSE && l.ksplit > 1 && splitk_ws) { probs[c].partial = splitk_ws; probs[c].ksplit = l.ksplit; }
    int rc = conv_simt_launch(probs[c], stream);
    if (rc != DEMON_OK) return rc;
  }
  return DEMON_OK;
}

int run_layer_profiled(demon_net* n, int idx, cudaStream_t stream) {
  const Layer& l = *n->layers[idx];
  static const bool sync_layers = getenv("DEMON_SYNC_LAYERS") && atoi(getenv("DEMON_SYNC_LAYERS")) != 0;   // debugging aid
  if (sync_layers) {
    int rc = run_layer(l, n->B, stream, n->splitk->p, n->tc_scratch);
    cudaError_t e = cudaStreamSynchronize(stream);
    if (rc == DEMON_OK && e != cudaSuccess) return fail(DEMON_E_CUDA, "layer %s: %s", l.name.c_str(), cudaGetErrorString(e));
    return rc;
  }
  if (!n->profiling) return run_layer(l, n->B, stream, n->splitk->p, n->tc_scratch);
  if (n->prof_used + 2 > n->prof_events.size()) {
    const size_t old = n->prof_events.size();
    n->prof_events.resize(old + 1024);
    for (size_t i = old; i < n->prof_events.size(); ++i) DEMON_CHECK_CUDA(cudaEventCreate(&n->prof_events[i]));
  }
  DEMON_CHECK_CUDA(cudaEventRecord(n->prof_events[n->prof_used], stream));
  int rc = run_layer(l, n->B, stream, n->splitk->p, n->tc_scratch);
  DEMON_CHECK_CUDA(cudaEventRecord(n->prof_events[n->prof_used + 1], stream));
  n->prof_layer.push_back(idx);
  n->prof_used += 2;
  return rc;
}

int run_range(demon_net* n, const std::string& first, const std::string& last, cudaStream_t stream) {
  bool on = false;
  for (size_t li = 0; li < n->layers.size(); ++li) {
    auto& l = n->layers[li];
    if (l->name == first) on = true;
    if (on) {
      int rc = run_layer_profiled(n, (int)li, stream);
      if (rc != DEMON_OK) return rc;
    }
    if (l->name == last) {
      if (!on) break;
      return DEMON_OK;
    }
  }
  return fail(DEMON_E_STATE, "run_range: layers %s .. %s not found in order", first.c_str(), last.c_str());
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

int strided_copy(const float* src, float* dst, int N, int P, int C, long sn, long sp, long sc, long dn, long dp, long dc,
                 cudaStream_t stream) {
  const long total = (long)N * P * C;
  if (total == 0) return DEMON_OK;
  long blocks = (total + 255) / 256;
  if (blocks > 132 * 32) blocks = 132 * 32;
  (void)launch_pdl(strided_copy_kernel, dim3((int)blocks), dim3(256), 0, stream, src, dst, N, P, C, sn, sp, sc, dn, dp, dc);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
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

// Flow2 extra inputs (blocks_original.py:155-183): depth_to_flow(inverse_depth, normalize_flow) ->
// zero where |flow| >= 1 or NaN -> warp2d(image2_2, normalized, 'value') -> NHWC12
// [warped(3), flow(2), depth(1), normal(3), 0, 0, 0].  dn2 = [depth, normal] NHWC4, motion [B,8] = rot|trans|scale.
__global__ void __launch_bounds__(256) flow_extra_kernel(const float* __restrict__ dn2, const float* __restrict__ motion,
                                                        const float* __restrict__ image2_2, float* __restrict__ extra, int H, int W,
                                                        int extra_pitch) {
  pdl_launch_dependents();   // common.cuh: programmatic dependent launch
  pdl_wait();
  __shared__ D2FCamera<float> cam;
  const int n = blockIdx.y;
  if (threadIdx.x == 0) {
    const float K[4] = {0.89115971f, 1.18821287f, 0.5f, 0.5f};  // networks_original.py:108
    d2f_camera(cam, K, motion + 8 * n, motion + 8 * n + 3, DEMON_ROT_ANGLEAXIS3, W, H);
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

// DM extra inputs (blocks_original.py:336-364): warp2d(image2_2, flow2) ++ flowconf2 (++ flow_to_depth) -> NHWC8
__global__ void __launch_bounds__(128) dm_extra_kernel(const float* __restrict__ flowconf2, const float* __restrict__ motion_prev,
                                                      const float* __restrict__ image2_2, float* __restrict__ extra, int H, int W,
                                                      int extra_pitch, bool with_depth) {
  pdl_launch_dependents();   // common.cuh: programmatic dependent launch
  pdl_wait();
  __shared__ F2DCamera cam;
  const int n = blockIdx.y;
  if (with_depth && threadIdx.x == 0) {
    const float K[4] = {0.89115971f, 1.18821287f, 0.5f, 0.5f};
    f2d_camera(cam, K, motion_prev + 8 * n, motion_prev + 8 * n + 3, DEMON_ROT_ANGLEAXIS3, W, H);
  }
  __syncthreads();
  const int hw = H * W;
  const int i = blockIdx.x * 128 + threadIdx.x;
  if (i >= hw) return;
  const int y = i / W, x = i - y * W;
  const float4 fc = __ldg(reinterpret_cast<const float4*>(flowconf2) + (size_t)n * hw + i);
  const WarpTap<float> t = warp2d_tap<float>(x, y, fc.x, fc.y, W, H, true);
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
  const float dff = with_depth ? f2d_pixel(fc.x, fc.y, x, y, cam, true, true) : 0.f;
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
  if (data_format == 0) return strided_copy(image_pair, n->img8->p, n->B, P, 6, 6L * P, 1, P, 8L * P, 8, 1, s);
  return strided_copy(image_pair, n->img8->p, n->B, P, 6, 6L * P, 6, 1, 8L * P, 8, 1, s);
}

int import_image2_2(demon_net* n, const float* image2_2, int data_format, cudaStream_t s) {
  const int P = 48 * 64;
  if (data_format == 0) {
    DEMON_CHECK_CUDA(cudaMemcpyAsync(n->i22->p, image2_2, (size_t)n->B * 3 * P * sizeof(float), cudaMemcpyDeviceToDevice, s));
    return DEMON_OK;
  }
  return strided_copy(image2_2, n->i22->p, n->B, P, 3, 3L * P, 3, 1, 3L * P, 1, P, s);
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

// export one NHWC channel slice to the API layout
int export_slice(demon_net* n, const Buf* b, int coff, int C, float* dst, int data_format, cudaStream_t s) {
  if (!dst) return DEMON_OK;
  const int P = b->H * b->W;
  if (data_format == 0) return strided_copy(b->p + coff, dst, n->B, P, C, (long)P * b->C, b->C, 1, (long)C * P, 1, P, s);
  return strided_copy(b->p + coff, dst, n->B, P, C, (long)P * b->C, b->C, 1, (long)C * P, C, 1, s);
}

int export_predictions(demon_net* n, float* flow5, float* flow2, float* depth2, float* normal2, float* rotation, float* translation,
                       int data_format, cudaStream_t s) {
  int rc;
  if ((rc = export_slice(n, n->pf5, 0, 2, flow5, data_format, s))) return rc;
  if ((rc = export_slice(n, n->flowconf2, 0, 2, flow2, data_format, s))) return rc;
  if ((rc = export_slice(n, n->dn2, 0, 1, depth2, data_format, s))) return rc;
  if ((rc = export_slice(n, n->dn2, 1, 3, normal2, data_format, s))) return rc;
  if (rotation && (rc = strided_copy(n->motion->p, rotation, n->B, 1, 3, 8, 0, 1, 3, 0, 1, s))) return rc;
  if (translation && (rc = strided_copy(n->motion->p + 3, translation, n->B, 1, 3, 8, 0, 1, 3, 0, 1, s))) return rc;
  return DEMON_OK;
}

// flow block, everything after the trunk's conv2 (blocks_original.py:190-235)
// `head`: run conv1 / conv2 (false when the pipeline has hoisted them out of the iteration loop)
int run_flow_block(demon_net* n, const std::string& scope, bool iterative, cudaStream_t s, bool head = true) {
  const std::string p = scope + "/";
  int rc;
  if (head && (rc = run_range(n, p + "conv1y", p + "conv2x", s))) return rc;
  if (iterative) {
    (void)launch_pdl(flow_extra_kernel, dim3(dim3(ceil_div(48 * 64, 256), n->B)), dim3(256), 0, s, n->dn2->p, n->motion->p, n->i22->p, n->extra_in->p, 48, 64, n->extra_in->C);
    DEMON_LAUNCH_CHECK();
    if ((rc = run_range(n, p + "conv2_extra_inputsy", p + "conv2_extra_inputsx", s))) return rc;
  }
  return run_range(n, p + "conv2_1y", p + "predict_flow2/conv2", s);
}

int run_dm_block(demon_net* n, const std::string& scope, bool iterative, cudaStream_t s, bool head = true) {
  const std::string p = scope + "/";
  int rc;
  if (head && (rc = run_range(n, p + "conv1y", p + "conv2x", s))) return rc;
  // the previous motion is still in n->motion here: this block's motion_fc3 overwrites it later
  (void)launch_pdl(dm_extra_kernel, dim3(dim3(ceil_div(48 * 64, 128), n->B)), dim3(128), 0, s, n->flowconf2->p, n->motion->p, n->i22->p, n->extra_in->p, 48, 64,
                                                                   n->extra_in->C, iterative);
  DEMON_LAUNCH_CHECK();
  return run_range(n, p + "conv2_extra_inputsy", p + "predict_depthnormal2/conv2", s);
}

int run_refine_block(demon_net* n, const float* image1, long img_sn, long img_sp, long img_sc, const float* depth, long d_sn, long d_sp,
                     int dh, int dw, float* depth0, cudaStream_t s) {
  const long total = (long)n->B * n->RH * n->RW;
  long blocks = (total + 255) / 256;
  if (blocks > 132 * 32) blocks = 132 * 32;
  (void)launch_pdl(refine_input_kernel, dim3((int)blocks), dim3(256), 0, s, image1, img_sn, img_sp, img_sc, depth, d_sn, d_sp, n->rin->p, n->B, n->RH, n->RW, dh, dw);
  DEMON_LAUNCH_CHECK();
  // the last layer writes straight into the caller's output (C = 1: NHWC == NCHW)
  Layer* last = n->by_name["netRefine/predict_depth0/conv2"];
  Buf out = *n->rdepth0;
  if (depth0) out.p = depth0;
  Buf* saved = last->out;
  last->out = &out;
  int rc = run_range(n, "netRefine/conv0", "netRefine/predict_depth0/conv2", s);
  last->out = saved;
  return rc;
}

}  // namespace
}  // namespace demon

// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------
extern "C" {

int demon_net_create(demon_net** out, int batch, int refine_h, int refine_w, int precision) {
  DEMON_REQUIRE(out, "demon_net_create: null out");
  DEMON_REQUIRE(batch >= 1 && batch <= 4096, "demon_net_create: batch %d", batch);
  DEMON_REQUIRE(refine_h >= 4 && refine_w >= 4 && refine_h % 4 == 0 && refine_w % 4 == 0, "demon_net_create: refine size %dx%d must be a multiple of 4", refine_h, refine_w);
  DEMON_REQUIRE(precision >= 0 && precision <= 2, "demon_net_create: precision %d", precision);
  std::unique_ptr<demon_net> n(new demon_net());
  n->B = batch; n->RH = refine_h; n->RW = refine_w; n->precision = precision;
  DEMON_CHECK_CUDA(cudaGetDevice(&n->device));
  build_plan(n.get());
  void* p = nullptr;
  DEMON_CHECK_CUDA(cudaMalloc(&p, n->ws_floats * sizeof(float)));
  n->ws = (float*)p;
  DEMON_CHECK_CUDA(cudaMemset(p, 0, n->ws_floats * sizeof(float)));
  for (auto& b : n->bufs) b->p = n->ws + b->offset;
  n->by_name["netDM1/predict_depthnormal2/conv2"]->scale = n->motion->p + 6;
  n->by_name["netDM2/predict_depthnormal2/conv2"]->scale = n->motion->p + 6;
  *out = n.release();
  return DEMON_OK;
}

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
  HostVar& hv = n->host_vars[nm];
  hv.data.assign(data, data + numel);
  hv.shape.assign(shape, shape + rank);
  return DEMON_OK;
}

int demon_net_finalize(demon_net* n) {
  DEMON_REQUIRE(n, "demon_net_finalize: null net");
  if (n->finalized) return DEMON_OK;
  for (auto& nm : n->var_names)
    if (!n->host_vars.count(nm)) return fail(DEMON_E_STATE, "demon_net_finalize: variable %s was not set", nm.c_str());
  std::vector<float> packed, bias;
  for (auto& lp : n->layers) {
    Layer& l = *lp;
    const HostVar& k = n->host_vars[l.name + "/kernel"];
    const HostVar& b = n->host_vars[l.name + "/bias"];
    bias.assign(l.cout_pad, 0.f);
    for (int i = 0; i < l.cout; ++i) bias[i] = b.data[i];
    int rc;
    if ((rc = upload(n, bias, &l.bias_dev))) return rc;
    if (l.kind == L_CONV) {
      pack_conv(l, k, packed);
      if ((rc = upload(n, packed, &l.w_dev[0]))) return rc;
    } else if (l.kind == L_DENSE) {
      pack_dense(l, k, packed);
      if ((rc = upload(n, packed, &l.w_dev[0]))) return rc;
    } else {
      for (int py = 0; py < 2; ++py)
        for (int px = 0; px < 2; ++px) {
          pack_deconv_class(l, k, py, px, packed);
          if ((rc = upload(n, packed, &l.w_dev[py * 2 + px]))) return rc;
        }
    }
    // tensor-core eligibility and packing
    if (n->precision != DEMON_PREC_FP32_SIMT && l.kind != L_DENSE) {
      ConvProblem probs[4];
      const int nclass = build_problems(l, n->B, probs);
      bool all = true;
      for (int c = 0; c < nclass; ++c) all = all && tc_layer_supported(probs[c]);
      const bool halo = use_halo_kernel() && tc_halo_supported(probs, nclass);   // also takes the 8-channel layers
      if (all || halo) {
        std::vector<float> cls_w[4];
        const float* ptrs[4] = {nullptr, nullptr, nullptr, nullptr};
        for (int c = 0; c < nclass; ++c) {
          if (l.kind == L_CONV) pack_conv(l, k, cls_w[c]); else pack_deconv_class(l, k, c / 2, c % 2, cls_w[c]);
          ptrs[c] = cls_w[c].data();
        }
        if (halo) rc = tc_halo_prepare(l.tc, probs, ptrs, nclass, n->precision);
        else rc = tc_layer_prepare(l.tc, probs, ptrs, nclass, n->precision);
        if (rc) return rc;
        l.use_tc = true;
      }
    }
  }
  // scratch of the split-K tensor-core layers: the largest need, owned by the net
  size_t need = 0;
  for (auto& lp : n->layers)
    if (lp->use_tc) need = std::max(need, lp->tc.splitk_bytes);
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
int demon_net_layer_uses_tensor_cores(const demon_net* n, const char* name) {
  if (!n || !name) return 0;
  auto it = n->by_name.find(name);
  return (it != n->by_name.end() && it->second->use_tc) ? 1 : 0;
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
  if (launches_per_call) *launches_per_call = n->layers[i]->use_tc ? 1 : (n->layers[i]->kind == L_DECONV ? 4 : (n->layers[i]->ksplit > 1 ? 2 : 1));
  // kernel family: 0 conv_simt_kernel, 2 conv_tc_halo_kernel (halo), 3 conv_tc_halo_kernel (per tap)
  if (uses_tc) *uses_tc = !n->layers[i]->use_tc ? 0 : (!n->layers[i]->tc.halo_plan ? 1 : (n->layers[i]->tc.per_tap ? 3 : 2));
  return DEMON_OK;
}

#define REQUIRE_READY(n)                                                         \
  do {                                                                           \
    DEMON_REQUIRE(n, "null net");                                                \
    if (!(n)->finalized) return fail(DEMON_E_STATE, "forward before demon_net_finalize"); \
    int _dev = -1;                                                               \
    cudaGetDevice(&_dev);                                                        \
    if (_dev != (n)->device)                                                     \
      return fail(DEMON_E_STATE, "net handle belongs to CUDA device %d but device %d is current", (n)->device, _dev); \
  } while (0)

int demon_bootstrap_forward(demon_net* n, const float* image_pair, const float* image2_2, float* flow5, float* flow2, float* depth2,
                            float* normal2, float* rotation, float* translation, int data_format, void* stream) {
  REQUIRE_READY(n);
  DEMON_REQUIRE(image_pair && image2_2, "bootstrap: null input");
  DEMON_REQUIRE(data_format == 0 || data_format == 1, "bootstrap: data_format %d", data_format);
  cudaStream_t s = (cudaStream_t)stream;
  int rc;
  if ((rc = import_image_pair(n, image_pair, data_format, s))) return rc;
  if ((rc = import_image2_2(n, image2_2, data_format, s))) return rc;
  if ((rc = run_flow_block(n, "netFlow1", false, s))) return rc;
  if ((rc = run_dm_block(n, "netDM1", false, s))) return rc;
  return export_predictions(n, flow5, flow2, depth2, normal2, rotation, translation, data_format, s);
}

int demon_iterative_forward(demon_net* n, const float* image_pair, const float* image2_2, const float* depth2_in, const float* normal2_in,
                            const float* rotation_in, const float* translation_in, float* flow5, float* flow2, float* depth2,
                            float* normal2, float* rotation, float* translation, int data_format, void* stream) {
  REQUIRE_READY(n);
  DEMON_REQUIRE(image_pair && image2_2 && depth2_in && normal2_in && rotation_in && translation_in, "iterative: null input");
  DEMON_REQUIRE(data_format == 0 || data_format == 1, "iterative: data_format %d", data_format);
  cudaStream_t s = (cudaStream_t)stream;
  const int P = 48 * 64;
  int rc;
  if ((rc = import_image_pair(n, image_pair, data_format, s))) return rc;
  if ((rc = import_image2_2(n, image2_2, data_format, s))) return rc;
  // previous predictions -> dn2 (NHWC4) and motion
  if (data_format == 0) {
    if ((rc = strided_copy(depth2_in, n->dn2->p, n->B, P, 1, P, 1, 0, 4L * P, 4, 1, s))) return rc;
    if ((rc = strided_copy(normal2_in, n->dn2->p + 1, n->B, P, 3, 3L * P, 1, P, 4L * P, 4, 1, s))) return rc;
  } else {
    if ((rc = strided_copy(depth2_in, n->dn2->p, n->B, P, 1, P, 1, 0, 4L * P, 4, 1, s))) return rc;
    if ((rc = strided_copy(normal2_in, n->dn2->p + 1, n->B, P, 3, 3L * P, 3, 1, 4L * P, 4, 1, s))) return rc;
  }
  if ((rc = strided_copy(rotation_in, n->motion->p, n->B, 1, 3, 3, 0, 1, 8, 0, 1, s))) return rc;
  if ((rc = strided_copy(translation_in, n->motion->p + 3, n->B, 1, 3, 3, 0, 1, 8, 0, 1, s))) return rc;
  if ((rc = run_flow_block(n, "netFlow2", true, s))) return rc;
  if ((rc = run_dm_block(n, "netDM2", true, s))) return rc;
  return export_predictions(n, flow5, flow2, depth2, normal2, rotation, translation, data_format, s);
}

int demon_refine_forward(demon_net* n, const float* image1, const float* depth2, float* depth0, int data_format, void* stream) {
  REQUIRE_READY(n);
  DEMON_REQUIRE(image1 && depth2 && depth0, "refine: null pointer");
  DEMON_REQUIRE(data_format == 0 || data_format == 1, "refine: data_format %d", data_format);
  const long P = (long)n->RH * n->RW;
  const int dh = n->RH / 4, dw = n->RW / 4;
  if (data_format == 0)
    return run_refine_block(n, image1, 3 * P, 1, P, depth2, (long)dh * dw, 1, dh, dw, depth0, (cudaStream_t)stream);
  return run_refine_block(n, image1, 3 * P, 3, 1, depth2, (long)dh * dw, 1, dh, dw, depth0, (cudaStream_t)stream);
}

// Input of the fused pipeline: fp32 NCHW (image_pair [B,6,192,256], image2_2 [B,3,48,64] or null) or uint8
// (images [B,2,192,256,3], image2_2 [B,48,64,3] or null).
struct PipelineInput {
  const float* image_pair = nullptr;
  const float* image2_2 = nullptr;
  const unsigned char* images_u8 = nullptr;
  const unsigned char* image2_2_u8 = nullptr;
};

static int pipeline_body(demon_net* n, const PipelineInput& in, int iterations, float* depth0, float* rotation,
                         float* translation, float* flow2, float* depth2, float* normal2, cudaStream_t s) {
  int rc;
  const long P = 192L * 256;
  if (in.images_u8) {
    // img8 straight from the bytes; image 2's planes go to c1y (free until conv1y runs) for the median pair
    float* planes2 = in.image2_2_u8 ? nullptr : n->c1y->p;
    long blocks = ((long)n->B * P + 255) / 256;
    if (blocks > 132 * 32) blocks = 132 * 32;
    (void)launch_pdl(u8_import_kernel, dim3((int)blocks), dim3(256), 0, s, in.images_u8, n->img8->p, planes2, n->B, (int)P);
    DEMON_LAUNCH_CHECK();
    if (in.image2_2_u8) {
      long b2 = ((long)n->B * 48 * 64 + 255) / 256;
      (void)launch_pdl(u8_planes_kernel, dim3((int)b2), dim3(256), 0, s, in.image2_2_u8, n->i22->p, n->B, 48 * 64);
      DEMON_LAUNCH_CHECK();
    } else if ((rc = median_image2_2(n, planes2, 3 * P, s))) {
      return rc;
    }
  } else {
    if ((rc = import_image_pair(n, in.image_pair, 0, s))) return rc;
    if (in.image2_2) {
      if ((rc = import_image2_2(n, in.image2_2, 0, s))) return rc;
    } else {
      if ((rc = median_image2_2(n, in.image_pair + 3 * P, 6 * P, s))) return rc;
    }
  }
  if ((rc = run_flow_block(n, "netFlow1", false, s))) return rc;
  if ((rc = run_dm_block(n, "netDM1", false, s))) return rc;
  // conv1 / conv2 of netFlow2 and netDM2 read only the image pair and fixed weights: once per call instead of once per
  // iteration (bit identical; 2 x 2 x 221.7 MMAC per pair less to execute at three iterations)
  if (iterations > 0) {
    if ((rc = run_range(n, "netFlow2/conv1y", "netFlow2/conv2x", s))) return rc;
    if ((rc = run_range(n, "netDM2/conv1y", "netDM2/conv2x", s))) return rc;
  }
  for (int it = 0; it < iterations; ++it) {
    if ((rc = run_flow_block(n, "netFlow2", true, s, false))) return rc;
    if ((rc = run_dm_block(n, "netDM2", true, s, false))) return rc;
  }
  if ((rc = export_predictions(n, nullptr, flow2, depth2, normal2, rotation, translation, 0, s))) return rc;
  // image1 for the refinement block is read back from img8 (NHWC8: the first three channels), whatever the input kind
  return run_refine_block(n, n->img8->p, 8 * P, 8, 1, n->dn2->p, 4L * 48 * 64, 4, 48, 64, depth0, s);
}

static int pipeline_forward_impl(demon_net* n, const PipelineInput& in, int iterations, float* depth0, float* rotation, float* translation,
                                 float* flow2, float* depth2, float* normal2, void* stream);

int demon_pipeline_forward(demon_net* n, const float* image_pair, const float* image2_2, int iterations, float* depth0, float* rotation,
                           float* translation, float* flow2, float* depth2, float* normal2, void* stream) {
  REQUIRE_READY(n);
  DEMON_REQUIRE(image_pair, "pipeline: null image_pair");
  PipelineInput in;
  in.image_pair = image_pair; in.image2_2 = image2_2;
  return pipeline_forward_impl(n, in, iterations, depth0, rotation, translation, flow2, depth2, normal2, stream);
}

int demon_pipeline_forward_u8(demon_net* n, const uint8_t* images, const uint8_t* image2_2, int iterations, float* depth0, float* rotation,
                              float* translation, float* flow2, float* depth2, float* normal2, void* stream) {
  REQUIRE_READY(n);
  DEMON_REQUIRE(images, "pipeline_u8: null images");
  PipelineInput in;
  in.images_u8 = images; in.image2_2_u8 = image2_2;
  return pipeline_forward_impl(n, in, iterations, depth0, rotation, translation, flow2, depth2, normal2, stream);
}

static int pipeline_forward_impl(demon_net* n, const PipelineInput& in, int iterations, float* depth0, float* rotation, float* translation,
                                 float* flow2, float* depth2, float* normal2, void* stream) {
  DEMON_REQUIRE(iterations >= 0 && iterations <= 7, "pipeline: iterations %d", iterations);
  DEMON_REQUIRE(n->RH == 192 && n->RW == 256, "pipeline: net was created with a %dx%d refinement block", n->RH, n->RW);
  cudaStream_t s = (cudaStream_t)stream;
  // The call is one CUDA graph per distinct set of pointer arguments (DEMON_GRAPH=0 disables): the first call with a new
  // set runs eagerly, the second captures, later ones replay.  Not used while per-layer profiling is on or when the
  // caller is itself capturing this stream.
  static const bool graphs_on = []() { const char* e = getenv("DEMON_GRAPH"); return !(e && e[0] == '0'); }();
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(s, &cap);
  if (graphs_on && !n->profiling && cap == cudaStreamCaptureStatusNone) {
    const std::vector<const void*> key = {in.image_pair, in.image2_2, in.images_u8, in.image2_2_u8, depth0, rotation, translation, flow2, depth2,
                                          normal2, reinterpret_cast<const void*>((intptr_t)iterations)};
    for (auto& g : n->graphs)
      if (g.key == key) {
        if (g.exec == nullptr) {   // second call: capture
          cudaGraph_t graph = nullptr;
          const int64_t l0 = g_launch_count.load();
          if (!n->cap_stream) DEMON_CHECK_CUDA(cudaStreamCreateWithFlags(&n->cap_stream, cudaStreamNonBlocking));
          DEMON_CHECK_CUDA(cudaStreamBeginCapture(n->cap_stream, cudaStreamCaptureModeThreadLocal));
          int rc = pipeline_body(n, in, iterations, depth0, rotation, translation, flow2, depth2, normal2, n->cap_stream);
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
        n->pipeline_launches[iterations] = g.launches;
        return DEMON_OK;
      }
    if (n->graphs.size() >= 32) {   // evict the oldest entry
      if (n->graphs.front().exec) cudaGraphExecDestroy(n->graphs.front().exec);
      n->graphs.erase(n->graphs.begin());
    }
    n->graphs.push_back({key, nullptr, 0});
  }
  const int64_t launches0 = g_launch_count.load();
  int rc = pipeline_body(n, in, iterations, depth0, rotation, translation, flow2, depth2, normal2, s);
  if (rc) return rc;
  n->pipeline_launches[iterations] = (int)(g_launch_count.load() - launches0);
  return DEMON_OK;
}

static int pipeline_host(demon_net* n, const void* images_host, const void* image2_2_host, bool u8, int iterations, float* depth0_host,
                         float* rotation_host, float* translation_host, void* stream, bool sync);

int demon_pipeline_forward_host(demon_net* n, const float* image_pair_host, const float* image2_2_host, int iterations, float* depth0_host,
                                float* rotation_host, float* translation_host, void* stream) {
  return pipeline_host(n, image_pair_host, image2_2_host, false, iterations, depth0_host, rotation_host, translation_host, stream, true);
}

int demon_pipeline_forward_host_async(demon_net* n, const float* image_pair_host, const float* image2_2_host, int iterations,
                                      float* depth0_host, float* rotation_host, float* translation_host, void* stream) {
  return pipeline_host(n, image_pair_host, image2_2_host, false, iterations, depth0_host, rotation_host, translation_host, stream, false);
}

int demon_pipeline_forward_host_u8(demon_net* n, const uint8_t* images_host, const uint8_t* image2_2_host, int iterations, float* depth0_host,
                                   float* rotation_host, float* translation_host, void* stream) {
  return pipeline_host(n, images_host, image2_2_host, true, iterations, depth0_host, rotation_host, translation_host, stream, true);
}

int demon_pipeline_forward_host_u8_async(demon_net* n, const uint8_t* images_host, const uint8_t* image2_2_host, int iterations,
                                         float* depth0_host, float* rotation_host, float* translation_host, void* stream) {
  return pipeline_host(n, images_host, image2_2_host, true, iterations, depth0_host, rotation_host, translation_host, stream, false);
}

static int pipeline_host(demon_net* n, const void* images_host, const void* image2_2_host, bool u8, int iterations, float* depth0_host,
                         float* rotation_host, float* translation_host, void* stream, bool sync) {
  REQUIRE_READY(n);
  DEMON_REQUIRE(images_host && depth0_host, "pipeline_host: null pointer");
  cudaStream_t s = (cudaStream_t)stream;
  // staging lives in buffers that are free at the respective moments:
  //   images     -> concat0 ([B,192,256,64]; only written by the refinement block, which reads image1 back from img8)
  //   image2_2   -> pd0a    (only written by netRefine/predict_depth0/conv1)
  const size_t px = (size_t)n->B * 192 * 256;
  const size_t ip_bytes = u8 ? px * 6 : px * 6 * sizeof(float);
  const size_t i22_bytes = (size_t)n->B * 3 * 48 * 64 * (u8 ? 1 : sizeof(float));
  void* ip_dev = n->concat0->p;
  void* i22_dev = n->pd0a->p;
  DEMON_CHECK_CUDA(cudaMemcpyAsync(ip_dev, images_host, ip_bytes, cudaMemcpyHostToDevice, s));
  if (image2_2_host) DEMON_CHECK_CUDA(cudaMemcpyAsync(i22_dev, image2_2_host, i22_bytes, cudaMemcpyHostToDevice, s));
  float* out_dev = n->rdepth0->p;
  float* rt_dev = n->fc1->p;                 // 6 floats per sample, fc1 is free after the last DM block
  PipelineInput in;
  if (u8) { in.images_u8 = static_cast<const unsigned char*>(ip_dev); in.image2_2_u8 = image2_2_host ? static_cast<const unsigned char*>(i22_dev) : nullptr; }
  else { in.image_pair = static_cast<const float*>(ip_dev); in.image2_2 = image2_2_host ? static_cast<const float*>(i22_dev) : nullptr; }
  int rc = pipeline_forward_impl(n, in, iterations, out_dev, rotation_host ? rt_dev : nullptr, translation_host ? rt_dev + 3 * n->B : nullptr,
                                 nullptr, nullptr, nullptr, stream);
  if (rc) return rc;
  DEMON_CHECK_CUDA(cudaMemcpyAsync(depth0_host, out_dev, (size_t)n->B * 192 * 256 * sizeof(float), cudaMemcpyDeviceToHost, s));
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

// debug: which kernel family / plan every layer of the net got (one line per layer)
int demon_debug_describe_layers(const demon_net* n, char* buf, int buflen) {
  DEMON_REQUIRE(n && buf && buflen > 0, "describe: null");
  int off = 0;
  for (auto& lp : n->layers) {
    const Layer& l = *lp;
    if (off >= buflen - 256) break;
    off += snprintf(buf + off, buflen - off, "%-40s ", l.name.c_str());
    if (l.kind == L_DENSE) { off += snprintf(buf + off, buflen - off, "dense simt\n"); continue; }
    ConvProblem probs[4];
    const int nclass = build_problems(l, n->B, probs);
    for (int c = 0; c < nclass; ++c) { probs[c].in = (const float*)0x1000; probs[c].out = (float*)0x1000; }
    if (n->precision != DEMON_PREC_FP32_SIMT && use_halo_kernel() && tc_halo_supported(probs, nclass))
      off += tc_halo_describe(probs, nclass, n->precision == DEMON_PREC_TF32 ? 1 : 3, buf + off, buflen - off);
    else {
      bool all = n->precision != DEMON_PREC_FP32_SIMT;
      for (int c = 0; c < nclass; ++c) all = all && tc_layer_supported(probs[c]);
      off += snprintf(buf + off, buflen - off, all ? "conv_tc_kernel" : "simt");
    }
    off += snprintf(buf + off, buflen - off, "\n");
  }
  return off;
}

// debug, no device needed: the plan of one convolution shape ([B,H,W,Cin] NHWC, channel pitches given)
int demon_debug_describe_conv(int B, int H, int W, int Cin, int in_pitch, int Cout, int out_pitch, int kh, int kw, int sy, int sx, int deconv,
                              int precision, char* buf, int buflen) {
  DEMON_REQUIRE(buf && buflen > 0, "describe: null");
  Buf bi, bo;
  bi.p = (float*)0x10000; bi.H = H; bi.W = W; bi.C = in_pitch;
  Layer l;
  l.name = "shape"; l.kind = deconv ? L_DECONV : L_CONV; l.in = &bi; l.cin = Cin; l.cin_buf = (Cin + 3) / 4 * 4; l.out = &bo; l.cout = Cout;
  l.cout_pad = (Cout + 3) / 4 * 4; l.kh = kh; l.kw = kw; l.sy = sy; l.sx = sx;
  bo.p = (float*)0x10000; bo.C = out_pitch;
  if (deconv) { bo.H = 2 * H; bo.W = 2 * W; } else { bo.H = ceil_div(H, sy); bo.W = ceil_div(W, sx); }
  ConvProblem probs[4];
  const int nclass = build_problems(l, B, probs);
  if (precision != DEMON_PREC_FP32_SIMT && use_halo_kernel() && tc_halo_supported(probs, nclass))
    return tc_halo_describe(probs, nclass, precision == DEMON_PREC_TF32 ? 1 : 3, buf, buflen);
  bool all = precision != DEMON_PREC_FP32_SIMT;
  for (int c = 0; c < nclass; ++c) all = all && tc_layer_supported(probs[c]);
  return snprintf(buf, buflen, all ? "conv_tc_kernel" : "simt");
}

// ---- standalone convolution entries (tests) ---------------------------------------------------
static double g_last_conv_ms = -1.0;
double demon_debug_last_conv_ms(void) { return g_last_conv_ms; }

static int standalone_conv(const float* in, float* out, int B, int H, int W, int Cin, int Cout, int kh, int kw, int sy, int sx,
                           const float* kernel_host, const float* bias_host, int leaky, int precision, bool deconv, void* stream) {
  DEMON_REQUIRE(in && out && kernel_host && bias_host, "conv: null pointer");
  DEMON_REQUIRE(Cin % 4 == 0, "conv test entry: Cin must be a multiple of 4");
  demon_net tmp;
  tmp.B = B;
  Buf bi, bo;
  bi.p = const_cast<float*>(in); bi.H = H; bi.W = W; bi.C = Cin;
  Layer l;
  l.name = "standalone"; l.kind = deconv ? L_DECONV : L_CONV; l.in = &bi; l.cin = Cin; l.cin_buf = Cin; l.out = &bo; l.cout = Cout;
  l.cout_pad = (Cout + 3) / 4 * 4; l.kh = kh; l.kw = kw; l.sy = sy; l.sx = sx; l.leaky = leaky != 0;
  bo.p = out; bo.C = Cout;
  if (deconv) { bo.H = 2 * H; bo.W = 2 * W; } else { bo.H = ceil_div(H, sy); bo.W = ceil_div(W, sx); }
  HostVar k;
  k.data.assign(kernel_host, kernel_host + (size_t)kh * kw * Cin * Cout);
  std::vector<float> packed, bias(l.cout_pad, 0.f);
  for (int i = 0; i < Cout; ++i) bias[i] = bias_host[i];
  int rc;
  if ((rc = upload(&tmp, bias, &l.bias_dev))) return rc;
  const int nclass = deconv ? 4 : 1;
  std::vector<float> cls_w[4];
  const float* ptrs[4] = {nullptr, nullptr, nullptr, nullptr};
  for (int c = 0; c < nclass; ++c) {
    if (deconv) pack_deconv_class(l, k, c / 2, c % 2, cls_w[c]); else pack_conv(l, k, cls_w[c]);
    ptrs[c] = cls_w[c].data();
    if ((rc = upload(&tmp, cls_w[c], &l.w_dev[c]))) return rc;
  }
  if (precision != DEMON_PREC_FP32_SIMT) {
    ConvProblem probs[4];
    build_problems(l, B, probs);
    bool all = true;
    for (int c = 0; c < nclass; ++c) all = all && tc_layer_supported(probs[c]);
    const bool halo = use_halo_kernel() && tc_halo_supported(probs, nclass);
    if (!all && !halo) {
      for (void* q : tmp.dev_allocs) cudaFree(q);
      return fail(DEMON_E_INVALID, "conv test entry: shape not supported by the tensor-core path");
    }
    if (halo) rc = tc_halo_prepare(l.tc, probs, ptrs, nclass, precision);
    else rc = tc_layer_prepare(l.tc, probs, ptrs, nclass, precision);
    if (rc) return rc;
    l.use_tc = true;
  }
  float* tc_ws = nullptr;
  if (l.use_tc && l.tc.splitk_bytes) {
    void* q = nullptr;
    if (cudaMalloc(&q, l.tc.splitk_bytes) != cudaSuccess) return fail(DEMON_E_CUDA, "conv test entry: scratch allocation failed");
    tmp.dev_allocs.push_back(q);
    tc_ws = static_cast<float*>(q);
  }
  cudaEvent_t ev0, ev1;
  cudaEventCreate(&ev0); cudaEventCreate(&ev1);
  cudaEventRecord(ev0, (cudaStream_t)stream);
  rc = run_layer(l, B, (cudaStream_t)stream, nullptr, tc_ws);
  cudaEventRecord(ev1, (cudaStream_t)stream);
  cudaError_t e = cudaStreamSynchronize((cudaStream_t)stream);
  float ms = -1.f;
  if (e == cudaSuccess && cudaEventElapsedTime(&ms, ev0, ev1) == cudaSuccess) g_last_conv_ms = ms;
  cudaEventDestroy(ev0); cudaEventDestroy(ev1);
  for (void* q : tmp.dev_allocs) cudaFree(q);
  tc_layer_free(l.tc);
  if (rc) return rc;
  if (e != cudaSuccess) return fail(DEMON_E_CUDA, "conv test entry: %s", cudaGetErrorString(e));
  return DEMON_OK;
}

int demon_conv2d_nhwc(const float* in, float* out, int B, int H, int W, int Cin, int Cout, int kh, int kw, int sy, int sx,
                      const float* kernel_host, const float* bias_host, int leaky, int precision, void* stream) {
  DEMON_REQUIRE(kh >= 1 && kw >= 1 && kh * kw <= kMaxTaps && (kh & 1) && (kw & 1), "conv: kernel %dx%d", kh, kw);
  DEMON_REQUIRE(sy >= 1 && sx >= 1, "conv: stride");
  return standalone_conv(in, out, B, H, W, Cin, Cout, kh, kw, sy, sx, kernel_host, bias_host, leaky, precision, false, stream);
}

int demon_deconv4x4s2_nhwc(const float* in, float* out, int B, int H, int W, int Cin, int Cout, const float* kernel_host,
                           const float* bias_host, int leaky, int precision, void* stream) {
  return standalone_conv(in, out, B, H, W, Cin, Cout, 4, 4, 2, 2, kernel_host, bias_host, leaky, precision, true, stream);
}

}  // extern "C"
