// Engine: builds the Faster R-CNN (slim resnet_v1_{50,101} + RPN + RCNN) or SSD
// (truncated VGG16 + extras + multibox heads) inference plan from the merged
// YAML config, owns weights + workspace on one GPU, and runs the forward pass
// as a fixed sequence of the kernels in conv.cu / elementwise.cu / roi.cu /
// postproc.cu on one stream.  Exposes the C ABI of include/luminoth_b200.h.
//
// Reference structure restated here (not ported):
//   models/fasterrcnn/fasterrcnn.py:70-156   FasterRCNN._build
//   models/base/truncated_base_network.py:18-169 endpoint / R101 block4 tail
//   models/fasterrcnn/rpn.py:136-180, rcnn.py:148-253
//   models/ssd/ssd.py:37-195, models/ssd/feature_extractor.py:39-132
#include "../../include/luminoth_b200.h"
#include "conv.cuh"
#include "ops.cuh"
#include "json.hpp"

#include <algorithm>
#include <array>
#include <cmath>
#include <cstring>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <tuple>
#include <vector>

using namespace lumi;

namespace {

struct HostTensor {
  std::vector<float> v;
  std::vector<int64_t> shape;
};

struct WeightSpec {
  std::string name;
  std::vector<int64_t> shape;
};

// A conv's padding: TF VALID, TF SAME, or slim conv2d_same (explicit pad + VALID when stride > 1)
enum Padding { PAD_VALID, PAD_SAME, PAD_CONV2D_SAME };

// What a layer record builds: a conv with folded slim batch norm; a conv or fc with biases, where several scopes fuse
// along C_out; a resnet_v2 `preact` batch norm; SSD's L2-norm gamma; or a tensor-core form of the conv of another
// record, from whose weights it is built (it reads no variables of its own)
enum LayerKind { LK_CONV_BN, LK_CONV_BIAS, LK_PREACT, LK_GAMMA, LK_STEM_S2D, LK_CONV1_1_PACK };
// Variable names of a bias conv: slim weights / biases, Sonnet w / b, or Sonnet Linear w / b with [C_in, C_out] weights
enum Naming { NM_SLIM, NM_SONNET, NM_LINEAR };

// One record of the engine's layer table (build_net): the variables a layer reads and how it runs
struct Layer {
  std::string key;                    // engine key: run_conv's name of the layer, or the dev_vecs prefix
  int kind = LK_CONV_BIAS, naming = NM_SLIM;
  std::vector<std::string> scopes;    // variable scopes
  int kh = 1, kw = 1, cin = 0;        // cin: the channels of a preact or gamma vector
  std::vector<int> couts;             // per scope
  int stride = 1, rate = 1, act = ACT_NONE;
  int padding = PAD_VALID;            // the derived layers read staging buffers that carry their padding
  ConvLayer conv;                     // the uploaded conv (lumi_finalize)
};

struct Arena {
  uint8_t* base = nullptr;
  size_t cap = 0, off = 0;
  void* alloc(size_t bytes, bool dry) {
    size_t a = (off + 1023) & ~(size_t)1023;
    off = a + bytes;
    if (dry) return nullptr;
    if (off > cap) throw Error(LUMI_ESTATE, "arena overflow (internal)");
    return base + a;
  }
};

struct Tap {
  const void* ptr = nullptr;   // device
  int kind = 0;                // 0 f32, 1 Act, 2 int32
  Act act;
  int64_t shape[4] = {0, 0, 0, 0};
};

// Faster R-CNN base networks (truncated_base_network.py:8-16): units per block; `preact` marks slim resnet_v2, the
// pre-activation ResNet (each unit starts with relu(BN(x)); conv3 and the projection shortcut carry biases)
struct ResnetArch { const char* name; int units[4]; bool preact; };
const ResnetArch RESNETS[6] = {
    {"resnet_v1_50", {3, 4, 6, 3}, false}, {"resnet_v1_101", {3, 4, 23, 3}, false},
    {"resnet_v1_152", {3, 8, 36, 3}, false}, {"resnet_v2_50", {3, 4, 6, 3}, true},
    {"resnet_v2_101", {3, 4, 23, 3}, true}, {"resnet_v2_152", {3, 8, 36, 3}, true}};
const int BASE_DEPTH[4] = {64, 128, 256, 512};
const int BLOCK_STRIDE[4] = {2, 2, 2, 1};
const float RGB_MEANS[3] = {123.68f, 116.78f, 103.94f};

// The part of a bottleneck unit a Faster R-CNN endpoint stops at: one of its collected convs, or the unit's output
enum UnitPart { UP_CONV1, UP_CONV2, UP_CONV3, UP_SHORTCUT, UP_UNIT };

// model.base_network.endpoint (truncated_base_network.py:18-37, 146-169): the trunk output that feeds the RPN and
// the ROI pool.  block -1 is the stem conv; a block endpoint is its last unit's output.
struct Endpoint {
  std::string name = "block3";
  int block = 0, unit = 0, part = UP_UNIT;
  int depth = 0;
  int stride = 0;               // feature stride of the endpoint map: the anchor grid is ceil(image size / stride)
};

}  // namespace

struct lumi_engine {
  std::string last_error;
  JVal cfg;
  int device = 0, max_batch = 1, max_h = 0, max_w = 0;
  cudaStream_t stream = nullptr;
  bool finalized = false;
  int conv_impl = 1;
  int launches = 0;
  bool debug_taps = false;      // materialise intermediates that the fused path skips (roi_pool)

  std::string type, arch;
  const ResnetArch* resnet = nullptr;         // Faster R-CNN base network
  int num_classes = 0;
  bool with_rcnn = true, use_tail = true, use_mean = true;
  bool tail = false;                          // the RCNN runs the ROIs through block4 (truncated_base_network.py:56-95)
  int output_stride = 16;
  Endpoint ep;

  std::vector<Layer> net;                     // the layer table, in the order of the variables (build_net)
  std::map<std::string, size_t> net_index;    // engine key -> record
  std::vector<WeightSpec> required;           // the variables of the table
  std::map<std::string, HostTensor> staged;
  std::map<std::string, float*> dev_vecs;     // misc device vectors (l2norm gamma, preact scale / bias)

  // Faster R-CNN
  int A = 0, anchor_stride = 16;
  std::vector<int> anchor_ref;                // A x 4 int32 (truncated, quirk Q1)
  int* d_anchor_ref = nullptr;
  float* d_anchors = nullptr; int anchors_fh = 0, anchors_fw = 0;   // current grid (owned by anchor_grids)
  std::map<std::pair<int, int>, float*> anchor_grids;
  RpnParams rpn{};
  int rpn_channels = 512, rpn_kh = 3, rpn_kw = 3, rpn_act = ACT_RELU6;
  std::vector<int> fc_sizes; int fc_act = ACT_RELU6;
  int pooled_w = 7, pooled_h = 7;
  DetParams det{};
  int kmax = 0;
  NmsWorkspace ws_rpn, ws_det;
  float* d_final_keys = nullptr;
  // SSD
  std::vector<int> ssd_app;                   // anchors per point
  std::vector<float> ssd_anchor_host;
  float* d_ssd_anchors = nullptr;
  int ssd_total_anchors = 0;
  int fixed_h = 300, fixed_w = 300;

  Arena arena, arena2;          // arena2: second half-batch when the forward is software-pipelined
  cudaStream_t stream2 = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  float* d_final_keys2 = nullptr;
  int pipeline = 1;             // 1: split the batch in two and run the halves on two streams (hides the
                                // latency-bound proposal / NMS kernels of one half under the other half's convs)
  int* d_overflow = nullptr;
  ConvWorkspace sk_ws[2];       // stream-K scratch, one per stream
  int conv_streamk = 1;         // 0 off, 1 auto, 2 whenever possible
  // conv kernel variants; the defaults are the fastest setting measured on the Faster R-CNN R50 workload (DESIGN 7.2):
  int conv_cta2 = 0;            // env LUMI_CONV_2CTA: 2-CTA cluster kernel on layers with at least this many K slices per tile
  int conv_halo = 0;            // env LUMI_CONV_HALO: 1 = halo-patch kernels on the 3x3 stride-1 layers
  int conv_halo_pct = 150;      // env LUMI_CONV_HALO_PCT: ... while the M-tile count stays within this percentage of the generic kernel's
  int conv_epi16 = 16;          // env LUMI_CONV_EPI16: four-warpgroup kernel on layers with at most this many K slices per tile
  int conv_pipe = 0;            // env LUMI_CONV_PIPE: 1 = double-buffered slice accumulators in the conv mainloop (slower on R50, DESIGN 7.1)
  int conv_epi_tma = 1;         // env LUMI_CONV_EPI_TMA: 1 = split outputs through the shared-memory slot epilogue, 0 = register epilogue
  uint8_t* d_images = nullptr; size_t images_cap = 0;
  float* d_boxes = nullptr; float* d_scores = nullptr; int* d_labels = nullptr; int* d_counts = nullptr;
  int* d_prop_counts = nullptr;
  float* d_records = nullptr;   // caller-owned device buffer [max_batch][1 + 6*kmax] (lumi_set_record_output) or null
  std::map<std::string, Tap> taps;
  int planned_n = 0, planned_h = 0, planned_w = 0;
  // CUDA graphs: one captured graph per (half-)batch forward, keyed by everything baked into its nodes
  struct GraphKey {
    int half, n, h, w, esz, img_off, conv_impl, streamk, reserve;
    const void* records;
    bool operator<(const GraphKey& o) const {
      return std::tie(half, n, h, w, esz, img_off, conv_impl, streamk, reserve, records) <
             std::tie(o.half, o.n, o.h, o.w, o.esz, o.img_off, o.conv_impl, o.streamk, o.reserve, o.records);
    }
  };
  struct GraphEntry { cudaGraphExec_t exec = nullptr; int launches = 0; int seen = 0; };
  std::map<GraphKey, GraphEntry> graphs;
  int use_graphs = 1;           // lumi_set_graphs / env LUMI_GRAPHS; off while profiling or tapping
  int graph_replays = 0;        // forwards served by a graph replay in the last lumi_predict
  void drop_graphs() {
    for (auto& kv : graphs) if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec);
    graphs.clear();
  }
  // per-category device timing (CUDA events on the engine stream), for bench.py's roofline
  bool profile = false;
  struct ProfSpan { int cat; cudaEvent_t a, b; double work; std::string label; };
  std::vector<ProfSpan> prof_spans;
  std::vector<cudaEvent_t> prof_pool;
  std::string prof_text, prof_layers_text;

  ~lumi_engine() {
    drop_graphs();
    for (auto& r : net) conv_layer_free(r.conv);
    for (auto& kv : dev_vecs) cudaFree(kv.second);
    nms_workspace_free(ws_rpn); nms_workspace_free(ws_det);
    conv_workspace_free(sk_ws[0]); conv_workspace_free(sk_ws[1]);
    cudaFree(d_anchor_ref); cudaFree(d_final_keys); cudaFree(d_ssd_anchors);
    for (auto& kv : anchor_grids) cudaFree(kv.second);
    cudaFree(arena.base); cudaFree(arena2.base); cudaFree(d_final_keys2); cudaFree(d_overflow); cudaFree(d_images);
    if (ev_fork) cudaEventDestroy(ev_fork);
    if (ev_join) cudaEventDestroy(ev_join);
    if (stream2) cudaStreamDestroy(stream2);
    cudaFree(d_boxes); cudaFree(d_scores); cudaFree(d_labels); cudaFree(d_counts); cudaFree(d_prop_counts);
    for (auto& sp : prof_spans) { cudaEventDestroy(sp.a); cudaEventDestroy(sp.b); }
    for (auto ev : prof_pool) cudaEventDestroy(ev);
    if (stream) cudaStreamDestroy(stream);
  }
};

namespace {

thread_local std::string g_create_error;

// ---------------------------------------------------------------- network structure
std::string unit_scope(const lumi_engine* e, int b, int u) {
  return "truncated_base_network/" + e->arch + "/block" + std::to_string(b + 1) + "/unit_" + std::to_string(u + 1) +
         (e->resnet->preact ? "/bottleneck_v2" : "/bottleneck_v1");
}

// Whether `part` of unit (b, u) is computed on the way to the endpoint: every part of an earlier unit, and of the
// endpoint's own unit what its output reads (the shortcut only feeds the sum).  The tail runs all of block4.
bool unit_part_runs(const lumi_engine* e, int b, int u, int part) {
  const Endpoint& ep = e->ep;
  if (b == 3 && e->tail) return true;
  if (b != ep.block || u != ep.unit) return b < ep.block || (b == ep.block && u < ep.unit);
  if (ep.part == UP_UNIT) return true;
  if (part == UP_SHORTCUT || ep.part == UP_SHORTCUT) return part == ep.part;
  return part <= ep.part;
}

const char* VGG_NAMES[5] = {"conv1", "conv2", "conv3", "conv4", "conv5"};
const int VGG_REPS[5] = {2, 2, 3, 3, 3};
const int VGG_CH[5] = {64, 128, 256, 512, 512};
struct Extra { const char* name; int k, cin, cout, stride, rate, padding; };
const Extra SSD_EXTRAS[10] = {
    {"conv6", 3, 512, 1024, 1, 6, PAD_SAME},      {"conv7", 1, 1024, 1024, 1, 1, PAD_SAME},
    {"conv8_1", 1, 1024, 256, 1, 1, PAD_SAME},    {"conv8_2", 3, 256, 512, 2, 1, PAD_SAME},
    {"conv9_1", 1, 512, 128, 1, 1, PAD_SAME},     {"conv9_2", 3, 128, 256, 2, 1, PAD_SAME},
    {"conv10_1", 1, 256, 128, 1, 1, PAD_SAME},    {"conv10_2", 3, 128, 256, 1, 1, PAD_VALID},
    {"conv11_1", 1, 256, 128, 1, 1, PAD_SAME},    {"conv11_2", 3, 128, 256, 1, 1, PAD_VALID}};
const int SSD_FMAP_CH[6] = {512, 1024, 512, 256, 256, 256};

// ---------------------------------------------------------------- config
int act_from_name(const std::string& n) {
  if (n == "relu6") return ACT_RELU6;
  if (n == "relu") return ACT_RELU;
  throw Error(LUMI_EINVAL, "unsupported activation_function '" + n + "' (relu | relu6)");
}

void compute_frcnn_anchor_ref(lumi_engine* e) {
  // utils/anchors.py:4-52 in float64, then truncation toward zero (fasterrcnn.py:299-302, quirk Q1)
  const double base = e->cfg.number("model.anchors.base_size", 256);
  std::vector<double> ratios = e->cfg.numbers("model.anchors.ratios");
  std::vector<double> scales = e->cfg.numbers("model.anchors.scales");
  LUMI_REQUIRE(!ratios.empty() && !scales.empty(), "model.anchors.ratios/scales must be non-empty lists");
  e->anchor_ref.clear();
  for (double r : ratios)
    for (double s : scales) {
      const double sq = std::sqrt(r);
      const double hgt = s * sq * base, wid = s / sq * base;
      const double a[4] = {0 - (wid - 1) / 2, 0 - (hgt - 1) / 2, 0 + (wid - 1) / 2, 0 + (hgt - 1) / 2};
      if ((long long)(a[3] - a[1]) == 0 || (long long)(a[2] - a[0]) == 0)
        throw Error(LUMI_EINVAL, "base_size " + std::to_string((int)base) + " is too small for aspect_ratios and scales.");
      for (double v : a) e->anchor_ref.push_back((int)std::trunc(v));
    }
  e->A = (int)(ratios.size() * scales.size());
}

// model.base_network.output_stride, checked as slim's resnet_v1/v2 and resnet_utils.stack_blocks_dense check it over
// all four blocks (luminoth builds the full network, then truncates it at block3).  null means no atrous
// convolution: block3 then ends at stride 32, which is the network output_stride 32 builds.
int frcnn_output_stride(const JVal& c) {
  const JVal* v = c.find("model.base_network.output_stride");
  if (v && v->t == JVal::Null) return 32;
  const double os = c.number("model.base_network.output_stride", 16);
  if (std::fmod(os, 4.0) != 0.0) throw Error(LUMI_EINVAL, "The output_stride needs to be a multiple of 4.");
  const double target = os / 4;
  double current = 1;
  for (int b = 0; b < 4; ++b)
    for (int u = 0; u < 3; ++u) {               // 3 units stand for any count: only the last one has a stride
      if (current > target) throw Error(LUMI_EINVAL, "The target output_stride cannot be reached.");
      if (current != target && u == 2) current *= BLOCK_STRIDE[b];
    }
  if (current != target) throw Error(LUMI_EINVAL, "The target output_stride cannot be reached.");
  return (int)os;
}

// The conv2 stride and atrous rate of unit (b, u), as slim's stack_blocks_dense sets them at output_stride: each
// block's last unit strides until the target stride is reached, after which its stride multiplies the rate of the
// units that follow.  A unit's shortcut (projection or subsampled identity) takes the same stride.
void unit_stride_rate(const lumi_engine* e, int b, int u, int& stride, int& rate) {
  const int target = e->output_stride / 4;
  int current = 1, r = 1;
  for (int bb = 0; bb <= b; ++bb)
    for (int uu = 0; uu < e->resnet->units[bb]; ++uu) {
      const int s = uu == e->resnet->units[bb] - 1 ? BLOCK_STRIDE[bb] : 1;
      const bool atrous = current == target;
      if (bb == b && uu == u) { stride = atrous ? 1 : s; rate = atrous ? r : 1; return; }
      if (atrous) r *= s;
      else current *= s;
    }
}

// model.base_network.endpoint (null or empty: block3), matched as _get_endpoint matches it against the outputs slim's
// resnet collects: the stem conv1, every bottleneck unit and its conv1 / conv2 / conv3 / projection shortcut, and
// every block.  Then the tail rule: resnet_v1_101's tail reuses block4's variables, whose first unit reads 1024
// channels.  Needs output_stride, use_tail and with_rcnn.
void parse_endpoint(lumi_engine* e) {
  Endpoint& ep = e->ep;
  const JVal* v = e->cfg.find("model.base_network.endpoint");
  if (v && v->t != JVal::Null) {
    if (v->t != JVal::Str) throw Error(LUMI_EINVAL, "model.base_network.endpoint must be a string");
    if (!v->s.empty()) ep.name = v->s;
  }
  const std::string root = "truncated_base_network/" + e->arch, n = root + "/" + ep.name;
  const char* PARTS[4] = {"/conv1", "/conv2", "/conv3", "/shortcut"};
  bool found = n == root + "/conv1";
  if (found) { ep.block = -1; ep.depth = 64; ep.stride = 2; }
  int stride = 4;                                  // after pool1
  for (int b = 0; b < 4 && !found; ++b) {
    const int units = e->resnet->units[b];
    for (int u = 0; u < units && !found; ++u) {
      const std::string s = unit_scope(e, b, u);
      int part = -1;
      if (n == s || (u == units - 1 && n == root + "/block" + std::to_string(b + 1))) part = UP_UNIT;
      for (int p = 0; p < 4; ++p)
        if (n == s + PARTS[p] && (p != UP_SHORTCUT || u == 0)) part = p;   // only a block's first unit projects
      int st, rt;
      unit_stride_rate(e, b, u, st, rt);
      if (part != UP_CONV1) stride *= st;
      if (part < 0) continue;
      found = true;
      ep.block = b; ep.unit = u; ep.part = part;
      ep.depth = BASE_DEPTH[b] * (part == UP_CONV1 || part == UP_CONV2 ? 1 : 4);
      ep.stride = stride;
    }
  }
  if (!found) throw Error(LUMI_EINVAL, "\"" + n + "\" is an invalid value of endpoint for this architecture.");
  e->tail = e->arch == "resnet_v1_101" && e->use_tail && e->with_rcnn;
  if (e->tail && ep.depth != 1024)
    throw Error(LUMI_EINVAL, "the resnet_v1_101 tail needs a 1024-channel endpoint: \"" + ep.name + "\" has " +
                                 std::to_string(ep.depth) + " channels (set model.base_network.use_tail to false)");
}

// the endpoint map's size along an image side of `size` pixels: every stride-2 stage (conv2d_same, SAME max pool,
// subsampled shortcut) gives ceil(x / 2)
int feature_size(const lumi_engine* e, int size) { return cdiv(size, e->ep.stride); }

void parse_config(lumi_engine* e) {
  const JVal& c = e->cfg;
  e->type = c.str("model.type", "");
  if (e->type != "fasterrcnn" && e->type != "ssd")
    throw Error(LUMI_EINVAL, "\"" + e->type + "\" is not a valid model_type");
  e->num_classes = (int)c.number("model.network.num_classes", 0);
  LUMI_REQUIRE(e->num_classes > 0, "model.network.num_classes must be positive");
  if (e->type == "fasterrcnn") {
    e->arch = c.str("model.base_network.architecture", "resnet_v1_101");
    std::string known;
    for (const ResnetArch& r : RESNETS) {
      if (e->arch == r.name) e->resnet = &r;
      known += std::string(known.empty() ? "" : " | ") + r.name;
    }
    if (!e->resnet)
      throw Error(LUMI_EINVAL, "base_network.architecture '" + e->arch + "' is not built yet (" + known + ")");
    e->with_rcnn = c.boolean("model.network.with_rcnn", false);
    e->use_tail = c.boolean("model.base_network.use_tail", true);
    e->output_stride = frcnn_output_stride(c);
    parse_endpoint(e);
    e->anchor_stride = (int)c.number("model.anchors.stride", 16);
    compute_frcnn_anchor_ref(e);
    e->rpn_channels = (int)c.number("model.rpn.num_channels", 512);
    std::vector<double> ks = c.numbers("model.rpn.kernel_shape");
    if (ks.size() == 2) { e->rpn_kh = (int)ks[0]; e->rpn_kw = (int)ks[1]; }
    e->rpn_act = act_from_name(c.str("model.rpn.activation_function", "relu6"));
    RpnParams& r = e->rpn;
    r.pre_nms_top_n = (int)c.number("model.rpn.proposals.pre_nms_top_n", 12000);
    r.post_nms_top_n = (int)c.number("model.rpn.proposals.post_nms_top_n", 2000);
    r.apply_nms = c.boolean("model.rpn.proposals.apply_nms", true);
    r.nms_threshold = (float)c.number("model.rpn.proposals.nms_threshold", 0.7);
    r.min_prob = (float)c.number("model.rpn.proposals.min_prob_threshold", 0.0);
    r.filter_outside = c.boolean("model.rpn.proposals.filter_outside_anchors", false);
    r.clip_after_nms = c.boolean("model.rpn.proposals.clip_after_nms", false);
    LUMI_REQUIRE(r.pre_nms_top_n > 0 && r.post_nms_top_n > 0, "pre/post_nms_top_n must be positive");
    if (!r.apply_nms) r.post_nms_top_n = r.pre_nms_top_n;   // rpn_proposal.py:172-174: all sorted top-n survive
    e->kmax = r.post_nms_top_n;
    if (e->with_rcnn) {
      for (double v : c.numbers("model.rcnn.layer_sizes")) e->fc_sizes.push_back((int)v);
      e->fc_act = act_from_name(c.str("model.rcnn.activation_function", "relu6"));
      e->use_mean = c.boolean("model.rcnn.use_mean", true);
      std::string mode = c.str("model.rcnn.roi.pooling_mode", "crop");
      std::transform(mode.begin(), mode.end(), mode.begin(), ::tolower);
      if (mode != "crop") throw Error(LUMI_EINVAL, "Pooling mode " + mode + " is not implemented (roi_pool.py:97-102)");
      e->pooled_w = (int)c.number("model.rcnn.roi.pooled_width", 7);
      e->pooled_h = (int)c.number("model.rcnn.roi.pooled_height", 7);
      // the ROI kernels keep the 2 * (pooled_width + pooled_height) crop sample coordinates of a roi in 64 slots
      if (e->pooled_w < 1 || e->pooled_h < 1 || 2 * (e->pooled_w + e->pooled_h) > 64)
        throw Error(LUMI_EINVAL, "model.rcnn.roi.pooled_width and pooled_height must be >= 1 with 2 * (pooled_width + "
                                 "pooled_height) <= 64, got " + std::to_string(e->pooled_w) + " x " +
                                 std::to_string(e->pooled_h));
      LUMI_REQUIRE(c.str("model.rcnn.roi.padding", "VALID") == "VALID", "roi.padding must be VALID");
      DetParams& d = e->det;
      d.nc = e->num_classes;
      std::vector<double> var = c.numbers("model.rcnn.target_normalization_variances");
      d.var0 = var.size() == 2 ? (float)var[0] : 1.f;
      d.var1 = var.size() == 2 ? (float)var[1] : 1.f;
      d.min_prob = (float)c.number("model.rcnn.proposals.min_prob_threshold", 0.0);
      d.nms_threshold = (float)c.number("model.rcnn.proposals.class_nms_threshold", 0.5);
      d.class_max = (int)c.number("model.rcnn.proposals.class_max_detections", 100);
      d.total_max = (int)c.number("model.rcnn.proposals.total_max_detections", 300);
      d.shared_deltas = 0;
      e->kmax = d.total_max;
    }
  } else {
    e->arch = c.str("model.base_network.architecture", "truncated_vgg_16");
    if (e->arch != "truncated_vgg_16") throw Error(LUMI_EINVAL, "Invalid architecture \"" + e->arch + "\"");
    e->fixed_h = (int)c.number("dataset.image_preprocessing.fixed_height", 300);
    e->fixed_w = (int)c.number("dataset.image_preprocessing.fixed_width", 300);
    for (double v : c.numbers("model.anchors.anchors_per_point")) e->ssd_app.push_back((int)v);
    LUMI_REQUIRE(e->ssd_app.size() == 6, "model.anchors.anchors_per_point must have 6 entries");
    DetParams& d = e->det;
    d.nc = e->num_classes;
    std::vector<double> var = c.numbers("model.variances");
    d.var0 = var.size() == 2 ? (float)var[0] : 1.f;
    d.var1 = var.size() == 2 ? (float)var[1] : 1.f;
    d.min_prob = (float)c.number("model.proposals.min_prob_threshold", 0.0);
    d.nms_threshold = (float)c.number("model.proposals.class_nms_threshold", 0.45);
    d.class_max = (int)c.number("model.proposals.class_max_detections", 100);
    d.total_max = (int)c.number("model.proposals.total_max_detections", 100);
    d.shared_deltas = 1;
    e->kmax = d.total_max;
  }
}

// ---------------------------------------------------------------- layer table
Layer& add_layer(lumi_engine* e, int kind, const std::string& key, std::vector<std::string> scopes) {
  e->net_index[key] = e->net.size();
  e->net.emplace_back();
  Layer& r = e->net.back();
  r.kind = kind; r.key = key; r.scopes = std::move(scopes);
  return r;
}

void add_conv(lumi_engine* e, int kind, int naming, const std::string& key, std::vector<std::string> scopes,
              std::vector<int> couts, int kh, int kw, int cin, int stride, int rate, int act, int padding) {
  Layer& r = add_layer(e, kind, key, std::move(scopes));
  r.naming = naming; r.couts = std::move(couts);
  r.kh = kh; r.kw = kw; r.cin = cin; r.stride = stride; r.rate = rate; r.act = act; r.padding = padding;
}

void add_vector(lumi_engine* e, int kind, const std::string& key, const std::string& scope, int channels) {
  add_layer(e, kind, key, {scope}).cin = channels;
}

// The layer table of the configured network, in the order of its variables.  Faster R-CNN: slim resnet_v1 / resnet_v2
// up to the endpoint (and block4 for the resnet_v1_101 tail; resnet_v2's `postnorm` follows block4 and is never
// reached), the RPN, the RCNN fcs and heads.  SSD: truncated VGG16, the L2-norm gamma, the extras, the multibox heads.
void build_net(lumi_engine* e) {
  if (e->type == "fasterrcnn") {
    const std::string root = "truncated_base_network/" + e->arch;
    const bool v2 = e->resnet->preact;
    // conv2d_same(64, 7, stride 2) + BN + relu (v2: + bias, no activation)
    add_conv(e, v2 ? LK_CONV_BIAS : LK_CONV_BN, NM_SLIM, root + "/conv1", {root + "/conv1"}, {64}, 7, 7, 3, 2, 1,
             v2 ? ACT_NONE : ACT_RELU, PAD_CONV2D_SAME);
    add_layer(e, LK_STEM_S2D, root + "/conv1#s2d", {root + "/conv1"});
    // bottleneck_v2: preact = relu(BN(x)); shortcut and conv3 with biases, no BN or activation; out = the raw sum
    const int kind3 = v2 ? LK_CONV_BIAS : LK_CONV_BN;   // of the shortcut and conv3
    for (int b = 0; b < 4; ++b) {
      const int bd = BASE_DEPTH[b], depth = bd * 4;
      for (int u = 0; u < e->resnet->units[b]; ++u) {
        auto runs = [&](int part) { return unit_part_runs(e, b, u, part); };
        if (!runs(UP_CONV1) && !runs(UP_SHORTCUT)) continue;
        const int cin = u > 0 ? depth : b > 0 ? BASE_DEPTH[b - 1] * 4 : 64;
        const std::string s = unit_scope(e, b, u);
        int st = 1, rt = 1;                                   // tail: stack_blocks_dense w/o output_stride, stride 1
        if (!(b == 3 && e->tail)) unit_stride_rate(e, b, u, st, rt);
        if (v2) add_vector(e, LK_PREACT, s + "/preact", s + "/preact", cin);
        if (cin != depth && runs(UP_SHORTCUT))
          add_conv(e, kind3, NM_SLIM, s + "/shortcut", {s + "/shortcut"}, {depth}, 1, 1, cin, st, 1, ACT_NONE,
                   PAD_SAME);
        if (runs(UP_CONV1))
          add_conv(e, LK_CONV_BN, NM_SLIM, s + "/conv1", {s + "/conv1"}, {bd}, 1, 1, cin, 1, 1, ACT_RELU, PAD_SAME);
        if (runs(UP_CONV2))
          add_conv(e, LK_CONV_BN, NM_SLIM, s + "/conv2", {s + "/conv2"}, {bd}, 3, 3, bd, st, rt, ACT_RELU,
                   PAD_CONV2D_SAME);
        // v1: relu applied after the residual add; a conv3 endpoint is collected before both
        const bool conv3_ep = b == e->ep.block && u == e->ep.unit && e->ep.part == UP_CONV3;
        if (runs(UP_CONV3))
          add_conv(e, kind3, NM_SLIM, s + "/conv3", {s + "/conv3"}, {depth}, 1, 1, bd, 1, 1,
                   v2 || conv3_ep ? ACT_NONE : ACT_RELU, PAD_SAME);
      }
    }
    const std::string r = "fasterrcnn/rpn";
    add_conv(e, LK_CONV_BIAS, NM_SONNET, r + "/conv", {r + "/conv"}, {e->rpn_channels}, e->rpn_kh, e->rpn_kw,
             e->ep.depth, 1, 1, e->rpn_act, PAD_SAME);
    add_conv(e, LK_CONV_BIAS, NM_SONNET, r + "/heads", {r + "/cls_conv", r + "/bbox_conv"}, {2 * e->A, 4 * e->A}, 1, 1,
             e->rpn_channels, 1, 1, ACT_NONE, PAD_SAME);
    if (e->with_rcnn) {
      int d = e->tail ? 2048 : e->ep.depth;
      if (!e->use_mean) d *= e->pooled_w * e->pooled_h;
      const std::string c = "fasterrcnn/rcnn";
      for (size_t i = 0; i < e->fc_sizes.size(); ++i) {
        const std::string fc = c + "/fc_" + std::to_string(i);
        add_conv(e, LK_CONV_BIAS, NM_LINEAR, fc, {fc}, {e->fc_sizes[i]}, 1, 1, d, 1, 1, e->fc_act, PAD_SAME);
        d = e->fc_sizes[i];
      }
      add_conv(e, LK_CONV_BIAS, NM_LINEAR, c + "/heads", {c + "/fc_classifier", c + "/fc_bbox"},
               {e->num_classes + 1, 4 * e->num_classes}, 1, 1, d, 1, 1, ACT_NONE, PAD_SAME);
    }
  } else {
    const std::string s = "ssd/ssd_feature_extractor";
    int cin = 3;
    for (int b = 0; b < 5; ++b)
      for (int r = 0; r < VGG_REPS[b]; ++r) {
        const std::string p = s + "/vgg_16/" + VGG_NAMES[b] + "/" + VGG_NAMES[b] + "_" + std::to_string(r + 1);
        add_conv(e, LK_CONV_BIAS, NM_SLIM, p, {p}, {VGG_CH[b]}, 3, 3, cin, 1, 1, ACT_RELU, PAD_SAME);
        if (b == 0 && r == 0) add_layer(e, LK_CONV1_1_PACK, p + "#pack", {p});
        cin = VGG_CH[b];
      }
    add_vector(e, LK_GAMMA, "gamma", s + "/conv_4_3_norm", 512);
    for (const Extra& x : SSD_EXTRAS) {
      const std::string p = s + "/extra_feature_layers/" + x.name;
      add_conv(e, LK_CONV_BIAS, NM_SONNET, p, {p}, {x.cout}, x.k, x.k, x.cin, x.stride, x.rate, ACT_RELU, x.padding);
    }
    for (int i = 0; i < 6; ++i) {
      const std::string n = "ssd/MultiBox_" + std::to_string(i);
      add_conv(e, LK_CONV_BIAS, NM_SONNET, n, {n + "_offsets_conv", n + "_classes_conv"},
               {4 * e->ssd_app[i], (e->num_classes + 1) * e->ssd_app[i]}, 3, 3, SSD_FMAP_CH[i], 1, 1, ACT_NONE,
               PAD_SAME);
    }
  }
}

Layer& layer(lumi_engine* e, const std::string& key) {
  auto it = e->net_index.find(key);
  if (it == e->net_index.end()) throw Error(LUMI_ESTATE, "layer '" + key + "' missing (internal)");
  return e->net[it->second];
}

const char* BN_VARS[4] = {"gamma", "beta", "moving_mean", "moving_variance"};
std::string weights_var(const Layer& r, size_t i) { return r.scopes[i] + (r.naming == NM_SLIM ? "/weights" : "/w"); }
std::string biases_var(const Layer& r, size_t i) { return r.scopes[i] + (r.naming == NM_SLIM ? "/biases" : "/b"); }

void build_specs(lumi_engine* e) {
  auto need = [e](const std::string& name, std::vector<int64_t> shape) { e->required.push_back({name, shape}); };
  for (const Layer& r : e->net) {
    if (r.kind == LK_CONV_BN) {
      need(weights_var(r, 0), {r.kh, r.kw, r.cin, r.couts[0]});
      for (const char* n : BN_VARS) need(r.scopes[0] + "/BatchNorm/" + n, {r.couts[0]});
    } else if (r.kind == LK_CONV_BIAS) {
      for (size_t i = 0; i < r.scopes.size(); ++i) {
        if (r.naming == NM_LINEAR) need(weights_var(r, i), {r.cin, r.couts[i]});
        else need(weights_var(r, i), {r.kh, r.kw, r.cin, r.couts[i]});
        need(biases_var(r, i), {r.couts[i]});
      }
    } else if (r.kind == LK_PREACT) {
      for (const char* n : BN_VARS) need(r.scopes[0] + "/" + n, {r.cin});
    } else if (r.kind == LK_GAMMA) {
      need(r.scopes[0] + "/gamma", {1, 1, 1, r.cin});
    }
  }
}

// ---------------------------------------------------------------- finalize helpers
const HostTensor& W(lumi_engine* e, const std::string& name) {
  auto it = e->staged.find(name);
  if (it == e->staged.end()) throw Error(LUMI_ENOWEIGHT, "variable '" + name + "' was never set");
  return it->second;
}

// conv + folded inference BN (slim batch_norm, eps 1e-5): y = conv*s + (beta - mean*s), s = gamma/sqrt(var+eps)
void make_conv_bn(lumi_engine* e, Layer& r) {
  const std::string& scope = r.scopes[0];
  const HostTensor& w = W(e, scope + "/weights");
  ConvLayer L;
  L.kh = (int)w.shape[0]; L.kw = (int)w.shape[1]; L.cin = (int)w.shape[2]; L.cout = (int)w.shape[3];
  L.stride = r.stride; L.rate = r.rate; L.act = r.act;
  const HostTensor& g = W(e, scope + "/BatchNorm/gamma");
  const HostTensor& b = W(e, scope + "/BatchNorm/beta");
  const HostTensor& m = W(e, scope + "/BatchNorm/moving_mean");
  const HostTensor& v = W(e, scope + "/BatchNorm/moving_variance");
  std::vector<float> sc(L.cout), bi(L.cout);
  for (int c = 0; c < L.cout; ++c) {
    const double s = (double)g.v[c] / std::sqrt((double)v.v[c] + 1e-5);
    sc[c] = (float)s;
    bi[c] = (float)((double)b.v[c] - (double)m.v[c] * s);
  }
  conv_layer_upload(L, w.v.data(), sc.data(), bi.data());
  r.conv = L;
}

// conv + bias (Sonnet / slim-VGG), fusing the convs of several same-input scopes along C_out
void make_conv_bias(lumi_engine* e, Layer& r) {
  const HostTensor& w0 = W(e, weights_var(r, 0));
  const bool linear = w0.shape.size() == 2;
  ConvLayer L;
  L.kh = linear ? 1 : (int)w0.shape[0]; L.kw = linear ? 1 : (int)w0.shape[1];
  L.cin = linear ? (int)w0.shape[0] : (int)w0.shape[2];
  L.stride = r.stride; L.rate = r.rate; L.act = r.act;
  int cout = 0;
  for (size_t i = 0; i < r.scopes.size(); ++i) cout += (int)W(e, weights_var(r, i)).shape.back();
  L.cout = cout;
  const size_t kdim = (size_t)L.kh * L.kw * L.cin;
  std::vector<float> w(kdim * cout), b(cout, 0.f);
  int off = 0;
  for (size_t i = 0; i < r.scopes.size(); ++i) {
    const HostTensor& wi = W(e, weights_var(r, i));
    const int co = (int)wi.shape.back();
    LUMI_REQUIRE(wi.v.size() == kdim * co, "fused conv '" + r.key + "': weight shapes disagree");
    for (size_t k = 0; k < kdim; ++k) std::memcpy(&w[k * cout + off], &wi.v[k * co], co * sizeof(float));
    std::memcpy(&b[off], W(e, biases_var(r, i)).v.data(), co * sizeof(float));
    off += co;
  }
  conv_layer_upload(L, w.data(), nullptr, b.data());
  r.conv = L;
}

// resnet_v2 `preact` batch norm (slim batch_norm, eps 1e-5) folded like make_conv_bn, as the device vectors
// <unit>/preact#scale and #bias that the producing conv epilogue (or the stem's max pool) applies; padded to a
// multiple of 128 channels for the tensor-core epilogue's vector loads
void make_preact(lumi_engine* e, const Layer& r) {
  const std::string& scope = r.scopes[0];
  const HostTensor& g = W(e, scope + "/gamma");
  const HostTensor& b = W(e, scope + "/beta");
  const HostTensor& m = W(e, scope + "/moving_mean");
  const HostTensor& v = W(e, scope + "/moving_variance");
  const int c = (int)g.v.size(), cpad = cdiv(c, 128) * 128;
  std::vector<float> sc(cpad, 0.f), bi(cpad, 0.f);
  for (int i = 0; i < c; ++i) {
    const double s = (double)g.v[i] / std::sqrt((double)v.v[i] + 1e-5);
    sc[i] = (float)s;
    bi[i] = (float)((double)b.v[i] - (double)m.v[i] * s);
  }
  for (int k = 0; k < 2; ++k) {
    float* d = nullptr;
    LUMI_CUDA_CHECK(cudaMalloc(&d, cpad * sizeof(float)));
    e->dev_vecs[r.key + (k ? "#bias" : "#scale")] = d;
    LUMI_CUDA_CHECK(cudaMemcpy(d, (k ? bi : sc).data(), cpad * sizeof(float), cudaMemcpyHostToDevice));
  }
}

// tensor-core form of the resnet stem: 7x7/2 over 3 channels == 4x4/1 over the 12(+4 pad)-channel space-to-depth
// input; one filter row r' = 4 taps x 16 ch = one K=64 slice  (kh=4, kw=1, cin=64)
void make_stem_s2d(lumi_engine* e, Layer& r) {
  const HostTensor& w = W(e, r.scopes[0] + "/weights");
  const ConvLayer& base = layer(e, r.scopes[0]).conv;
  std::vector<float> w2((size_t)4 * 64 * 64, 0.f);
  for (int rp = 0; rp < 4; ++rp)
    for (int sp = 0; sp < 4; ++sp)
      for (int dy = 0; dy < 2; ++dy)
        for (int dx = 0; dx < 2; ++dx) {
          const int ry = 2 * rp + dy, sx = 2 * sp + dx;
          if (ry >= 7 || sx >= 7) continue;
          for (int c = 0; c < 3; ++c)
            for (int co = 0; co < 64; ++co)
              w2[((size_t)rp * 64 + sp * 16 + dy * 6 + dx * 3 + c) * 64 + co] = w.v[(((size_t)ry * 7 + sx) * 3 + c) * 64 + co];
        }
  std::vector<float> sc(64), bi(64);
  LUMI_CUDA_CHECK(cudaMemcpy(sc.data(), base.scale, 64 * sizeof(float), cudaMemcpyDeviceToHost));
  LUMI_CUDA_CHECK(cudaMemcpy(bi.data(), base.bias, 64 * sizeof(float), cudaMemcpyDeviceToHost));
  ConvLayer L;
  L.kh = 4; L.kw = 1; L.cin = 64; L.cout = 64; L.stride = 1; L.rate = 1; L.act = base.act;
  conv_layer_upload(L, w2.data(), sc.data(), bi.data());
  r.conv = L;
}

// tensor-core form of SSD's conv1_1 (3x3 over 3 channels): one filter row = 4 pixels x 16 ch = one K=64 slice
// (kh=3, kw=1, cin=64) over the padded 16-channel staging written by launch_pack_c3
void make_conv1_1_pack(lumi_engine* e, Layer& r) {
  const HostTensor& w = W(e, r.scopes[0] + "/weights");
  const HostTensor& b = W(e, r.scopes[0] + "/biases");
  const int co_n = (int)w.shape[3];
  LUMI_REQUIRE(w.shape[0] == 3 && w.shape[1] == 3 && w.shape[2] == 3, "conv1_1 must be 3x3x3");
  std::vector<float> w2((size_t)3 * 64 * co_n, 0.f);
  for (int ry = 0; ry < 3; ++ry)
    for (int sx = 0; sx < 3; ++sx)
      for (int c = 0; c < 3; ++c)
        for (int co = 0; co < co_n; ++co)
          w2[((size_t)ry * 64 + sx * 16 + c) * co_n + co] = w.v[(((size_t)ry * 3 + sx) * 3 + c) * co_n + co];
  ConvLayer L;
  L.kh = 3; L.kw = 1; L.cin = 64; L.cout = co_n; L.stride = 1; L.rate = 1; L.act = ACT_RELU;
  conv_layer_upload(L, w2.data(), nullptr, b.v.data());
  r.conv = L;
}

void build_layers(lumi_engine* e) {
  for (Layer& r : e->net) {
    if (r.kind == LK_CONV_BN) make_conv_bn(e, r);
    else if (r.kind == LK_CONV_BIAS) make_conv_bias(e, r);
    else if (r.kind == LK_PREACT) make_preact(e, r);
    else if (r.kind == LK_STEM_S2D) make_stem_s2d(e, r);
    else if (r.kind == LK_CONV1_1_PACK) make_conv1_1_pack(e, r);
    else if (r.kind == LK_GAMMA) {
      const HostTensor& g = W(e, r.scopes[0] + "/gamma");
      float* d = nullptr;
      LUMI_CUDA_CHECK(cudaMalloc(&d, g.v.size() * sizeof(float)));
      LUMI_CUDA_CHECK(cudaMemcpy(d, g.v.data(), g.v.size() * sizeof(float), cudaMemcpyHostToDevice));
      e->dev_vecs[r.key] = d;
    }
  }
}

// ---------------------------------------------------------------- per-category timing
enum ProfCat { PC_CONV_TC = 0, PC_CONV_SIMT, PC_POOL, PC_PREP, PC_RPN_POST, PC_ROI, PC_HEAD_MISC, PC_DET_POST, PC_COUNT };
const char* PROF_NAMES[PC_COUNT] = {"conv_tc", "conv_simt", "pool", "preprocess", "rpn_proposals", "roi_pool",
                                    "head_misc", "detections"};

cudaEvent_t prof_event(lumi_engine* e) {
  if (!e->prof_pool.empty()) { cudaEvent_t ev = e->prof_pool.back(); e->prof_pool.pop_back(); return ev; }
  cudaEvent_t ev;
  LUMI_CUDA_CHECK(cudaEventCreate(&ev));
  return ev;
}
struct ProfScope {
  lumi_engine* e; int idx = -1;
  // work: algorithmic FLOPs (conv) or bytes (HBM-bound stages) of the kernels inside the span
  ProfScope(lumi_engine* eng, bool dry, int cat, double work = 0.0, const std::string& label = std::string()) : e(eng) {
    if (dry || !e->profile) return;
    lumi_engine::ProfSpan sp{cat, prof_event(e), prof_event(e), work, label};
    LUMI_CUDA_CHECK(cudaEventRecord(sp.a, e->stream));
    e->prof_spans.push_back(sp);
    idx = (int)e->prof_spans.size() - 1;
  }
  ~ProfScope() { if (idx >= 0) cudaEventRecord(e->prof_spans[idx].b, e->stream); }
};

// ---------------------------------------------------------------- execution context
struct Ctx {
  lumi_engine* e;
  bool dry;
  cudaStream_t st;
  Arena* arena = nullptr;       // workspace of this (half-)batch
  int img_off = 0;              // first image of this (half-)batch inside the engine-level batch buffers
  float* final_keys = nullptr;  // scratch of the final top-k sort
  ConvWorkspace* sk = nullptr;  // stream-K scratch of this stream
  bool taps = true;             // record debug taps (first half only)
  bool img_f32 = false;         // input pixels are float32 (resized images) instead of uint8
  int sm_reserve = 0;           // SMs the persistent conv launches of this forward leave to the other stream
  Act act(int n, int h, int w, int c) {
    Act a; a.n = n; a.h = h; a.w = w; a.c = c;
    const size_t bytes = a.numel() * sizeof(__half);
    a.hi = (__half*)arena->alloc(bytes, dry);
    a.lo = (__half*)arena->alloc(bytes, dry);
    return a;
  }
  float* f32(size_t count) { return (float*)arena->alloc(count * sizeof(float), dry); }
  void tap_f32(const std::string& name, const float* p, int64_t a, int64_t b, int64_t c, int64_t d) {
    if (!taps) return;
    Tap t; t.ptr = p; t.kind = 0; t.shape[0] = a; t.shape[1] = b; t.shape[2] = c; t.shape[3] = d;
    e->taps[name] = t;
  }
  void tap_act(const std::string& name, Act a) {
    if (!taps) return;
    Tap t; t.kind = 1; t.act = a; t.shape[0] = a.n; t.shape[1] = a.h; t.shape[2] = a.w; t.shape[3] = a.c;
    e->taps[name] = t;
  }
  void tap_i32(const std::string& name, const int* p, int64_t a) {
    if (!taps) return;
    Tap t; t.ptr = p; t.kind = 2; t.shape[0] = a; t.shape[1] = 1; t.shape[2] = 1; t.shape[3] = 1;
    e->taps[name] = t;
  }
};

// problems [off, ...) of a batched NMS workspace (the second half-batch works on its own slice)
NmsWorkspace ws_view(const NmsWorkspace& ws, int off) {
  NmsWorkspace v = ws;
  v.problems = ws.problems - off;
  v.keys = ws.keys + (size_t)off * ws.cap;
  v.boxes = ws.boxes + (size_t)off * ws.cap * 4;
  v.order = ws.order + (size_t)off * ws.cap;
  v.nvalid = ws.nvalid + off;
  v.sboxes = ws.sboxes + (size_t)off * ws.ncap * 4;
  v.sscores = ws.sscores + (size_t)off * ws.ncap;
  v.mask = ws.mask + (size_t)off * ws.ncap * ws.words;
  v.keep = ws.keep + (size_t)off * ws.max_out;
  v.nkeep = ws.nkeep + off;
  v.sort_tmp = ws.sort_tmp + (size_t)off * 2 * ws.cap;
  if (ws.sboxes2) {
    v.sboxes2 = ws.sboxes2 + (size_t)off * ws.ncap * 4;
    v.index_map = ws.index_map + (size_t)off * ws.ncap;
    v.alive = ws.alive + (size_t)off * ws.ncap;
    v.nvalid2 = ws.nvalid2 + off;
  }
  if (ws.cut_hist) {
    v.cut_hist = ws.cut_hist + (size_t)off * 4 * 256;
    v.cut_counts = ws.cut_counts + (size_t)off * ws.cut_blocks;
  }
  return v;
}

// Pre-activation output of a conv (ConvIO::pre): the next resnet_v2 unit's relu(BN(x)), written by the epilogue as
// p; keep_x = false leaves x unwritten (run_conv then returns an Act without planes).
struct PreAct {
  const float* scale = nullptr;
  const float* bias = nullptr;
  bool keep_x = true;
  Act p;
};
PreAct preact_of(lumi_engine* e, const std::string& unit, bool keep_x) {
  PreAct pa;
  pa.scale = e->dev_vecs.at(unit + "/preact#scale");
  pa.bias = e->dev_vecs.at(unit + "/preact#bias");
  pa.keep_x = keep_x;
  return pa;
}

Act run_conv(Ctx& cx, const std::string& key, Act in, const Act* res, int res_stride, float** out_f32,
             const long* view_pitch = nullptr, double algorithmic_flops = -1.0, PreAct* pre = nullptr) {
  const Layer& R = layer(cx.e, key);
  const ConvLayer& L = R.conv;
  ConvIO io;
  io.in = in;
  int ho, wo, pt = 0, pl = 0;
  if (R.padding == PAD_SAME || (R.padding == PAD_CONV2D_SAME && L.stride == 1)) {
    tf_same(in.h, L.kh, L.stride, L.rate, ho, pt);
    tf_same(in.w, L.kw, L.stride, L.rate, wo, pl);
  } else if (R.padding == PAD_CONV2D_SAME) {
    const int keff = L.kh + (L.kh - 1) * (L.rate - 1);
    pt = pl = (keff - 1) / 2;
    ho = (in.h + (keff - 1) - keff) / L.stride + 1;
    wo = (in.w + (keff - 1) - keff) / L.stride + 1;
  } else {
    ho = tf_valid(in.h, L.kh, L.stride, L.rate);
    wo = tf_valid(in.w, L.kw, L.stride, L.rate);
  }
  LUMI_REQUIRE(ho > 0 && wo > 0, "conv '" + key + "': input too small");
  io.pad_t = pt; io.pad_l = pl; io.ho = ho; io.wo = wo;
  Act out; out.n = in.n; out.h = ho; out.w = wo; out.c = L.cout;
  if (out_f32) {
    *out_f32 = cx.f32((size_t)in.n * ho * wo * L.cout);
    io.out_f32 = *out_f32;
  } else if (!pre || pre->keep_x) {
    out = cx.act(in.n, ho, wo, L.cout);
    io.out = out;
  }
  if (pre) {
    LUMI_REQUIRE(!out_f32, "conv '" + key + "': pre-activation outputs are split planes (internal)");
    pre->p = cx.act(in.n, ho, wo, L.cout);
    io.pre = pre->p; io.pre_scale = pre->scale; io.pre_bias = pre->bias;
  }
  if (res) { io.res = *res; io.res_stride = res_stride; }
  if (view_pitch) { io.in_pix_pitch = view_pitch[0]; io.in_row_pitch = view_pitch[1]; io.in_img_pitch = view_pitch[2]; }
  io.overflow_flag = cx.e->d_overflow;
  io.sk = cx.sk;
  io.streamk = cx.e->conv_streamk;
  io.sm_reserve = cx.sm_reserve;
  io.cta2 = cx.e->conv_cta2;
  io.halo = cx.e->conv_halo;
  io.halo_tiles_pct = cx.e->conv_halo_pct;
  io.epi16 = cx.e->conv_epi16;
  io.pipe = cx.e->conv_pipe;
  io.epi_tma = cx.e->conv_epi_tma;
  if (!cx.dry) {
    const bool tc = cx.e->conv_impl == 1 && conv_tc_supported(L, io);
    const double flops = algorithmic_flops >= 0 ? algorithmic_flops
                                                : 2.0 * (double)in.n * ho * wo * (double)L.kh * L.kw * L.cin * L.cout;
    LUMI_REQUIRE(tc || !view_pitch, "strided input views exist only on the tensor-core path (internal)");
    ProfScope ps(cx.e, cx.dry, tc ? PC_CONV_TC : PC_CONV_SIMT, flops, key);
    if (tc) launch_conv_tc(L, io, cx.st);
    else launch_conv_simt(L, io, cx.st);
  }
  return out;
}

// pre: returns relu(BN(max pool)) instead of the max pool (the resnet_v2 stem feeds only the first unit's preact)
Act run_pool(Ctx& cx, Act in, int k, int stride, bool same, const PreAct* pre = nullptr) {
  int ho, wo, pt = 0, pl = 0;
  if (same) { tf_same(in.h, k, stride, 1, ho, pt); tf_same(in.w, k, stride, 1, wo, pl); }
  else { ho = tf_valid(in.h, k, stride, 1); wo = tf_valid(in.w, k, stride, 1); }
  LUMI_REQUIRE(ho > 0 && wo > 0, "max_pool: input too small");
  Act out = cx.act(in.n, ho, wo, in.c);
  if (!cx.dry) {
    ProfScope ps(cx.e, cx.dry, PC_POOL);
    launch_max_pool(in, out, k, stride, pt, pl, cx.st, pre ? pre->scale : nullptr, pre ? pre->bias : nullptr);
  }
  return out;
}

// slim bottleneck_v2 on (x, p = relu(BN_preact(x))); x may be absent when the unit projects its shortcut from p.
// A slim bottleneck_v1 unit is the same computation with p = x and no `next`.
// conv3 writes what the next unit reads, from `next` (nullptr: the endpoint, x only): p always, and x as well when
// that unit's shortcut is the identity (its depth equals this unit's).  `stop` (a UnitPart) returns that collected
// conv output instead of the unit's.
Act bottleneck_v2(Ctx& cx, const std::string& s, Act x, Act p, int depth, PreAct* next, int stop = UP_UNIT) {
  if (stop == UP_SHORTCUT) return run_conv(cx, s + "/shortcut", p, nullptr, 1, nullptr);
  Act shortcut = x;
  int res_stride = 1;
  if (stop == UP_UNIT) {
    res_stride = layer(cx.e, s + "/conv2").stride;   // subsample(x, stride)
    if (p.c != depth) { shortcut = run_conv(cx, s + "/shortcut", p, nullptr, 1, nullptr); res_stride = 1; }
  }
  Act r = run_conv(cx, s + "/conv1", p, nullptr, 1, nullptr);
  if (stop == UP_CONV1) return r;
  r = run_conv(cx, s + "/conv2", r, nullptr, 1, nullptr);
  if (stop == UP_CONV2) return r;
  return run_conv(cx, s + "/conv3", r, stop == UP_UNIT ? &shortcut : nullptr, res_stride, nullptr, nullptr, -1.0,
                  next);
}

// ---------------------------------------------------------------- Faster R-CNN forward
void ensure_frcnn_anchors(lumi_engine* e, int h, int w, cudaStream_t st) {
  // fasterrcnn.py:261-308; the grid follows the endpoint's feature map.
  // One buffer per grid shape, kept for the engine's lifetime: captured graphs of other image sizes keep pointing
  // at theirs (a server sees a handful of distinct sizes).
  const int fh = feature_size(e, h), fw = feature_size(e, w);
  if (e->anchors_fh == fh && e->anchors_fw == fw) return;
  auto it = e->anchor_grids.find({fh, fw});
  if (it == e->anchor_grids.end()) {
    if (e->anchor_grids.size() >= 64) {          // bound the cache: forget everything (and the graphs that used it)
      e->drop_graphs();
      LUMI_CUDA_CHECK(cudaStreamSynchronize(e->stream));
      if (e->stream2) LUMI_CUDA_CHECK(cudaStreamSynchronize(e->stream2));
      for (auto& kv : e->anchor_grids) cudaFree(kv.second);
      e->anchor_grids.clear();
    }
    const int na = fh * fw * e->A;
    float* buf = nullptr;
    LUMI_CUDA_CHECK(cudaMalloc(&buf, (size_t)na * 4 * sizeof(float)));
    launch_frcnn_anchors(e->d_anchor_ref, e->A, fh, fw, e->anchor_stride, buf, st);
    it = e->anchor_grids.emplace(std::make_pair(fh, fw), buf).first;
  }
  e->d_anchors = it->second;
  e->anchors_fh = fh; e->anchors_fw = fw;
}

void forward_frcnn(Ctx& cx, const void* images, int n, int h, int w) {
  lumi_engine* e = cx.e;
  const int io = cx.img_off;                      // this (half-)batch's slice of the engine-level buffers
  int* prop_counts = e->d_prop_counts + io;
  float* out_boxes = e->d_boxes + (size_t)io * e->kmax * 4;
  float* out_scores = e->d_scores + (size_t)io * e->kmax;
  int* out_labels = e->d_labels + (size_t)io * e->kmax;
  int* out_counts = e->d_counts + io;
  float* out_records = e->d_records ? e->d_records + (size_t)io * (1 + 6 * (size_t)e->kmax) : nullptr;
  const std::string root = "truncated_base_network/" + e->arch;
  const int* units = e->resnet->units;
  const bool v2 = e->resnet->preact;
  Act x;
  if (e->conv_impl == 1) {
    // stem on the tensor cores: mean-subtract + zero-pad + space-to-depth staging, then 4 taps of K=64
    const int ho = (h + 6 - 7) / 2 + 1, wo = (w + 6 - 7) / 2 + 1;
    Act x2 = cx.act(n, ho + 3, wo + 3, 16);
    if (!cx.dry) { ProfScope ps(cx.e, cx.dry, PC_PREP); launch_stem_s2d(images, cx.img_f32, n, h, w, x2, RGB_MEANS, cx.st); }
    Act view = x2;                      // Toeplitz view: pixel (y, x) -> the 64 contiguous fp16 starting at x2[y][x]
    view.w = wo; view.c = 64;
    const long pitch[3] = {16, (long)(wo + 3) * 16, (long)(ho + 3) * (wo + 3) * 16};
    x = run_conv(cx, root + "/conv1#s2d", view, nullptr, 1, nullptr, pitch, 2.0 * n * ho * wo * 147.0 * 64.0);
  } else {
    x = cx.act(n, h, w, 3);
    if (!cx.dry) { ProfScope ps(cx.e, cx.dry, PC_PREP); launch_u8_to_act(images, cx.img_f32, x, RGB_MEANS, cx.st); }  // base_network.py:153-177
    x = run_conv(cx, root + "/conv1", x, nullptr, 1, nullptr);           // conv2d_same(64, 7, stride 2) + BN + relu
  }                                                                      // (v2: + bias, no activation)
  const Endpoint& ep = e->ep;
  if (ep.block < 0) {
    // the stem conv is the endpoint
  } else if (!v2) {
    x = run_pool(cx, x, 3, 2, true);                                     // pool1 3x3/2 SAME
    for (int b = 0; b <= ep.block; ++b)
      for (int u = 0; u < units[b]; ++u) {
        const bool at_ep = b == ep.block && u == ep.unit;
        x = bottleneck_v2(cx, unit_scope(e, b, u), x, x, BASE_DEPTH[b] * 4, nullptr, at_ep ? ep.part : UP_UNIT);
        if (at_ep) break;
      }
  } else {
    // block1/unit_1 projects from its preact: the stem's pool emits only p = relu(BN(pool1))
    const PreAct first = preact_of(e, unit_scope(e, 0, 0), false);
    Act p = run_pool(cx, x, 3, 2, true, &first);
    x = Act();
    for (int b = 0; b <= ep.block; ++b)
      for (int u = 0; u < units[b]; ++u) {
        const bool last_of_block = u + 1 == units[b];
        if (b == ep.block && u == ep.unit) {                             // the endpoint: x only
          x = bottleneck_v2(cx, unit_scope(e, b, u), x, p, BASE_DEPTH[b] * 4, nullptr, ep.part);
          break;
        }
        // the next unit's shortcut is the identity (reads x) unless it opens the next block (projects from p)
        PreAct next = last_of_block ? preact_of(e, unit_scope(e, b + 1, 0), false)
                                    : preact_of(e, unit_scope(e, b, u + 1), true);
        x = bottleneck_v2(cx, unit_scope(e, b, u), x, p, BASE_DEPTH[b] * 4, &next);
        p = next.p;
      }
  }
  const Act fmap = x;                                                    // the endpoint
  cx.tap_act("conv_feature_map", fmap);
  const int fh = fmap.h, fw = fmap.w;

  // anchors (fasterrcnn.py:261-308): made by ensure_frcnn_anchors() before the forward starts
  const int na = fh * fw * e->A;
  if (!cx.dry) LUMI_REQUIRE(e->anchors_fh == fh && e->anchors_fw == fw, "anchor grid mismatch (internal)");
  cx.tap_f32("all_anchors", e->d_anchors, na, 4, 1, 1);

  // RPN (rpn.py:136-180): 3x3 conv + act, fused 1x1 heads [cls 2A | bbox 4A], softmax fused into the decode
  Act rf = run_conv(cx, "fasterrcnn/rpn/conv", fmap, nullptr, 1, nullptr);
  float* heads = nullptr;
  run_conv(cx, "fasterrcnn/rpn/heads", rf, nullptr, 1, &heads);
  const int hc = 6 * e->A;
  cx.tap_f32("rpn_heads", heads, n, fh * fw, hc, 1);

  RpnParams rp = e->rpn;
  rp.na = na; rp.im_h = (float)h; rp.im_w = (float)w; rp.logits = 1;
  rp.cls_stride = hc; rp.cls_off = 0; rp.box_stride = hc; rp.box_off = 2 * e->A;
  const int post = rp.post_nms_top_n;
  float* proposals = cx.f32((size_t)n * post * 4);
  float* pscores = cx.f32((size_t)n * post);
  if (!cx.dry) {
    LUMI_REQUIRE(na <= e->ws_rpn.cap, "image too large for the RPN workspace (max_h/max_w at lumi_create)");
    NmsWorkspace wsr = ws_view(e->ws_rpn, io);
    // algorithmic bytes (SURVEY 8d): decode N*(36 in + 20 out), sort N*4 + K*20, bitmask NMS K*16 + 2*K*ceil(K/64)*8 + P*4
    const double kk = std::min(na, rp.pre_nms_top_n);
    const double bytes = (double)n * (56.0 * na + 4.0 * na + 20.0 * kk + 16.0 * kk + 16.0 * kk * std::ceil(kk / 64.0) + 4.0 * post);
    ProfScope ps(cx.e, cx.dry, PC_RPN_POST, bytes);
    launch_rpn_proposals(heads, heads, (long)fh * fw * hc, (long)fh * fw * hc, e->A, e->d_anchors, n, rp, wsr,
                         proposals, pscores, prop_counts, cx.st);
  }
  cx.tap_f32("proposals", proposals, n, post, 4, 1);
  cx.tap_f32("proposal_scores", pscores, n, post, 1, 1);
  cx.tap_i32("proposal_counts", prop_counts, n);
  cx.tap_f32("rpn_sorted_scores", e->ws_rpn.sscores, n, e->ws_rpn.ncap, 1, 1);
  cx.tap_i32("rpn_sorted_counts", e->ws_rpn.nvalid, n);

  if (!e->with_rcnn) {
    if (!cx.dry) {     // predicting.py:85-92: objects = proposals, probs = scores, labels = 0
      LUMI_CUDA_CHECK(cudaMemcpyAsync(out_boxes, proposals, (size_t)n * post * 4 * sizeof(float),
                                      cudaMemcpyDeviceToDevice, cx.st));
      LUMI_CUDA_CHECK(cudaMemcpyAsync(out_scores, pscores, (size_t)n * post * sizeof(float), cudaMemcpyDeviceToDevice,
                                      cx.st));
      LUMI_CUDA_CHECK(cudaMemsetAsync(out_labels, 0, (size_t)n * post * sizeof(int), cx.st));
      LUMI_CUDA_CHECK(cudaMemcpyAsync(out_counts, prop_counts, n * sizeof(int), cudaMemcpyDeviceToDevice, cx.st));
      if (out_records) launch_pack_records(out_boxes, out_scores, out_labels, out_counts, n, e->kmax, out_records, cx.st);
    }
    return;
  }

  // RCNN (rcnn.py:174-232)
  const bool fuse_mean = e->use_mean && !e->tail;                         // ROI crop+max-pool+mean in one kernel
  const bool need_pooled = !fuse_mean || e->debug_taps;
  Act pooled, feat;
  float* fmap_f32 = cx.f32(fmap.numel());                                  // gather source of the ROI kernel
  if (need_pooled) pooled = cx.act(n * post, e->pooled_w, e->pooled_h, fmap.c);
  if (fuse_mean) feat = cx.act(n * post, 1, 1, fmap.c);
  if (!cx.dry) {
    // algorithmic bytes (SURVEY 8d): feature map once + rois + output (fp16x2 planes = 4 B / element)
    const double bytes = 4.0 * fmap.numel() + 16.0 * n * post + 4.0 * (double)(need_pooled ? pooled.numel() : 0) +
                         4.0 * (double)(fuse_mean ? feat.numel() : 0);
    ProfScope ps(cx.e, cx.dry, PC_ROI, bytes);
    launch_act_to_f32(fmap, fmap_f32, cx.st);
    launch_roi_pool(fmap_f32, fmap.n, fmap.h, fmap.w, fmap.c, proposals, prop_counts, post, (float)h, (float)w,
                    e->pooled_h, e->pooled_w, pooled, fuse_mean ? feat : Act(), cx.st);
  }
  if (need_pooled) cx.tap_act("roi_pool", pooled);
  if (!fuse_mean) {
    feat = pooled;
    if (e->tail)                                                         // truncated_base_network.py:56-95
      for (int u = 0; u < 3; ++u)
        feat = bottleneck_v2(cx, root + "/block4/unit_" + std::to_string(u + 1) + "/bottleneck_v1", feat, feat, 2048,
                             nullptr);
    if (e->use_mean) {
      Act m = cx.act(feat.n, 1, 1, feat.c);
      if (!cx.dry) { ProfScope ps(cx.e, cx.dry, PC_HEAD_MISC); launch_spatial_mean(feat, m, cx.st); }
      feat = m;
    } else {
      feat.c = feat.h * feat.w * feat.c; feat.h = 1; feat.w = 1;         // flatten (NHWC order == tf flatten)
    }
  }
  cx.tap_act("rcnn_features", feat);
  for (size_t i = 0; i < e->fc_sizes.size(); ++i)
    feat = run_conv(cx, "fasterrcnn/rcnn/fc_" + std::to_string(i), feat, nullptr, 1, nullptr);
  float* fc = nullptr;
  run_conv(cx, "fasterrcnn/rcnn/heads", feat, nullptr, 1, &fc);
  const int C = e->num_classes, fcw = 5 * C + 1;
  float* cls_prob = cx.f32((size_t)n * post * (C + 1));
  if (!cx.dry) { ProfScope ps(cx.e, cx.dry, PC_HEAD_MISC); launch_softmax_rows(fc, cls_prob, n * post, C + 1, fcw, cx.st); }
  cx.tap_f32("rcnn_cls_prob", cls_prob, n, post, C + 1, 1);
  cx.tap_f32("rcnn_fc", fc, n, post, fcw, 1);
  DetParams dp = e->det;
  dp.r = post; dp.im_h = (float)h; dp.im_w = (float)w;
  dp.prob_stride = C + 1; dp.delta_stride = fcw;
  if (!cx.dry) {
    ProfScope ps(cx.e, cx.dry, PC_DET_POST);
    NmsWorkspace wsd = ws_view(e->ws_det, io * C);
    launch_class_detections(proposals, (long)post * 4, prop_counts, fc + (C + 1), cls_prob, n, dp, wsd, cx.final_keys,
                            out_boxes, out_labels, out_scores, out_counts, cx.st, out_records);
  }
}

// ---------------------------------------------------------------- SSD forward
__global__ void ssd_repack_kernel(const float* __restrict__ head, int cells, int A, int nc1, int total, int off,
                                  float* __restrict__ loc, float* __restrict__ cls) {
  // head [n][cells][4A + nc1*A] -> loc [n][total][4], cls [n][total][nc1] at anchor offset `off`
  const int img = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int per_cell = A * (4 + nc1);
  if (i >= cells * per_cell) return;
  const int cell = i / per_cell, j = i % per_cell;
  const float v = head[((size_t)img * cells + cell) * per_cell + j];
  if (j < 4 * A) {
    loc[((size_t)img * total + off + (size_t)cell * A) * 4 + j] = v;
  } else {
    cls[((size_t)img * total + off + (size_t)cell * A) * nc1 + (j - 4 * A)] = v;
  }
}

void ssd_fmap_shapes(int h, int w, int (&fh)[6], int (&fw)[6]) {
  int a = h, b = w;
  for (int i = 0; i < 3; ++i) { a = tf_valid(a, 2, 2, 1); b = tf_valid(b, 2, 2, 1); }   // 300 -> 37 (quirk Q8)
  fh[0] = a; fw[0] = b;
  a = tf_valid(a, 2, 2, 1); b = tf_valid(b, 2, 2, 1);                                   // 18
  fh[1] = a; fw[1] = b;
  int d;
  tf_same(a, 3, 2, 1, a, d); tf_same(b, 3, 2, 1, b, d); fh[2] = a; fw[2] = b;           // 9
  tf_same(a, 3, 2, 1, a, d); tf_same(b, 3, 2, 1, b, d); fh[3] = a; fw[3] = b;           // 5
  a = tf_valid(a, 3, 1, 1); b = tf_valid(b, 3, 1, 1); fh[4] = a; fw[4] = b;             // 3
  a = tf_valid(a, 3, 1, 1); b = tf_valid(b, 3, 1, 1); fh[5] = a; fw[5] = b;             // 1
}

void compute_ssd_anchors(lumi_engine* e) {
  // ssd/utils.py:5-145 + ssd.py:112-129, float64 until the final float32 cast
  int fh[6], fw[6];
  ssd_fmap_shapes(e->fixed_h, e->fixed_w, fh, fw);
  for (int i = 0; i < 6; ++i) LUMI_REQUIRE(fh[i] > 0 && fw[i] > 0, "SSD input too small");
  const double mn = e->cfg.number("model.anchors.min_scale", 0.1), mx = e->cfg.number("model.anchors.max_scale", 0.88);
  std::vector<double> ratios = e->cfg.numbers("model.anchors.ratios");
  double scales[6];
  const double step = (mx - mn) / 5.0;
  for (int i = 0; i < 6; ++i) scales[i] = i * step + mn;
  scales[5] = mx;
  std::vector<float>& out = e->ssd_anchor_host;
  out.clear();
  for (int i = 0; i < 6; ++i) {
    const int A = e->ssd_app[i];
    LUMI_REQUIRE((int)ratios.size() >= A - 1, "model.anchors.ratios too short for anchors_per_point");
    std::vector<double> hs(A), wsz(A);
    if (i < 5) { hs[0] = wsz[0] = std::sqrt(scales[i] * scales[i + 1]) * fh[i]; }
    else { hs[0] = scales[i] * fh[i] * 0.99; wsz[0] = scales[i] * fw[i] * 0.99; }
    for (int a = 1; a < A; ++a) {
      hs[a] = scales[i] / std::sqrt(ratios[a - 1]) * fh[i];
      wsz[a] = scales[i] * std::sqrt(ratios[a - 1]) * fw[i];
    }
    const double H = e->fixed_h, Wd = e->fixed_w;
    for (int y = 0; y < fh[i]; ++y)
      for (int x = 0; x < fw[i]; ++x)
        for (int a = 0; a < A; ++a) {
          double b[4] = {0.5 - wsz[a] / 2 + x, 0.5 - hs[a] / 2 + y, 0.5 + wsz[a] / 2 + x, 0.5 + hs[a] / 2 + y};
          b[0] = b[0] / fw[i] * Wd; b[1] = b[1] / fh[i] * H; b[2] = b[2] / fw[i] * Wd; b[3] = b[3] / fh[i] * H;
          b[0] = std::fmax(std::fmin(b[0], Wd - 1), 0.0); b[2] = std::fmax(std::fmin(b[2], Wd - 1), 0.0);
          b[1] = std::fmax(std::fmin(b[1], H - 1), 0.0);  b[3] = std::fmax(std::fmin(b[3], H - 1), 0.0);
          for (double v : b) out.push_back((float)v);
        }
  }
  e->ssd_total_anchors = (int)(out.size() / 4);
}

void forward_ssd(Ctx& cx, const void* images, int n, int h, int w) {
  lumi_engine* e = cx.e;
  LUMI_REQUIRE(h == e->fixed_h && w == e->fixed_w, "SSD expects images of the configured fixed size");
  const std::string s = "ssd/ssd_feature_extractor";
  Act x;
  const bool c11_tc = e->conv_impl == 1;
  if (c11_tc) {
    // conv1_1 on the tensor cores: zero-padded 16-channel staging, Toeplitz view, 3 filter rows of K=64
    Act x2 = cx.act(n, h + 2, w + 3, 16);
    if (!cx.dry) { ProfScope ps(cx.e, cx.dry, PC_PREP); launch_pack_c3(images, cx.img_f32, n, h, w, x2, cx.st); }   // no mean subtraction (quirk Q7)
    Act view = x2;
    view.w = w; view.c = 64;
    const long pitch[3] = {16, (long)(w + 3) * 16, (long)(h + 2) * (w + 3) * 16};
    x = run_conv(cx, s + "/vgg_16/conv1/conv1_1#pack", view, nullptr, 1, nullptr, pitch, 2.0 * n * h * w * 27.0 * 64.0);
  } else {
    x = cx.act(n, h, w, 3);
    if (!cx.dry) { ProfScope ps(cx.e, cx.dry, PC_PREP); launch_u8_to_act(images, cx.img_f32, x, nullptr, cx.st); }  // no mean subtraction (quirk Q7)
  }
  Act fmaps[6];
  for (int b = 0; b < 5; ++b) {
    for (int r = (b == 0 && c11_tc) ? 1 : 0; r < VGG_REPS[b]; ++r)
      x = run_conv(cx, s + "/vgg_16/" + VGG_NAMES[b] + "/" + VGG_NAMES[b] + "_" + std::to_string(r + 1), x, nullptr, 1,
                   nullptr);
    if (b == 3) {                                                         // conv4_3 -> l2norm x gamma
      Act nrm = cx.act(x.n, x.h, x.w, x.c);
      if (!cx.dry) { ProfScope ps(cx.e, cx.dry, PC_HEAD_MISC); launch_l2norm_scale(x, nrm, e->dev_vecs.at("gamma"), 1e-12f, cx.st); }
      fmaps[0] = nrm;
    }
    if (b < 4) x = run_pool(cx, x, 2, 2, false);                          // slim default VALID (quirk Q8)
  }
  x = run_pool(cx, x, 3, 1, true);                                        // pool5 3x3/1 SAME
  const std::string ex = s + "/extra_feature_layers/";
  int fi = 1;
  for (int i = 0; i < 10; ++i) {
    x = run_conv(cx, ex + SSD_EXTRAS[i].name, x, nullptr, 1, nullptr);
    if (i == 1 || i == 3 || i == 5 || i == 7 || i == 9) fmaps[fi++] = x;
  }
  const int C1 = e->num_classes + 1, total = e->ssd_total_anchors;
  float* loc = cx.f32((size_t)n * total * 4);
  float* cls = cx.f32((size_t)n * total * C1);
  int off = 0;
  for (int i = 0; i < 6; ++i) {
    cx.tap_act("fmap_" + std::to_string(i), fmaps[i]);
    float* head = nullptr;
    Act o = run_conv(cx, "ssd/MultiBox_" + std::to_string(i), fmaps[i], nullptr, 1, &head);
    const int A = e->ssd_app[i], cells = o.h * o.w, per_cell = A * (4 + C1);
    if (!cx.dry) {
      ProfScope ps(cx.e, cx.dry, PC_HEAD_MISC);
      dim3 g(cdiv(cells * per_cell, 256), n);
      ssd_repack_kernel<<<g, 256, 0, cx.st>>>(head, cells, A, C1, total, off, loc, cls);
      count_launch();
      LUMI_CUDA_CHECK(cudaGetLastError());
    }
    off += cells * A;
  }
  LUMI_REQUIRE(off == total, "SSD anchor count mismatch (internal)");
  float* prob = cx.f32((size_t)n * total * C1);
  if (!cx.dry) { ProfScope ps(cx.e, cx.dry, PC_HEAD_MISC); launch_softmax_rows(cls, prob, n * total, C1, C1, cx.st); }
  cx.tap_f32("loc_pred", loc, n, total, 4, 1);
  cx.tap_f32("cls_prob", prob, n, total, C1, 1);
  cx.tap_f32("all_anchors", e->d_ssd_anchors, total, 4, 1, 1);
  DetParams dp = e->det;
  dp.r = total; dp.im_h = (float)h; dp.im_w = (float)w; dp.prob_stride = C1; dp.delta_stride = 4;
  if (!cx.dry) {
    ProfScope ps(cx.e, cx.dry, PC_DET_POST);
    const int io = cx.img_off;
    NmsWorkspace wsd = ws_view(e->ws_det, io * e->num_classes);
    launch_class_detections(e->d_ssd_anchors, 0, nullptr, loc, prob, n, dp, wsd, cx.final_keys,
                            e->d_boxes + (size_t)io * e->kmax * 4, e->d_labels + (size_t)io * e->kmax,
                            e->d_scores + (size_t)io * e->kmax, e->d_counts + io, cx.st,
                            e->d_records ? e->d_records + (size_t)io * (1 + 6 * (size_t)e->kmax) : nullptr);
  }
}

void forward(Ctx& cx, const void* images, int n, int h, int w) {
  cx.arena->off = 0;
  if (cx.taps) cx.e->taps.clear();
  if (cx.e->type == "fasterrcnn") forward_frcnn(cx, images, n, h, w);
  else forward_ssd(cx, images, n, h, w);
}

Ctx make_ctx(lumi_engine* e, bool dry, int half) {
  Ctx cx;
  cx.e = e; cx.dry = dry;
  cx.st = half ? e->stream2 : e->stream;
  cx.arena = half ? &e->arena2 : &e->arena;
  cx.final_keys = half ? e->d_final_keys2 : e->d_final_keys;
  cx.sk = &e->sk_ws[half ? 1 : 0];
  cx.taps = half == 0;
  return cx;
}

void ensure_arena(lumi_engine* e, Arena& a, size_t need_bytes) {
  if (need_bytes <= a.cap) return;
  e->drop_graphs();                            // captured nodes point into the old arena
  LUMI_CUDA_CHECK(cudaStreamSynchronize(e->stream));
  if (e->stream2) LUMI_CUDA_CHECK(cudaStreamSynchronize(e->stream2));
  cudaFree(a.base);
  a.base = nullptr; a.cap = 0;
  LUMI_CUDA_CHECK(cudaMalloc(&a.base, need_bytes));
  a.cap = need_bytes;
}

// max_h x max_w at lumi_create is a sizing HINT, not a limit: the reference's resize_image multiplies its up- and
// down-scale factors (utils/image.py:66-86), so e.g. a 300x600 input becomes 600x1200 -- beyond max_size.  The
// RPN workspace (the only buffer sized by the image) grows on demand; arenas are re-planned per shape anyway.
void ensure_image_capacity(lumi_engine* e, int h, int w) {
  if (e->type != "fasterrcnn") return;                 // SSD runs at its configured fixed size only
  const long na = (long)feature_size(e, h) * feature_size(e, w) * e->A;
  LUMI_REQUIRE(na < (1L << 30), "lumi_predict: image too large");
  if (na <= e->ws_rpn.cap) return;
  e->drop_graphs();
  LUMI_CUDA_CHECK(cudaStreamSynchronize(e->stream));
  if (e->stream2) LUMI_CUDA_CHECK(cudaStreamSynchronize(e->stream2));
  nms_workspace_free(e->ws_rpn);
  nms_workspace_alloc(e->ws_rpn, e->max_batch, (int)na, e->rpn.post_nms_top_n, std::min((int)na, e->rpn.pre_nms_top_n));
  e->max_h = std::max(e->max_h, h); e->max_w = std::max(e->max_w, w);
}

int fail(lumi_engine* e, const Error& err) {
  if (e) e->last_error = err.what(); else g_create_error = err.what();
  return err.code;
}
int fail(lumi_engine* e, int code, const std::string& msg) {
  if (e) e->last_error = msg; else g_create_error = msg;
  return code;
}

#define LUMI_API_BEGIN try {
#define LUMI_API_END(e)                                                   \
  }                                                                       \
  catch (const Error& err) { return fail(e, err); }                       \
  catch (const std::exception& ex) { return fail(e, LUMI_EINVAL, ex.what()); }

}  // namespace

// ======================================================================================
// C ABI
// ======================================================================================
extern "C" {

const char* lumi_version(void) { return "luminoth_b200 0.1 (sm_90a)"; }

int lumi_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

int lumi_create(const char* cfg_json, int device, int max_batch, int max_h, int max_w, lumi_engine** out) {
  lumi_engine* e = nullptr;
  LUMI_API_BEGIN
  LUMI_REQUIRE(cfg_json && out, "lumi_create: null argument");
  LUMI_REQUIRE(max_batch > 0 && max_h > 0 && max_w > 0, "lumi_create: max_batch/max_h/max_w must be positive");
  std::unique_ptr<lumi_engine> eng(new lumi_engine());
  std::string s(cfg_json);
  eng->cfg = JParser(s).parse();
  eng->device = device; eng->max_batch = max_batch; eng->max_h = max_h; eng->max_w = max_w;
  parse_config(eng.get());
  if (eng->type == "ssd") compute_ssd_anchors(eng.get());
  build_net(eng.get());
  build_specs(eng.get());
  int ndev = lumi_device_count();
  if (ndev <= 0) throw Error(LUMI_ECUDA, "no CUDA device visible: the luminoth_b200 engine has no CPU fallback");
  LUMI_REQUIRE(device >= 0 && device < ndev, "lumi_create: invalid device index");
  LUMI_CUDA_CHECK(cudaSetDevice(device));
  LUMI_CUDA_CHECK(cudaStreamCreateWithFlags(&eng->stream, cudaStreamNonBlocking));
  *out = eng.release();
  return LUMI_OK;
  LUMI_API_END(e)
}

int lumi_set_weight(lumi_engine* e, const char* name, const float* data, const int64_t* shape, int ndim) {
  if (!e) return LUMI_EINVAL;
  LUMI_API_BEGIN
  LUMI_REQUIRE(!e->finalized, "lumi_set_weight after lumi_finalize");
  LUMI_REQUIRE(name && data && shape && ndim >= 1 && ndim <= 4, "lumi_set_weight: bad argument");
  const WeightSpec* spec = nullptr;
  for (const auto& w : e->required) if (w.name == name) { spec = &w; break; }
  if (!spec) return LUMI_OK;    // variables the inference graph does not use are ignored (Saver(allow_empty) spirit)
  std::vector<int64_t> shp(shape, shape + ndim);
  if (shp != spec->shape) {
    std::string m = "variable '" + std::string(name) + "' has shape [";
    for (auto d : shp) m += std::to_string(d) + ",";
    m += "] but the graph expects [";
    for (auto d : spec->shape) m += std::to_string(d) + ",";
    throw Error(LUMI_EINVAL, m + "]");
  }
  size_t count = 1;
  for (auto d : shp) count *= (size_t)d;
  HostTensor t;
  t.shape = shp;
  t.v.assign(data, data + count);
  e->staged[name] = std::move(t);
  return LUMI_OK;
  LUMI_API_END(e)
}

int lumi_num_weights(lumi_engine* e) { return e ? (int)e->required.size() : 0; }

int lumi_weight_info(lumi_engine* e, int index, const char** name, int64_t* shape4, int* ndim) {
  if (!e || index < 0 || index >= (int)e->required.size()) return LUMI_EINVAL;
  const WeightSpec& w = e->required[index];
  if (name) *name = w.name.c_str();
  if (ndim) *ndim = (int)w.shape.size();
  if (shape4) for (size_t i = 0; i < 4; ++i) shape4[i] = i < w.shape.size() ? w.shape[i] : 1;
  return LUMI_OK;
}

int lumi_finalize(lumi_engine* e) {
  if (!e) return LUMI_EINVAL;
  LUMI_API_BEGIN
  LUMI_REQUIRE(!e->finalized, "lumi_finalize called twice");
  LUMI_CUDA_CHECK(cudaSetDevice(e->device));
  for (const auto& w : e->required)
    if (!e->staged.count(w.name)) throw Error(LUMI_ENOWEIGHT, "variable '" + w.name + "' was never set");
  build_layers(e);
  e->staged.clear();
  LUMI_CUDA_CHECK(cudaMalloc(&e->d_overflow, sizeof(int)));
  LUMI_CUDA_CHECK(cudaMemset(e->d_overflow, 0, sizeof(int)));
  const int nb = e->max_batch;
  LUMI_CUDA_CHECK(cudaMalloc(&e->d_boxes, (size_t)nb * e->kmax * 4 * sizeof(float)));
  LUMI_CUDA_CHECK(cudaMalloc(&e->d_scores, (size_t)nb * e->kmax * sizeof(float)));
  LUMI_CUDA_CHECK(cudaMalloc(&e->d_labels, (size_t)nb * e->kmax * sizeof(int)));
  LUMI_CUDA_CHECK(cudaMalloc(&e->d_counts, nb * sizeof(int)));
  LUMI_CUDA_CHECK(cudaMalloc(&e->d_prop_counts, nb * sizeof(int)));
  if (e->type == "fasterrcnn") {
    LUMI_CUDA_CHECK(cudaMalloc(&e->d_anchor_ref, e->anchor_ref.size() * sizeof(int)));
    LUMI_CUDA_CHECK(cudaMemcpy(e->d_anchor_ref, e->anchor_ref.data(), e->anchor_ref.size() * sizeof(int),
                               cudaMemcpyHostToDevice));
    const int fh = feature_size(e, e->max_h), fw = feature_size(e, e->max_w);
    nms_workspace_alloc(e->ws_rpn, nb, fh * fw * e->A, e->rpn.post_nms_top_n,
                        std::min(fh * fw * e->A, e->rpn.pre_nms_top_n));
    if (e->with_rcnn) {
      nms_workspace_alloc(e->ws_det, nb * e->num_classes, e->rpn.post_nms_top_n, e->det.class_max);
      LUMI_CUDA_CHECK(cudaMalloc(&e->d_final_keys, det_final_scratch_bytes(nb, e->num_classes, e->det.class_max)));
    }
  } else {
    LUMI_CUDA_CHECK(cudaMalloc(&e->d_ssd_anchors, e->ssd_anchor_host.size() * sizeof(float)));
    LUMI_CUDA_CHECK(cudaMemcpy(e->d_ssd_anchors, e->ssd_anchor_host.data(), e->ssd_anchor_host.size() * sizeof(float),
                               cudaMemcpyHostToDevice));
    nms_workspace_alloc(e->ws_det, nb * e->num_classes, e->ssd_total_anchors, e->det.class_max);
    LUMI_CUDA_CHECK(cudaMalloc(&e->d_final_keys, det_final_scratch_bytes(nb, e->num_classes, e->det.class_max)));
  }
  conv_workspace_create(e->sk_ws[0]);
  if (const char* v = std::getenv("LUMI_CONV_STREAMK")) e->conv_streamk = std::max(0, std::min(2, std::atoi(v)));
  if (const char* v = std::getenv("LUMI_CONV_2CTA")) e->conv_cta2 = std::max(0, std::atoi(v));
  if (const char* v = std::getenv("LUMI_CONV_HALO")) e->conv_halo = std::max(0, std::min(1, std::atoi(v)));
  if (const char* v = std::getenv("LUMI_CONV_HALO_PCT")) e->conv_halo_pct = std::max(0, std::atoi(v));
  if (const char* v = std::getenv("LUMI_CONV_EPI16")) e->conv_epi16 = std::max(0, std::atoi(v));
  if (const char* v = std::getenv("LUMI_CONV_PIPE")) e->conv_pipe = std::atoi(v) != 0;
  if (const char* v = std::getenv("LUMI_CONV_EPI_TMA")) e->conv_epi_tma = std::atoi(v) != 0;
  if (const char* v = std::getenv("LUMI_GRAPHS")) e->use_graphs = std::atoi(v) != 0;
  if (e->max_batch >= 2) {
    conv_workspace_create(e->sk_ws[1]);
    LUMI_CUDA_CHECK(cudaStreamCreateWithFlags(&e->stream2, cudaStreamNonBlocking));
    LUMI_CUDA_CHECK(cudaEventCreateWithFlags(&e->ev_fork, cudaEventDisableTiming));
    LUMI_CUDA_CHECK(cudaEventCreateWithFlags(&e->ev_join, cudaEventDisableTiming));
    if (e->d_final_keys)
      LUMI_CUDA_CHECK(cudaMalloc(&e->d_final_keys2, det_final_scratch_bytes(nb, e->num_classes, e->det.class_max)));
  }
  e->finalized = true;
  return LUMI_OK;
  LUMI_API_END(e)
}

// One (half-)batch forward on cx.st: eager the first time a shape is seen (tensor maps, function attributes and the
// arena plan settle), captured into a CUDA graph the second time, replayed from then on.  A replay is ONE launch
// instead of ~40-75: the inter-kernel gaps (2-3 us each) and the CPU launch cost disappear, which is what bounds the
// small-batch latency (`lumi predict` on single images, video frames).  Everything a node bakes in is part of the key.
static void run_forward(lumi_engine* e, Ctx& cx, int half, const void* images, int n, int h, int w, int esz) {
  const bool graphable = e->use_graphs && !e->profile && !e->debug_taps;
  if (!graphable) { forward(cx, images, n, h, w); return; }
  lumi_engine::GraphKey key{half, n, h, w, esz, cx.img_off, e->conv_impl, e->conv_streamk, cx.sm_reserve, e->d_records};
  lumi_engine::GraphEntry& ent = e->graphs[key];
  if (ent.exec) {
    LUMI_CUDA_CHECK(cudaGraphLaunch(ent.exec, cx.st));
    g_launch_count += ent.launches;
    e->graph_replays++;
    return;
  }
  if (ent.seen++ == 0) { forward(cx, images, n, h, w); return; }     // first sight: eager warm-up of this shape
  const int before = g_launch_count;
  cudaGraph_t graph = nullptr;
  LUMI_CUDA_CHECK(cudaStreamBeginCapture(cx.st, cudaStreamCaptureModeThreadLocal));
  try {
    forward(cx, images, n, h, w);
  } catch (...) {
    cudaStreamEndCapture(cx.st, &graph);
    if (graph) cudaGraphDestroy(graph);
    cudaGetLastError();
    throw;
  }
  LUMI_CUDA_CHECK(cudaStreamEndCapture(cx.st, &graph));
  cudaGraphExec_t exec = nullptr;
  cudaError_t ce = cudaGraphInstantiate(&exec, graph, 0);
  cudaGraphDestroy(graph);
  LUMI_CUDA_CHECK(ce);
  ent.exec = exec;
  ent.launches = g_launch_count - before;
  LUMI_CUDA_CHECK(cudaGraphLaunch(ent.exec, cx.st));
  e->graph_replays++;
}

static int predict_impl(lumi_engine* e, const void* images, int esz, int images_on_device, int n, int h, int w,
                        float* boxes, float* scores, int* labels, int* counts, int outputs_on_device) {
  if (!e) return LUMI_EINVAL;
  LUMI_API_BEGIN
  if (!e->finalized) throw Error(LUMI_ESTATE, "lumi_predict before lumi_finalize");
  LUMI_REQUIRE(images && boxes && scores && labels && counts, "lumi_predict: null buffer");
  LUMI_REQUIRE(n > 0 && n <= e->max_batch, "lumi_predict: batch size exceeds max_batch");
  LUMI_REQUIRE(h > 0 && w > 0, "lumi_predict: empty image");
  LUMI_CUDA_CHECK(cudaSetDevice(e->device));
  ensure_image_capacity(e, h, w);
  // software pipelining: two half-batches on two streams (off while profiling / tapping intermediates)
  const bool piped = e->pipeline && n >= 2 && !e->profile && !e->debug_taps && e->stream2 != nullptr;
  const int nA = piped ? (n + 1) / 2 : n, nB = n - nA;
  const int plan_key = piped ? -n : n;
  if (plan_key != e->planned_n || h != e->planned_h || w != e->planned_w) {   // size the arenas for this shape
    Ctx dry = make_ctx(e, true, 0);
    forward(dry, nullptr, nA, h, w);
    const size_t need_bytes = e->arena.off + 4096;
    ensure_arena(e, e->arena, need_bytes);
    if (piped) ensure_arena(e, e->arena2, need_bytes);
    e->planned_n = plan_key; e->planned_h = h; e->planned_w = w;
  }
  const uint8_t* dimg = static_cast<const uint8_t*>(images);
  const size_t img_bytes = (size_t)n * h * w * 3 * esz;
  const size_t bytes_a = (size_t)nA * h * w * 3 * esz;
  // graphs read their pixels from the engine's own staging buffer (a caller's device pointer changes per call)
  const bool graphs_on = e->use_graphs && !e->profile && !e->debug_taps;
  const bool stage = !images_on_device || graphs_on;
  if (stage) {
    if (img_bytes > e->images_cap) {
      e->drop_graphs();
      LUMI_CUDA_CHECK(cudaStreamSynchronize(e->stream));
      if (e->stream2) LUMI_CUDA_CHECK(cudaStreamSynchronize(e->stream2));
      cudaFree(e->d_images);
      e->d_images = nullptr; e->images_cap = 0;
      LUMI_CUDA_CHECK(cudaMalloc(&e->d_images, img_bytes));
      e->images_cap = img_bytes;
    }
    dimg = e->d_images;
  }
  const cudaMemcpyKind up = images_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  g_launch_count = 0;
  e->graph_replays = 0;
  if (e->type == "fasterrcnn") ensure_frcnn_anchors(e, h, w, e->stream);
  Ctx cx = make_ctx(e, false, 0);
  cx.img_f32 = esz == 4;
  cx.sm_reserve = piped ? 8 : 0;
  if (piped) {
    LUMI_CUDA_CHECK(cudaEventRecord(e->ev_fork, e->stream));
    LUMI_CUDA_CHECK(cudaStreamWaitEvent(e->stream2, e->ev_fork, 0));
    Ctx cb = make_ctx(e, false, 1);
    cb.img_off = nA;
    cb.img_f32 = cx.img_f32;
    cb.sm_reserve = cx.sm_reserve;
    // each half uploads its own images on its own stream: the second half's H2D overlaps the first half's kernels
    if (stage) {
      LUMI_CUDA_CHECK(cudaMemcpyAsync(e->d_images, images, bytes_a, up, e->stream));
      LUMI_CUDA_CHECK(cudaMemcpyAsync(e->d_images + bytes_a, static_cast<const uint8_t*>(images) + bytes_a,
                                      img_bytes - bytes_a, up, e->stream2));
    }
    run_forward(e, cx, 0, dimg, nA, h, w, esz);
    run_forward(e, cb, 1, dimg + bytes_a, nB, h, w, esz);
    LUMI_CUDA_CHECK(cudaEventRecord(e->ev_join, e->stream2));
    LUMI_CUDA_CHECK(cudaStreamWaitEvent(e->stream, e->ev_join, 0));
  } else {
    if (stage) LUMI_CUDA_CHECK(cudaMemcpyAsync(e->d_images, images, img_bytes, up, e->stream));
    run_forward(e, cx, 0, dimg, n, h, w, esz);
  }
  e->launches = g_launch_count;
  const size_t k = (size_t)e->kmax;
  const cudaMemcpyKind kind = outputs_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
  LUMI_CUDA_CHECK(cudaMemcpyAsync(boxes, e->d_boxes, n * k * 4 * sizeof(float), kind, e->stream));
  LUMI_CUDA_CHECK(cudaMemcpyAsync(scores, e->d_scores, n * k * sizeof(float), kind, e->stream));
  LUMI_CUDA_CHECK(cudaMemcpyAsync(labels, e->d_labels, n * k * sizeof(int), kind, e->stream));
  LUMI_CUDA_CHECK(cudaMemcpyAsync(counts, e->d_counts, n * sizeof(int), kind, e->stream));
  if (!outputs_on_device) {
    int ovf = 0;
    LUMI_CUDA_CHECK(cudaMemcpyAsync(&ovf, e->d_overflow, sizeof(int), cudaMemcpyDeviceToHost, e->stream));
    LUMI_CUDA_CHECK(cudaStreamSynchronize(e->stream));
    if (ovf) {
      LUMI_CUDA_CHECK(cudaMemset(e->d_overflow, 0, sizeof(int)));
      throw Error(LUMI_EOVERFLOW, "an activation exceeded the fp16x2 split range (|x| > 65504); results are invalid");
    }
  }
  return LUMI_OK;
  LUMI_API_END(e)
}

int lumi_predict(lumi_engine* e, const void* images, int images_on_device, int n, int h, int w, float* boxes,
                 float* scores, int* labels, int* counts, int outputs_on_device) {
  return predict_impl(e, images, 1, images_on_device, n, h, w, boxes, scores, labels, counts, outputs_on_device);
}

int lumi_predict_f32(lumi_engine* e, const float* images, int images_on_device, int n, int h, int w, float* boxes,
                     float* scores, int* labels, int* counts, int outputs_on_device) {
  return predict_impl(e, images, 4, images_on_device, n, h, w, boxes, scores, labels, counts, outputs_on_device);
}

int lumi_max_detections(lumi_engine* e) { return e ? e->kmax : 0; }

int lumi_set_record_output(lumi_engine* e, float* device_records) {
  if (!e) return LUMI_EINVAL;
  e->d_records = device_records;
  return LUMI_OK;
}
void* lumi_stream(lumi_engine* e) { return e ? (void*)e->stream : nullptr; }

int lumi_synchronize(lumi_engine* e) {
  if (!e) return LUMI_EINVAL;
  LUMI_API_BEGIN
  LUMI_CUDA_CHECK(cudaSetDevice(e->device));
  LUMI_CUDA_CHECK(cudaStreamSynchronize(e->stream));
  int ovf = 0;
  if (e->d_overflow) {
    LUMI_CUDA_CHECK(cudaMemcpy(&ovf, e->d_overflow, sizeof(int), cudaMemcpyDeviceToHost));
    if (ovf) {
      LUMI_CUDA_CHECK(cudaMemset(e->d_overflow, 0, sizeof(int)));
      throw Error(LUMI_EOVERFLOW, "an activation exceeded the fp16x2 split range (|x| > 65504); results are invalid");
    }
  }
  return LUMI_OK;
  LUMI_API_END(e)
}

int lumi_last_launch_count(lumi_engine* e) { return e ? e->launches : 0; }

int lumi_set_pipeline(lumi_engine* e, int enable) {
  if (!e) return LUMI_EINVAL;
  e->pipeline = enable != 0;
  return LUMI_OK;
}

int lumi_set_graphs(lumi_engine* e, int enable) {
  if (!e) return LUMI_EINVAL;
  e->use_graphs = enable != 0;
  return LUMI_OK;
}

int lumi_last_graph_replays(lumi_engine* e) { return e ? e->graph_replays : 0; }

int lumi_set_debug_taps(lumi_engine* e, int enable) {
  if (!e) return LUMI_EINVAL;
  e->debug_taps = enable != 0;
  e->planned_n = 0;          // the plan (arena layout) changes
  return LUMI_OK;
}

int lumi_set_conv_impl(lumi_engine* e, int impl) {
  if (!e || (impl != 0 && impl != 1)) return LUMI_EINVAL;
  e->conv_impl = impl;
  e->planned_n = 0;          // the plan differs (stem staging buffers)
  return LUMI_OK;
}

int lumi_set_conv_streamk(lumi_engine* e, int mode) {
  if (!e || mode < 0 || mode > 2) return LUMI_EINVAL;
  e->conv_streamk = mode;
  return LUMI_OK;
}

int lumi_profile_enable(lumi_engine* e, int enable) {
  if (!e) return LUMI_EINVAL;
  e->profile = enable != 0;
  return LUMI_OK;
}

// Drains the recorded spans: "name:spans:total_ms:work;..." accumulated since the last read
// (work = algorithmic FLOPs for conv categories, algorithmic bytes for roi_pool, 0 otherwise).
const char* lumi_profile_read(lumi_engine* e) {
  if (!e) return "";
  try {
    cudaSetDevice(e->device);
    LUMI_CUDA_CHECK(cudaStreamSynchronize(e->stream));
    double ms[PC_COUNT] = {0}, work[PC_COUNT] = {0};
    int cnt[PC_COUNT] = {0};
    std::map<std::string, std::array<double, 3>> per_layer;     // label -> {spans, ms, work}
    std::vector<std::string> order;
    for (auto& sp : e->prof_spans) {
      float t = 0.f;
      if (cudaEventElapsedTime(&t, sp.a, sp.b) == cudaSuccess) {
        ms[sp.cat] += t; cnt[sp.cat]++; work[sp.cat] += sp.work;
        if (!sp.label.empty()) {
          auto it = per_layer.find(sp.label);
          if (it == per_layer.end()) { it = per_layer.emplace(sp.label, std::array<double, 3>{0, 0, 0}).first; order.push_back(sp.label); }
          it->second[0] += 1; it->second[1] += t; it->second[2] += sp.work;
        }
      }
      e->prof_pool.push_back(sp.a); e->prof_pool.push_back(sp.b);
    }
    e->prof_spans.clear();
    e->prof_layers_text.clear();
    for (const std::string& k : order) {
      const auto& v = per_layer[k];
      e->prof_layers_text += k + ":" + std::to_string((long)v[0]) + ":" + std::to_string(v[1]) + ":" + std::to_string(v[2]) + ";";
    }
    e->prof_text.clear();
    for (int c = 0; c < PC_COUNT; ++c)
      e->prof_text += std::string(PROF_NAMES[c]) + ":" + std::to_string(cnt[c]) + ":" + std::to_string(ms[c]) + ":" +
                      std::to_string(work[c]) + ";";
  } catch (const Error& err) { e->last_error = err.what(); return ""; }
  return e->prof_text.c_str();
}

// Per-conv-layer breakdown of the spans drained by the LAST lumi_profile_read: "layer:spans:total_ms:flops;..."
// in execution order.
const char* lumi_profile_read_layers(lumi_engine* e) { return e ? e->prof_layers_text.c_str() : ""; }

int lumi_get_tensor(lumi_engine* e, const char* name, float* out, int64_t capacity, int64_t* numel, int64_t* shape4) {
  if (!e) return LUMI_EINVAL;
  LUMI_API_BEGIN
  LUMI_REQUIRE(name, "lumi_get_tensor: null name");
  auto it = e->taps.find(name);
  if (it == e->taps.end()) throw Error(LUMI_EINVAL, "unknown tensor '" + std::string(name) + "'");
  const Tap& t = it->second;
  const int64_t count = t.shape[0] * t.shape[1] * t.shape[2] * t.shape[3];
  if (numel) *numel = count;
  if (shape4) for (int i = 0; i < 4; ++i) shape4[i] = t.shape[i];
  if (!out) return LUMI_OK;
  LUMI_REQUIRE(capacity >= count, "lumi_get_tensor: output buffer too small");
  LUMI_CUDA_CHECK(cudaSetDevice(e->device));
  LUMI_CUDA_CHECK(cudaStreamSynchronize(e->stream));
  if (t.kind == 0) {
    LUMI_CUDA_CHECK(cudaMemcpy(out, t.ptr, count * sizeof(float), cudaMemcpyDeviceToHost));
  } else if (t.kind == 2) {
    std::vector<int> tmp(count);
    LUMI_CUDA_CHECK(cudaMemcpy(tmp.data(), t.ptr, count * sizeof(int), cudaMemcpyDeviceToHost));
    for (int64_t i = 0; i < count; ++i) out[i] = (float)tmp[i];
  } else {
    float* d = nullptr;
    LUMI_CUDA_CHECK(cudaMalloc(&d, count * sizeof(float)));
    launch_act_to_f32(t.act, d, e->stream);
    LUMI_CUDA_CHECK(cudaStreamSynchronize(e->stream));
    cudaError_t ce = cudaMemcpy(out, d, count * sizeof(float), cudaMemcpyDeviceToHost);
    cudaFree(d);
    LUMI_CUDA_CHECK(ce);
  }
  return LUMI_OK;
  LUMI_API_END(e)
}

const char* lumi_last_error(lumi_engine* e) { return e ? e->last_error.c_str() : g_create_error.c_str(); }

void lumi_destroy(lumi_engine* e) {
  if (!e) return;
  cudaSetDevice(e->device);
  if (e->stream) cudaStreamSynchronize(e->stream);
  delete e;
}

}  // extern "C"
