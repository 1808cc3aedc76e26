// Convolution layer descriptors shared by the engine and the stand-alone op.
#pragma once
#include "common.cuh"
#include <vector>

namespace lumi {

// One conv layer, device-resident, both weight forms.
struct ConvLayer {
  int kh = 1, kw = 1, cin = 0, cout = 0;
  int stride = 1, rate = 1;
  int act = ACT_NONE;
  // SIMT form: TF layout [kh*kw*cin][cout] fp32, epilogue v = acc*scale + bias
  float* w_f32 = nullptr;
  float* scale = nullptr;   // [cout]  (BN gamma*rsqrt(var+eps), or 1)
  float* bias = nullptr;    // [cout]  (BN beta - mean*scale, or conv bias)
  // tensor-core form: [cout_pad][kh*kw*cin] fp16 hi/lo planes of w * 2^e[c]; scale_tc = scale * 2^-e[c]
  __half* w_hi = nullptr;
  __half* w_lo = nullptr;
  float* scale_tc = nullptr;
  int cout_pad = 0;
  bool tc_ready = false;
};

// Scratch of the stream-K schedule (see conv.cu): one partial-accumulator slot + flag per persistent CTA.
// One workspace per stream: launches that share it must be stream-ordered.
struct ConvWorkspace {
  float* partials = nullptr;
  int* flags = nullptr;
  unsigned epoch = 0;
  int ctas = 0;
};
void conv_workspace_create(ConvWorkspace& w);
void conv_workspace_free(ConvWorkspace& w);
// Per-device facts (SM count, opt-in dynamic shared memory of a kernel) are cached per CUDA device, never per
// process: two engines on two devices, or on two threads, share no mutable launch state.
int device_sm_count();            // SMs of the CURRENT device
constexpr int LUMI_MAX_DEVICES = 64;

struct ConvIO {
  Act in;
  Act out;                  // split-plane output (used when out_f32 == nullptr)
  float* out_f32 = nullptr; // optional fp32 NHWC output [n,ho,wo,cout]
  // optional pre-activation output (pre.hi == nullptr -> none), split planes like `out`:
  //   p = relu(fmaf(x^, pre_scale[c], pre_bias[c])),  x^ = float(hi) + float(lo) of the layer's output x as split,
  // i.e. exactly what a separate "read x, batch norm, relu" pass over the stored x gives.  out.hi == nullptr with
  // pre.hi set writes p only.  pre_scale / pre_bias are padded to a multiple of 128 channels.
  Act pre;
  const float* pre_scale = nullptr;
  const float* pre_bias = nullptr;
  Act res;                  // optional residual (res.hi == nullptr -> none)
  int res_stride = 1;       // residual sampled at (oy*res_stride, ox*res_stride)  (slim `subsample`)
  int pad_t = 0, pad_l = 0;
  int ho = 0, wo = 0;
  int* overflow_flag = nullptr;
  ConvWorkspace* sk = nullptr;  // enables stream-K scheduling on the tensor-core path (nullptr: whole tiles only)
  int streamk = 1;              // stream-K policy of THIS launch: 0 off, 1 auto (wave-quantisation heuristic), 2 whenever possible
  int cta2 = 0;                 // 2-CTA cluster kernel (weight tile multicast) on layers with at least this many K slices per tile (0 = never)
  int halo = 0;                 // halo-patch kernels on 3x3 stride-1 SAME layers without residual or fp32 output (0 never; on CTA pairs with cta2)
  int halo_tiles_pct = 150;     // ... while their M-tile count stays within this percentage of the generic kernel's
  int pipe = 1;                 // 1: double-buffered slice accumulators (slice k + 1's MMAs overlap slice k's fold); 0: single (the engine's default, LUMI_CONV_PIPE)
  int epi16 = 0;                // four-consumer-warpgroup (16 epilogue warps) kernel on layers with at most this many K slices per tile (0 = never)
  int wide = 16;                // 128 x 256 tiles on split-output layers with cout_pad % 256 == 0 and at least this many K slices per tile (0 = never)
  int wide_sm_pct = 50;         // ... while those tiles number at least this percentage of the SMs the launch may use
  int epi_tma = 1;              // 1: split outputs of the generic kernel leave through the shared-memory slot epilogue (TMA); 0: register epilogue
  int sm_reserve = 0;           // SMs a persistent launch leaves free (the engine's two-stream pipeline sets 8)
  // Optional strided ("Toeplitz") view of the input for the tensor-core path: element pitches between
  // consecutive pixels / rows / images (0 = dense NHWC).  Used by the space-to-depth stem, where each
  // A row is the 64 contiguous fp16 of four horizontally adjacent 16-channel pixels.
  long in_pix_pitch = 0, in_row_pitch = 0, in_img_pitch = 0;
};

// Tensor-core weight packing, host only (no CUDA calls).  w: TF layout [kdim][cout] on host.  For every output channel
// c < cout: rows c of hi / lo ([cout][kdim] fp16) hold the split of w[:, c] * 2^e[c], and scale_tc[c] = scale[c] * 2^-e[c]
// (scale == nullptr: 1), computed in double and rounded once.  e[c] puts max|w[:, c]| in [2^13, 2^14) so the lo plane
// stays in fp16's normal range; it is clamped to [-126, 126] so 2^e and 2^-e are normal fp32.  A clamped column
// (0 < max|w[:, c]| < 2^-112) packs to small or subnormal fp16; its whole contribution is below 2^-112 * |s| * sum|x|.
// An all-zero (or non-finite) column gets e = 0.
constexpr int CONV_PACK_EXP_MAX = 126;
void pack_conv_weights(const float* w, size_t kdim, int cout, const float* scale, __half* hi, __half* lo,
                       float* scale_tc);

// host-side packing (w: TF layout on host)
void conv_layer_upload(ConvLayer& L, const float* w_host, const float* scale_host, const float* bias_host);
void conv_layer_free(ConvLayer& L);

bool conv_tc_supported(const ConvLayer& L, const ConvIO& io);
void launch_conv_simt(const ConvLayer& L, const ConvIO& io, cudaStream_t st);
void launch_conv_tc(const ConvLayer& L, const ConvIO& io, cudaStream_t st);

// TF padding arithmetic (SURVEY Appendix A)
inline void tf_same(int in, int k, int stride, int rate, int& out, int& pad_before) {
  int keff = k + (k - 1) * (rate - 1);
  out = (in + stride - 1) / stride;
  int total = (out - 1) * stride + keff - in;
  if (total < 0) total = 0;
  pad_before = total / 2;
}
inline int tf_valid(int in, int k, int stride, int rate) {
  int keff = k + (k - 1) * (rate - 1);
  return (in - keff) / stride + 1;
}

}  // namespace lumi
