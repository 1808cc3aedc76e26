// Stand-alone C-ABI operators (per-kernel parity tests and micro-benchmarks).
// Each wraps exactly the launcher the engine uses; temporaries are allocated per
// call and the stream is synchronised before they are released.
#include "../../include/luminoth_b200.h"
#include "conv.cuh"
#include "ops.cuh"

#include <cstdlib>
#include <memory>
#include <string>
#include <vector>

using namespace lumi;

namespace {
thread_local std::string g_op_error;

struct DevBuf {
  void* p = nullptr;
  explicit DevBuf(size_t bytes) { if (bytes) LUMI_CUDA_CHECK(cudaMalloc(&p, bytes)); }
  ~DevBuf() { cudaFree(p); }
  DevBuf(const DevBuf&) = delete;
  template <typename T> T* as() { return static_cast<T*>(p); }
};

struct ActBuf {
  DevBuf hi, lo;
  Act a;
  ActBuf(int n, int h, int w, int c) : hi((size_t)n * h * w * c * 2), lo((size_t)n * h * w * c * 2) {
    a.n = n; a.h = h; a.w = w; a.c = c; a.hi = hi.as<__half>(); a.lo = lo.as<__half>();
  }
};

int op_fail(const Error& e) { g_op_error = e.what(); return e.code; }

constexpr int CONV_OP_PIPE = 32;   // impl flag of lumi_op_conv2d*: the double-buffered mainloop

// The arguments of lumi_op_conv2d_io: those of lumi_op_conv2d, the residual's own resolution and sampling stride
// (res_h <= 0: the output's, stride 1) and the pre-activation output of lumi_op_conv2d_preact (pre_scale == nullptr:
// none; then y is required, else y == nullptr writes p only), and the schedule of lumi_op_conv2d_sched: the SM budget
// (0: the device's) and how many times the conv runs back to back on one stream-K workspace.
int op_conv2d(const float* x, int n, int h, int w, int cin, const float* wgt, int kh, int kw, int cout, int stride,
              int rate, int padding, const float* scale, const float* bias, const float* residual, int res_h,
              int res_w, int res_stride, int act, int impl, const float* pre_scale, const float* pre_bias, float* y,
              float* p, int* ho_out, int* wo_out, int sm_limit, int launches, cudaStream_t st) {
  LUMI_REQUIRE(sm_limit >= 0, "conv2d: sm_limit must be >= 0 (0: the device's SM count)");
  LUMI_REQUIRE(launches >= 1, "conv2d: launches must be >= 1");
  const bool preact = pre_scale != nullptr;
  const bool pipe = (impl & CONV_OP_PIPE) != 0;
  impl &= ~CONV_OP_PIPE;
  LUMI_REQUIRE(impl >= 0 && impl <= 19, "conv2d: impl must be one of 0-19");
  LUMI_REQUIRE(!pipe || (impl >= 1 && impl <= 12), "conv2d: impl | 32 (double-buffered mainloop) needs one of 1-12");
  ConvLayer L;
  L.kh = kh; L.kw = kw; L.cin = cin; L.cout = cout; L.stride = stride; L.rate = rate; L.act = act;
  const size_t nw = (size_t)kh * kw * cin * cout;
  std::vector<float> hw(nw), hs, hb;
  LUMI_CUDA_CHECK(cudaMemcpy(hw.data(), wgt, nw * sizeof(float), cudaMemcpyDeviceToHost));
  if (scale) { hs.resize(cout); LUMI_CUDA_CHECK(cudaMemcpy(hs.data(), scale, cout * sizeof(float), cudaMemcpyDeviceToHost)); }
  if (bias) { hb.resize(cout); LUMI_CUDA_CHECK(cudaMemcpy(hb.data(), bias, cout * sizeof(float), cudaMemcpyDeviceToHost)); }
  conv_layer_upload(L, hw.data(), scale ? hs.data() : nullptr, bias ? hb.data() : nullptr);
  struct Guard { ConvLayer& l; ~Guard() { conv_layer_free(l); } } guard{L};
  int ho, wo, pt = 0, pl = 0;
  if (padding == 1 || (padding == 2 && stride == 1)) {
    tf_same(h, kh, stride, rate, ho, pt); tf_same(w, kw, stride, rate, wo, pl);
  } else if (padding == 2) {
    const int keff = kh + (kh - 1) * (rate - 1);
    pt = pl = (keff - 1) / 2;
    ho = (h + (keff - 1) - keff) / stride + 1; wo = (w + (keff - 1) - keff) / stride + 1;
  } else {
    ho = tf_valid(h, kh, stride, rate); wo = tf_valid(w, kw, stride, rate);
  }
  LUMI_REQUIRE(ho > 0 && wo > 0, "conv2d: empty output");
  if (ho_out) *ho_out = ho;
  if (wo_out) *wo_out = wo;
  if (!y && !p) return LUMI_OK;           // shape query
  LUMI_REQUIRE(preact ? (p && pre_bias) : (y && !p), "conv2d: bad output arguments");
  // 0: SIMT, fp32 outputs; 1 whole tiles, 2 stream-K forced (fp32 outputs written by the epilogue);
  // 3 / 4 / 5: the engine's inter-layer form -- fp16x2 split planes -- with two consumer warpgroups (3), the
  // four-warpgroup short-K kernel allowed up to the engine's CONV_EPI16_DEFAULT K slices (4), and 4 + stream-K (5), all
  // through the shared-memory slot epilogue; 6 / 7: the 2-CTA cluster kernel wherever it applies (7: + stream-K); 8-11:
  // the halo-patch kernels (10, 11 on cluster pairs; 9, 11: + stream-K); 12: as 3 with the register epilogue; 13: SIMT
  // writing split planes (the engine's conv_impl = simt); 14 / 15: as 3 on 128 x 256 tiles whatever the K-slice and tile
  // counts (15: + stream-K), for layers with cout_pad % 256 == 0.  Codes 1-12 never take the 128 x 256 tile, and run the
  // engine's single-buffered mainloop; impl | 32 (CONV_OP_PIPE) on them runs the double-buffered one (LUMI_CONV_PIPE=1).
  // 16-19: as the engine launches the layer, every switch at run_conv's default (auto stream-K on a workspace, the
  // four-warpgroup bound, the 128 x 256 tile by its shape rule, slot epilogue, single-buffered, no 2-CTA or halo
  // kernels): 16 split outputs on all SMs, 17 split outputs leaving CONV_PIPELINE_SM_RESERVE SMs free (a pipelined
  // half-batch), 18 / 19 the same with fp32 outputs (the RPN and RCNN heads, the RCNN FC layers).  A pre-activation
  // output is written in split planes only: SIMT (0 or 13), 3-7, 12, 16 or 17.
  const bool simt = impl == 0 || impl == 13;
  const bool as_engine = impl >= 16;
  const bool split = preact || (impl >= 3 && impl <= 17);
  if (preact)
    LUMI_REQUIRE(simt || (impl >= 3 && impl <= 7) || impl == 12 || impl == 16 || impl == 17,
                 "conv2d_preact: impl must be 0 or 13 (SIMT) or one of the split-output codes 3-7, 12, 16, 17");
  if (split) LUMI_REQUIRE(cout % 32 == 0, "conv2d: split outputs need cout % 32 == 0");
  ActBuf in(n, h, w, cin);
  launch_f32_to_act(x, in.a, st);
  ConvIO io;
  io.in = in.a; io.pad_t = pt; io.pad_l = pl; io.ho = ho; io.wo = wo; io.out_f32 = y;
  io.sm_limit = sm_limit;
  std::unique_ptr<ActBuf> res;
  if (residual) {
    if (res_h <= 0) { res_h = ho; res_w = wo; res_stride = 1; }
    LUMI_REQUIRE((res_stride == 1 || res_stride == 2) && (ho - 1) * res_stride < res_h &&
                     (wo - 1) * res_stride < res_w,
                 "conv2d: the residual (sampling stride 1 or 2) must cover every output pixel");
    res.reset(new ActBuf(n, res_h, res_w, cout));
    launch_f32_to_act(residual, res->a, st);
    io.res = res->a; io.res_stride = res_stride;
  }
  // split planes: x (when y is given) and p, each read back as fp32; the pre-activation vectors padded like the layer's
  std::unique_ptr<ActBuf> xo, po;
  std::unique_ptr<DevBuf> ps, pb;
  DevBuf ovf(sizeof(int));
  LUMI_CUDA_CHECK(cudaMemset(ovf.p, 0, sizeof(int)));
  if (split) {
    io.out_f32 = nullptr;
    io.overflow_flag = ovf.as<int>();
    if (y) { xo.reset(new ActBuf(n, ho, wo, cout)); io.out = xo->a; }
  }
  if (preact) {
    const int cpad = cdiv(cout, 128) * 128;
    std::vector<float> hv(cpad, 0.f);
    ps.reset(new DevBuf(cpad * sizeof(float)));
    pb.reset(new DevBuf(cpad * sizeof(float)));
    LUMI_CUDA_CHECK(cudaMemcpy(hv.data(), pre_scale, cout * sizeof(float), cudaMemcpyDeviceToHost));
    LUMI_CUDA_CHECK(cudaMemcpy(ps->p, hv.data(), cpad * sizeof(float), cudaMemcpyHostToDevice));
    LUMI_CUDA_CHECK(cudaMemcpy(hv.data(), pre_bias, cout * sizeof(float), cudaMemcpyDeviceToHost));
    LUMI_CUDA_CHECK(cudaMemcpy(pb->p, hv.data(), cpad * sizeof(float), cudaMemcpyHostToDevice));
    po.reset(new ActBuf(n, ho, wo, cout));
    io.pre = po->a; io.pre_scale = ps->as<float>(); io.pre_bias = pb->as<float>();
  }
  ConvWorkspace sk;
  struct SkGuard { ConvWorkspace& w; ~SkGuard() { conv_workspace_free(w); } } skg{sk};
  if (simt) {
    for (int i = 0; i < launches; ++i) launch_conv_simt(L, io, st);
  } else if (as_engine) {
    io.epi16 = CONV_EPI16_DEFAULT;
    io.sm_reserve = (impl == 17 || impl == 19) ? CONV_PIPELINE_SM_RESERVE : 0;
    LUMI_REQUIRE(conv_tc_supported(L, io), "conv2d: this layer shape is not handled by the tensor-core kernel");
    conv_workspace_create(sk);
    io.sk = &sk;
    for (int i = 0; i < launches; ++i) launch_conv_tc(L, io, st);
  } else {
    io.pipe = pipe ? 1 : 0;
    io.epi_tma = impl == 12 ? 0 : 1;
    io.epi16 = (impl == 4 || impl == 5) ? CONV_EPI16_DEFAULT : 0;
    io.cta2 = (impl == 6 || impl == 7 || impl == 10 || impl == 11) ? 1 : 0;
    io.halo = (impl >= 8 && impl <= 11) ? 1 : 0;
    io.halo_tiles_pct = 1000000;                    // test hook: whenever the shape allows
    const bool wide = impl == 14 || impl == 15;
    io.wide = wide ? 1 : 0;
    io.wide_sm_pct = 0;
    LUMI_REQUIRE(conv_tc_supported(L, io), "conv2d: this layer shape is not handled by the tensor-core kernel");
    if (wide) LUMI_REQUIRE(L.cout_pad % 256 == 0, "conv2d: impl 14 / 15 need C_out padded to a multiple of 256");
    if (impl == 2 || impl == 5 || impl == 7 || impl == 9 || impl == 11 || impl == 15) {
      conv_workspace_create(sk);
      io.sk = &sk;
      io.streamk = 2;
    }
    for (int i = 0; i < launches; ++i) launch_conv_tc(L, io, st);
  }
  if (xo) launch_act_to_f32(xo->a, y, st);
  if (po) launch_act_to_f32(po->a, p, st);
  int flag = 0;
  LUMI_CUDA_CHECK(cudaMemcpyAsync(&flag, ovf.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  LUMI_CUDA_CHECK(cudaStreamSynchronize(st));
  if (flag) throw Error(LUMI_EOVERFLOW, "conv2d: an output exceeded the fp16x2 split range (|x| > 65504)");
  return LUMI_OK;
}
}  // namespace

#define OP_BEGIN try {
#define OP_END                                           \
  }                                                      \
  catch (const Error& err) { return op_fail(err); }      \
  catch (const std::exception& ex) { g_op_error = ex.what(); return LUMI_EINVAL; }

extern "C" {

const char* lumi_op_last_error(void) { return g_op_error.c_str(); }

int lumi_op_conv2d(const float* x, int n, int h, int w, int cin, const float* wgt, int kh, int kw, int cout, int stride,
                   int rate, int padding, const float* scale, const float* bias, const float* residual, int act,
                   int impl, float* y, int* ho_out, int* wo_out, void* stream) {
  OP_BEGIN
  return op_conv2d(x, n, h, w, cin, wgt, kh, kw, cout, stride, rate, padding, scale, bias, residual, 0, 0, 1, act, impl,
                   nullptr, nullptr, y, nullptr, ho_out, wo_out, 0, 1, static_cast<cudaStream_t>(stream));
  OP_END
}

int lumi_op_conv2d_preact(const float* x, int n, int h, int w, int cin, const float* wgt, int kh, int kw, int cout,
                          int stride, int rate, int padding, const float* scale, const float* bias,
                          const float* residual, int act, int impl, const float* pre_scale, const float* pre_bias,
                          float* y, float* p, int* ho_out, int* wo_out, void* stream) {
  OP_BEGIN
  LUMI_REQUIRE(pre_scale && pre_bias, "conv2d_preact: pre_scale and pre_bias are required");
  return op_conv2d(x, n, h, w, cin, wgt, kh, kw, cout, stride, rate, padding, scale, bias, residual, 0, 0, 1, act, impl,
                   pre_scale, pre_bias, y, p, ho_out, wo_out, 0, 1, static_cast<cudaStream_t>(stream));
  OP_END
}

int lumi_op_conv2d_io(const float* x, int n, int h, int w, int cin, const float* wgt, int kh, int kw, int cout,
                      int stride, int rate, int padding, const float* scale, const float* bias, const float* residual,
                      int res_h, int res_w, int res_stride, int act, int impl, const float* pre_scale,
                      const float* pre_bias, float* y, float* p, int* ho_out, int* wo_out, void* stream) {
  OP_BEGIN
  LUMI_REQUIRE(!residual || res_h > 0, "conv2d_io: res_h and res_w are required with a residual");
  LUMI_REQUIRE(!pre_scale == !pre_bias, "conv2d_io: pre_scale and pre_bias go together");
  return op_conv2d(x, n, h, w, cin, wgt, kh, kw, cout, stride, rate, padding, scale, bias, residual, res_h, res_w,
                   res_stride, act, impl, pre_scale, pre_bias, y, p, ho_out, wo_out, 0, 1,
                   static_cast<cudaStream_t>(stream));
  OP_END
}

int lumi_op_conv2d_sched(const float* x, int n, int h, int w, int cin, const float* wgt, int kh, int kw, int cout,
                         int stride, int rate, int padding, const float* scale, const float* bias, const float* residual,
                         int res_h, int res_w, int res_stride, int act, int impl, const float* pre_scale,
                         const float* pre_bias, int sm_limit, int launches, float* y, float* p, int* ho_out, int* wo_out,
                         void* stream) {
  OP_BEGIN
  LUMI_REQUIRE(!residual || res_h > 0, "conv2d_sched: res_h and res_w are required with a residual");
  LUMI_REQUIRE(!pre_scale == !pre_bias, "conv2d_sched: pre_scale and pre_bias go together");
  return op_conv2d(x, n, h, w, cin, wgt, kh, kw, cout, stride, rate, padding, scale, bias, residual, res_h, res_w,
                   res_stride, act, impl, pre_scale, pre_bias, y, p, ho_out, wo_out, sm_limit, launches,
                   static_cast<cudaStream_t>(stream));
  OP_END
}

int lumi_pack_conv_weights(const float* w, int kdim, int cout, const float* scale, uint16_t* hi, uint16_t* lo,
                           float* scale_tc) {
  OP_BEGIN
  LUMI_REQUIRE(w && hi && lo && scale_tc && kdim > 0 && cout > 0, "pack_conv_weights: bad arguments");
  static_assert(sizeof(__half) == sizeof(uint16_t), "fp16 bits");
  pack_conv_weights(w, (size_t)kdim, cout, scale, reinterpret_cast<__half*>(hi), reinterpret_cast<__half*>(lo),
                    scale_tc);
  return LUMI_OK;
  OP_END
}

int lumi_op_resize_bilinear(const void* src, int src_is_f32, int h0, int w0, float* dst, int h, int w, void* stream) {
  OP_BEGIN
  LUMI_REQUIRE(src && dst && h0 > 0 && w0 > 0 && h > 0 && w > 0, "resize_bilinear: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  launch_resize_bilinear(src, src_is_f32 != 0, h0, w0, dst, h, w, st);
  LUMI_CUDA_CHECK(cudaStreamSynchronize(st));
  return LUMI_OK;
  OP_END
}

int lumi_op_pixels_to_rgb(const void* src, int format, int is_f32, int h, int w, void* dst, void* stream) {
  OP_BEGIN
  LUMI_REQUIRE(src && dst && h > 0 && w > 0, "pixels_to_rgb: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  launch_pixels_to_rgb(src, format, is_f32 != 0, h, w, dst, st);
  LUMI_CUDA_CHECK(cudaStreamSynchronize(st));
  return LUMI_OK;
  OP_END
}

int lumi_op_max_pool(const float* x, int n, int h, int w, int c, int k, int stride, int padding, float* y, void* stream) {
  OP_BEGIN
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int ho, wo, pt = 0, pl = 0;
  if (padding == 1) { tf_same(h, k, stride, 1, ho, pt); tf_same(w, k, stride, 1, wo, pl); }
  else { ho = tf_valid(h, k, stride, 1); wo = tf_valid(w, k, stride, 1); }
  ActBuf in(n, h, w, c), out(n, ho, wo, c);
  launch_f32_to_act(x, in.a, st);
  launch_max_pool(in.a, out.a, k, stride, pt, pl, st);
  launch_act_to_f32(out.a, y, st);
  LUMI_CUDA_CHECK(cudaStreamSynchronize(st));
  return LUMI_OK;
  OP_END
}

int lumi_op_max_pool_preact(const float* x, int n, int h, int w, int c, int k, int stride, int padding,
                            const float* pre_scale, const float* pre_bias, float* y, void* stream) {
  OP_BEGIN
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  LUMI_REQUIRE(pre_scale && pre_bias, "max_pool_preact: pre_scale and pre_bias are required");
  int ho, wo, pt = 0, pl = 0;
  if (padding == 1) { tf_same(h, k, stride, 1, ho, pt); tf_same(w, k, stride, 1, wo, pl); }
  else { ho = tf_valid(h, k, stride, 1); wo = tf_valid(w, k, stride, 1); }
  ActBuf in(n, h, w, c), out(n, ho, wo, c);
  launch_f32_to_act(x, in.a, st);
  launch_max_pool(in.a, out.a, k, stride, pt, pl, st, pre_scale, pre_bias);
  launch_act_to_f32(out.a, y, st);
  LUMI_CUDA_CHECK(cudaStreamSynchronize(st));
  return LUMI_OK;
  OP_END
}

int lumi_op_roi_pool(const float* fmap, int n, int fh, int fw, int c, const float* rois, const int32_t* roi_batch, int r,
                     float im_h, float im_w, int ph, int pw, float* y, void* stream) {
  OP_BEGIN
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  LUMI_REQUIRE(n == 1 || roi_batch == nullptr, "roi_pool op: single image (roi_batch must be NULL or n == 1)");
  (void)roi_batch;
  ActBuf out(r, pw, ph, c);
  // every roi is pooled from image 0 (the launcher reads n * r rows: n images of r rois each)
  launch_roi_pool(fmap, 1, fh, fw, c, rois, nullptr, r, im_h, im_w, ph, pw, out.a, Act(), st);
  launch_act_to_f32(out.a, y, st);
  LUMI_CUDA_CHECK(cudaStreamSynchronize(st));
  return LUMI_OK;
  OP_END
}

int lumi_roi_kernel(int c, int ph, int pw) { return roi_kernel(c, ph, pw); }

int lumi_op_roi_pool_batched(const float* fmap, int n, int fh, int fw, int c, const float* rois, const int32_t* counts,
                             int rmax, float im_h, float im_w, int ph, int pw, int kernel, float* pooled, float* mean,
                             void* stream) {
  OP_BEGIN
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  LUMI_REQUIRE(n > 0 && fh > 0 && fw > 0 && c > 0 && rmax > 0, "roi_pool_batched: sizes must be positive");
  LUMI_REQUIRE(pooled || mean, "roi_pool_batched: pooled or mean is required");
  LUMI_REQUIRE(ph >= 1 && pw >= 1, "roi_pool_batched: pooled size must be >= 1");
  const int rows = n * rmax;
  // both split planes start as 0xFFFF (an fp16 NaN): a cell or row the kernel skips reads back as NaN
  std::unique_ptr<ActBuf> out, m;
  if (pooled) {
    out.reset(new ActBuf(rows, pw, ph, c));
    LUMI_CUDA_CHECK(cudaMemsetAsync(out->a.hi, 0xFF, out->a.numel() * sizeof(__half), st));
    LUMI_CUDA_CHECK(cudaMemsetAsync(out->a.lo, 0xFF, out->a.numel() * sizeof(__half), st));
  }
  if (mean) {
    m.reset(new ActBuf(rows, 1, 1, c));
    LUMI_CUDA_CHECK(cudaMemsetAsync(m->a.hi, 0xFF, m->a.numel() * sizeof(__half), st));
    LUMI_CUDA_CHECK(cudaMemsetAsync(m->a.lo, 0xFF, m->a.numel() * sizeof(__half), st));
  }
  launch_roi_pool(fmap, n, fh, fw, c, rois, counts, rmax, im_h, im_w, ph, pw, out ? out->a : Act(), m ? m->a : Act(),
                  st, kernel);
  if (out) launch_act_to_f32(out->a, pooled, st);
  if (m) launch_act_to_f32(m->a, mean, st);
  LUMI_CUDA_CHECK(cudaStreamSynchronize(st));
  return LUMI_OK;
  OP_END
}

int lumi_op_spatial_mean(const float* x, int r, int h, int w, int c, float* y, void* stream) {
  OP_BEGIN
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  LUMI_REQUIRE(r > 0 && h > 0 && w > 0 && c > 0, "spatial_mean: sizes must be positive");
  ActBuf in(r, h, w, c), out(r, 1, 1, c);
  launch_f32_to_act(x, in.a, st);
  LUMI_CUDA_CHECK(cudaMemsetAsync(out.a.hi, 0xFF, out.a.numel() * sizeof(__half), st));
  LUMI_CUDA_CHECK(cudaMemsetAsync(out.a.lo, 0xFF, out.a.numel() * sizeof(__half), st));
  launch_spatial_mean(in.a, out.a, st);
  launch_act_to_f32(out.a, y, st);
  LUMI_CUDA_CHECK(cudaStreamSynchronize(st));
  return LUMI_OK;
  OP_END
}

int lumi_op_l2norm_scale(const float* x, int n, int h, int w, int c, const float* gamma, float eps, float* y,
                         void* stream) {
  OP_BEGIN
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  LUMI_REQUIRE(n > 0 && h > 0 && w > 0 && c > 0, "l2norm_scale: sizes must be positive");
  LUMI_REQUIRE(gamma, "l2norm_scale: gamma is required");
  ActBuf in(n, h, w, c), out(n, h, w, c);
  launch_f32_to_act(x, in.a, st);
  LUMI_CUDA_CHECK(cudaMemsetAsync(out.a.hi, 0xFF, out.a.numel() * sizeof(__half), st));
  LUMI_CUDA_CHECK(cudaMemsetAsync(out.a.lo, 0xFF, out.a.numel() * sizeof(__half), st));
  launch_l2norm_scale(in.a, out.a, gamma, eps, st);
  launch_act_to_f32(out.a, y, st);
  LUMI_CUDA_CHECK(cudaStreamSynchronize(st));
  return LUMI_OK;
  OP_END
}

int lumi_op_softmax_rows(const float* x, int rows, int cols, int in_stride, float* y, void* stream) {
  OP_BEGIN
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  LUMI_REQUIRE(rows > 0 && cols > 0 && in_stride >= cols, "softmax_rows: need rows, cols > 0 and in_stride >= cols");
  launch_softmax_rows(x, y, rows, cols, in_stride, st);
  LUMI_CUDA_CHECK(cudaStreamSynchronize(st));
  return LUMI_OK;
  OP_END
}

int lumi_op_sort_desc(const float* scores, int n, int32_t* idx_out, void* stream) {
  OP_BEGIN
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (n <= 0) return LUMI_OK;
  NmsWorkspace ws;
  struct G { NmsWorkspace& w; ~G() { nms_workspace_free(w); } } g{ws};
  nms_workspace_alloc(ws, 1, n, 1);
  launch_sort_desc(scores, n, idx_out, ws, st);
  LUMI_CUDA_CHECK(cudaStreamSynchronize(st));
  return LUMI_OK;
  OP_END
}

int lumi_op_nms_sorted(const float* boxes_sorted, int n, float iou_threshold, int max_out, int32_t* keep,
                       int32_t* num_keep, void* stream) {
  OP_BEGIN
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  LUMI_REQUIRE(n > 0 && max_out > 0, "nms_sorted: n and max_out must be positive");
  NmsWorkspace ws;
  struct G { NmsWorkspace& w; ~G() { nms_workspace_free(w); } } g{ws};
  nms_workspace_alloc(ws, 1, n, max_out);
  launch_nms_sorted(boxes_sorted, n, iou_threshold, max_out, ws, keep, num_keep, st);
  LUMI_CUDA_CHECK(cudaStreamSynchronize(st));
  return LUMI_OK;
  OP_END
}

int lumi_nms_path(int problems, int ncap, float iou_threshold) { return nms_path(problems, ncap, iou_threshold); }

int lumi_op_nms_batched(const float* boxes_sorted, const int32_t* nvalid, int problems, int cap, float iou_threshold,
                        int max_out, int32_t* keep, int32_t* num_keep, void* stream) {
  OP_BEGIN
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  LUMI_REQUIRE(problems > 0 && cap > 0 && max_out > 0, "nms_batched: problems, cap and max_out must be positive");
  std::vector<int> hn(problems);
  LUMI_CUDA_CHECK(cudaMemcpy(hn.data(), nvalid, problems * sizeof(int), cudaMemcpyDeviceToHost));
  for (int v : hn) LUMI_REQUIRE(v >= 0 && v <= cap, "nms_batched: nvalid must lie in [0, cap]");
  NmsWorkspace ws;
  struct G { NmsWorkspace& w; ~G() { nms_workspace_free(w); } } g{ws};
  nms_workspace_alloc(ws, problems, cap, max_out);
  launch_nms_batched(boxes_sorted, nvalid, problems, iou_threshold, max_out, ws, keep, num_keep, st);
  LUMI_CUDA_CHECK(cudaStreamSynchronize(st));
  return LUMI_OK;
  OP_END
}

int lumi_op_window_merge(const float* wboxes, const float* wscores, const int32_t* wlabels, const int32_t* wcounts,
                         int nwin, int kmax, const int32_t* win_src, const float* wmap, int nsrc, int nc, int class_max,
                         int total_max, float iou_threshold, int sm_limit, float* boxes, float* scores,
                         int32_t* labels, int32_t* counts, int64_t* merge_stats, void* stream) {
  OP_BEGIN
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  LUMI_REQUIRE(wboxes && wscores && wlabels && wcounts && win_src && wmap && boxes && scores && labels && counts,
               "window_merge: null buffer");
  LUMI_REQUIRE(nwin >= 1 && kmax >= 1 && sm_limit >= 0, "window_merge: need nwin, kmax >= 1 and sm_limit >= 0");
  DevBuf map((size_t)nwin * sizeof(float4));
  LUMI_CUDA_CHECK(cudaMemcpyAsync(map.p, wmap, (size_t)nwin * sizeof(float4), cudaMemcpyHostToDevice, st));
  std::unique_ptr<DevBuf> scratch;
  int64_t stats[4];
  run_window_merge(wboxes, wscores, wlabels, wcounts, win_src, map.as<float4>(), nwin, kmax, nsrc, nc, class_max,
                   total_max, iou_threshold, sm_limit,
                   [&scratch](size_t bytes) { scratch.reset(new DevBuf(bytes)); return scratch->as<uint8_t>(); },
                   boxes, scores, labels, counts, stats, st);
  LUMI_CUDA_CHECK(cudaStreamSynchronize(st));
  if (merge_stats) for (int i = 0; i < 4; ++i) merge_stats[i] = stats[i];
  return LUMI_OK;
  OP_END
}

int lumi_op_rpn_proposals_batched(const float* cls, const float* box, int64_t img_stride_cls, int64_t img_stride_box,
                                  int A, const float* anchors, int nimg, int na, int cap, float im_h, float im_w,
                                  int pre_nms_top_n, int post_nms_top_n, float nms_threshold, float min_prob,
                                  int filter_outside, int clip_after_nms, int apply_nms, int logits, int cls_stride,
                                  int cls_off, int box_stride, int box_off, float* proposals, float* scores,
                                  int32_t* counts, void* stream) {
  OP_BEGIN
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  LUMI_REQUIRE(nimg > 0 && A > 0 && na > 0 && na % A == 0 && cap >= na && pre_nms_top_n > 0 && post_nms_top_n > 0,
               "rpn_proposals_batched: need positive sizes, na a multiple of A and cap >= na");
  NmsWorkspace ws;
  struct G { NmsWorkspace& w; ~G() { nms_workspace_free(w); } } g{ws};
  nms_workspace_alloc(ws, nimg, cap, post_nms_top_n, std::min(cap, pre_nms_top_n));   // as the engine sizes ws_rpn
  RpnParams p{};
  p.na = na; p.im_h = im_h; p.im_w = im_w; p.pre_nms_top_n = pre_nms_top_n; p.post_nms_top_n = post_nms_top_n;
  p.nms_threshold = nms_threshold; p.min_prob = min_prob; p.filter_outside = filter_outside;
  p.clip_after_nms = clip_after_nms; p.apply_nms = apply_nms; p.logits = logits;
  p.cls_stride = cls_stride; p.cls_off = cls_off; p.box_stride = box_stride; p.box_off = box_off;
  launch_rpn_proposals(cls, box, (long)img_stride_cls, (long)img_stride_box, A, anchors, nimg, p, ws, proposals, scores,
                       counts, st);
  LUMI_CUDA_CHECK(cudaStreamSynchronize(st));
  return LUMI_OK;
  OP_END
}

int lumi_op_class_detections_batched(const float* boxes_in, int64_t boxes_img_stride, const int32_t* row_counts,
                                     const float* deltas, const float* cls_prob, int nimg, int r, int nc, float im_h,
                                     float im_w, float var0, float var1, float min_prob, float nms_threshold,
                                     int class_max, int total_max, int shared_deltas, int prob_stride,
                                     int delta_stride, float* objects, int32_t* labels, float* probs, int32_t* count,
                                     float* records, void* stream) {
  OP_BEGIN
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  LUMI_REQUIRE(nimg > 0 && r > 0 && nc > 0 && class_max > 0 && total_max > 0 && boxes_img_stride >= 0 &&
                   prob_stride >= nc + 1 && delta_stride >= (shared_deltas ? 4 : 4 * nc),
               "class_detections_batched: bad sizes or strides");
  NmsWorkspace ws;
  struct G { NmsWorkspace& w; ~G() { nms_workspace_free(w); } } g{ws};
  nms_workspace_alloc(ws, nimg * nc, r, class_max);
  DevBuf fk(det_final_scratch_bytes(nimg, nc, class_max));
  DetParams p{};
  p.r = r; p.nc = nc; p.im_h = im_h; p.im_w = im_w; p.var0 = var0; p.var1 = var1; p.min_prob = min_prob;
  p.nms_threshold = nms_threshold; p.class_max = class_max; p.total_max = total_max;
  p.shared_deltas = shared_deltas ? 1 : 0; p.prob_stride = prob_stride; p.delta_stride = delta_stride;
  launch_class_detections(boxes_in, (long)boxes_img_stride, row_counts, deltas, cls_prob, nimg, p, ws, fk.as<float>(),
                          objects, labels, probs, count, st, records);
  LUMI_CUDA_CHECK(cudaStreamSynchronize(st));
  return LUMI_OK;
  OP_END
}

int lumi_op_rpn_proposals(const float* cls_prob, const float* bbox_pred, const float* anchors, int na, float im_h,
                          float im_w, int pre_nms_top_n, int post_nms_top_n, float nms_threshold, float min_prob,
                          int filter_outside, int clip_after_nms, float* proposals, float* scores, int32_t* count,
                          void* stream) {
  OP_BEGIN
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  LUMI_REQUIRE(na > 0 && pre_nms_top_n > 0 && post_nms_top_n > 0, "rpn_proposals: sizes must be positive");
  NmsWorkspace ws;
  struct G { NmsWorkspace& w; ~G() { nms_workspace_free(w); } } g{ws};
  nms_workspace_alloc(ws, 1, na, post_nms_top_n, pre_nms_top_n < na ? pre_nms_top_n : na);
  RpnParams p{};
  p.na = na; p.im_h = im_h; p.im_w = im_w; p.pre_nms_top_n = pre_nms_top_n; p.post_nms_top_n = post_nms_top_n;
  p.nms_threshold = nms_threshold; p.min_prob = min_prob; p.filter_outside = filter_outside;
  p.clip_after_nms = clip_after_nms; p.apply_nms = 1; p.logits = 0;
  p.cls_stride = 2; p.cls_off = 0; p.box_stride = 4; p.box_off = 0;
  launch_rpn_proposals(cls_prob, bbox_pred, 0, 0, 1, anchors, 1, p, ws, proposals, scores, count, st);
  LUMI_CUDA_CHECK(cudaStreamSynchronize(st));
  return LUMI_OK;
  OP_END
}

int lumi_op_class_detections(const float* boxes_in, const float* deltas, const float* cls_prob, int r, int nc, float im_h,
                             float im_w, float var0, float var1, float min_prob, float nms_threshold, int class_max,
                             int total_max, int ssd_order, float* objects, int32_t* labels, float* probs, int32_t* count,
                             void* stream) {
  OP_BEGIN
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  LUMI_REQUIRE(r > 0 && nc > 0 && class_max > 0 && total_max > 0, "class_detections: sizes must be positive");
  NmsWorkspace ws;
  struct G { NmsWorkspace& w; ~G() { nms_workspace_free(w); } } g{ws};
  nms_workspace_alloc(ws, nc, r, class_max);
  DevBuf fk(det_final_scratch_bytes(1, nc, class_max));
  DetParams p{};
  p.r = r; p.nc = nc; p.im_h = im_h; p.im_w = im_w; p.var0 = var0; p.var1 = var1; p.min_prob = min_prob;
  p.nms_threshold = nms_threshold; p.class_max = class_max; p.total_max = total_max;
  p.shared_deltas = ssd_order ? 1 : 0;
  p.prob_stride = nc + 1; p.delta_stride = ssd_order ? 4 : 4 * nc;
  launch_class_detections(boxes_in, (long)r * 4, nullptr, deltas, cls_prob, 1, p, ws, fk.as<float>(), objects, labels,
                          probs, count, st);
  LUMI_CUDA_CHECK(cudaStreamSynchronize(st));
  return LUMI_OK;
  OP_END
}

}  // extern "C"
