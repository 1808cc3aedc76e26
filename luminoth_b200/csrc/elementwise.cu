// HBM-bound elementwise / pooling / normalisation kernels (vectorised NHWC).
#include "ops.cuh"
#include <cstdint>

namespace lumi {

// uint8 RGB image -> (optionally mean-subtracted) fp16x2 planes.
// base_network.py:153-177 (`inputs - [means]`, only for resnet*/vgg* architectures).
template <typename PIX>
__global__ void u8_to_act_kernel(const PIX* __restrict__ img, __half* __restrict__ hi, __half* __restrict__ lo,
                                 size_t numel, int c, float m0, float m1, float m2) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= numel) return;
  int ch = (int)(i % c);
  float mean = ch == 0 ? m0 : (ch == 1 ? m1 : m2);
  float v = __fsub_rn((float)img[i], mean);
  __half h, l;
  split_f32(v, h, l);
  hi[i] = h; lo[i] = l;
}
void launch_u8_to_act(const void* img, bool img_f32, Act out, const float* means, cudaStream_t st) {
  size_t n = out.numel();
  if (!n) return;
  float m0 = means ? means[0] : 0.f, m1 = means ? means[1] : 0.f, m2 = means ? means[2] : 0.f;
  if (img_f32)
    u8_to_act_kernel<float><<<(unsigned)cdiv64(n, 256), 256, 0, st>>>(static_cast<const float*>(img), out.hi, out.lo, n,
                                                                      out.c, m0, m1, m2);
  else
    u8_to_act_kernel<uint8_t><<<(unsigned)cdiv64(n, 256), 256, 0, st>>>(static_cast<const uint8_t*>(img), out.hi,
                                                                        out.lo, n, out.c, m0, m1, m2);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
}

// tf.image.resize_images(BILINEAR) of TF 1.x (legacy kernel: align_corners=False, src = dst * (in / out), no
// half-pixel offset) -- luminoth/utils/image.py:94-97,139-142.  Same float32 operation order as the oracle
// (tf_ops.resize_bilinear), no FMA contraction, so the result is bit-identical to it.
template <typename PIX>
__global__ void resize_bilinear_kernel(const PIX* __restrict__ src, int h0, int w0, float* __restrict__ dst, int h, int w,
                                       float hs, float ws) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)h * w) return;
  const int x = (int)(i % w), y = (int)(i / w);
  const float fy = __fmul_rn((float)y, hs), fx = __fmul_rn((float)x, ws);
  const int y0 = (int)floorf(fy), x0 = (int)floorf(fx);
  const int y1 = min(y0 + 1, h0 - 1), x1 = min(x0 + 1, w0 - 1);
  const float yl = __fsub_rn(fy, (float)y0), xl = __fsub_rn(fx, (float)x0);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float tl = (float)src[((size_t)y0 * w0 + x0) * 3 + c], tr = (float)src[((size_t)y0 * w0 + x1) * 3 + c];
    const float bl = (float)src[((size_t)y1 * w0 + x0) * 3 + c], br = (float)src[((size_t)y1 * w0 + x1) * 3 + c];
    const float top = __fadd_rn(tl, __fmul_rn(__fsub_rn(tr, tl), xl));
    const float bot = __fadd_rn(bl, __fmul_rn(__fsub_rn(br, bl), xl));
    dst[i * 3 + c] = __fadd_rn(top, __fmul_rn(__fsub_rn(bot, top), yl));
  }
}
void launch_resize_bilinear(const void* src, bool src_f32, int h0, int w0, float* dst, int h, int w, cudaStream_t st) {
  if (!h || !w) return;
  const float hs = (float)h0 / (float)h, ws = (float)w0 / (float)w;      // float32 division, like the oracle
  const size_t total = (size_t)h * w;
  if (src_f32)
    resize_bilinear_kernel<float><<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(static_cast<const float*>(src), h0, w0,
                                                                                dst, h, w, hs, ws);
  else
    resize_bilinear_kernel<uint8_t><<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(static_cast<const uint8_t*>(src), h0,
                                                                                  w0, dst, h, w, hs, ws);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
}

// Space-to-depth staging of the 7x7/2 stem (slim conv2d_same: zero pad 3/3 AFTER mean subtraction):
// X2[n][Y][X][dy*6 + dx*3 + c] = xp[2Y+dy][2X+dx][c], xp = padded (image - mean); channels 12..15 = 0.
// The stem then is a 4x4/1 VALID conv over X2 that the tensor-core kernel runs as 4 taps of K = 64.
template <typename PIX>
__global__ void stem_s2d_kernel(const PIX* __restrict__ img, __half* __restrict__ hi, __half* __restrict__ lo, int n,
                                int h, int w, int h2, int w2, float m0, float m1, float m2) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t total = (size_t)n * h2 * w2;
  if (i >= total) return;
  const int X = (int)(i % w2), Y = (int)((i / w2) % h2), ni = (int)(i / ((size_t)w2 * h2));
  uint4 vh[2], vl[2];
  __half* ph = reinterpret_cast<__half*>(vh);
  __half* pl = reinterpret_cast<__half*>(vl);
#pragma unroll
  for (int j = 0; j < 16; ++j) { ph[j] = __float2half_rn(0.f); pl[j] = __float2half_rn(0.f); }
#pragma unroll
  for (int dy = 0; dy < 2; ++dy)
#pragma unroll
    for (int dx = 0; dx < 2; ++dx) {
      const int py = 2 * Y + dy - 3, px = 2 * X + dx - 3;
      if (py >= 0 && py < h && px >= 0 && px < w) {
        const PIX* p = img + (((size_t)ni * h + py) * w + px) * 3;
        const float v0 = __fsub_rn((float)p[0], m0), v1 = __fsub_rn((float)p[1], m1), v2 = __fsub_rn((float)p[2], m2);
        const int o = dy * 6 + dx * 3;
        split_f32(v0, ph[o], pl[o]); split_f32(v1, ph[o + 1], pl[o + 1]); split_f32(v2, ph[o + 2], pl[o + 2]);
      }
    }
  uint4* oh = reinterpret_cast<uint4*>(hi + i * 16);
  uint4* ol = reinterpret_cast<uint4*>(lo + i * 16);
  oh[0] = vh[0]; oh[1] = vh[1]; ol[0] = vl[0]; ol[1] = vl[1];
}
void launch_stem_s2d(const void* img, bool img_f32, int n, int h, int w, Act x2, const float* means, cudaStream_t st) {
  size_t total = (size_t)n * x2.h * x2.w;
  if (!total) return;
  if (img_f32)
    stem_s2d_kernel<float><<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(static_cast<const float*>(img), x2.hi, x2.lo, n,
                                                                         h, w, x2.h, x2.w, means[0], means[1], means[2]);
  else
    stem_s2d_kernel<uint8_t><<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(static_cast<const uint8_t*>(img), x2.hi, x2.lo,
                                                                           n, h, w, x2.h, x2.w, means[0], means[1], means[2]);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
}

// SSD conv1_1 (3x3, C_in = 3) staging for the tensor-core path: zero-padded image with 16-channel
// pixels (3 real), so that the 64 contiguous fp16 starting at pixel (y, x) are the filter-row window
// x-1 .. x+2 of row y-1 (the 4th pixel meets zero weights).  uint8 values are exact in fp16: lo = 0.
template <typename PIX>
__global__ void pack_c3_kernel(const PIX* __restrict__ img, __half* __restrict__ hi, __half* __restrict__ lo, int n,
                               int h, int w, int h2, int w2) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t total = (size_t)n * h2 * w2;
  if (i >= total) return;
  const int X = (int)(i % w2), Y = (int)((i / w2) % h2), ni = (int)(i / ((size_t)w2 * h2));
  uint4 vh[2], vl[2];
  __half* ph = reinterpret_cast<__half*>(vh);
  __half* pl = reinterpret_cast<__half*>(vl);
#pragma unroll
  for (int j = 0; j < 16; ++j) { ph[j] = __float2half_rn(0.f); pl[j] = __float2half_rn(0.f); }
  const int py = Y - 1, px = X - 1;
  if (py >= 0 && py < h && px >= 0 && px < w) {
    const PIX* p = img + (((size_t)ni * h + py) * w + px) * 3;
    // uint8 pixels are exact in fp16 (lo = 0); resized float pixels keep their low part
    split_f32((float)p[0], ph[0], pl[0]); split_f32((float)p[1], ph[1], pl[1]); split_f32((float)p[2], ph[2], pl[2]);
  }
  uint4* oh = reinterpret_cast<uint4*>(hi + i * 16);
  uint4* ol = reinterpret_cast<uint4*>(lo + i * 16);
  oh[0] = vh[0]; oh[1] = vh[1];
  ol[0] = vl[0]; ol[1] = vl[1];
}
void launch_pack_c3(const void* img, bool img_f32, int n, int h, int w, Act x2, cudaStream_t st) {
  size_t total = (size_t)n * x2.h * x2.w;
  if (!total) return;
  if (img_f32)
    pack_c3_kernel<float><<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(static_cast<const float*>(img), x2.hi, x2.lo, n, h,
                                                                        w, x2.h, x2.w);
  else
    pack_c3_kernel<uint8_t><<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(static_cast<const uint8_t*>(img), x2.hi, x2.lo,
                                                                          n, h, w, x2.h, x2.w);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
}

__global__ void f32_to_act_kernel(const float* __restrict__ x, __half* __restrict__ hi, __half* __restrict__ lo,
                                  size_t numel) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= numel) return;
  __half h, l;
  split_f32(x[i], h, l);
  hi[i] = h; lo[i] = l;
}
void launch_f32_to_act(const float* x, Act out, cudaStream_t st) {
  size_t n = out.numel();
  if (!n) return;
  f32_to_act_kernel<<<(unsigned)cdiv64(n, 256), 256, 0, st>>>(x, out.hi, out.lo, n);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
}

__global__ void act_to_f32_kernel(const __half* __restrict__ hi, const __half* __restrict__ lo, float* __restrict__ y,
                                  size_t numel) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= numel) return;
  y[i] = join_f16(hi[i], lo[i]);
}
// eight elements per thread: one 16 B load per plane, two 16 B stores (numel % 8 == 0, 16 B aligned planes)
__global__ void act_to_f32_vec8_kernel(const uint4* __restrict__ hi, const uint4* __restrict__ lo, float4* __restrict__ y,
                                       size_t nvec) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nvec) return;
  const uint4 h = __ldg(hi + i), l = __ldg(lo + i);
  const __half* ph = reinterpret_cast<const __half*>(&h);
  const __half* pl = reinterpret_cast<const __half*>(&l);
  float v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = join_f16(ph[j], pl[j]);
  y[2 * i] = make_float4(v[0], v[1], v[2], v[3]);
  y[2 * i + 1] = make_float4(v[4], v[5], v[6], v[7]);
}
void launch_act_to_f32(Act in, float* y, cudaStream_t st) {
  size_t n = in.numel();
  if (!n) return;
  const bool aligned = ((reinterpret_cast<uintptr_t>(in.hi) | reinterpret_cast<uintptr_t>(in.lo) |
                         reinterpret_cast<uintptr_t>(y)) & 15u) == 0;
  if ((n % 8) == 0 && aligned)
    act_to_f32_vec8_kernel<<<(unsigned)cdiv64(n / 8, 256), 256, 0, st>>>(
        reinterpret_cast<const uint4*>(in.hi), reinterpret_cast<const uint4*>(in.lo), reinterpret_cast<float4*>(y), n / 8);
  else
    act_to_f32_kernel<<<(unsigned)cdiv64(n, 256), 256, 0, st>>>(in.hi, in.lo, y, n);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
}

// max pool, 8 channels per thread (C % 8 == 0) -- slim max_pool2d / tf.nn.max_pool.
// Padded cells are ignored (TF pads with -inf).
// PRE: writes p = relu(fmaf(m^, pre_scale[c], pre_bias[c])) instead of the max m, with m^ = m as split and rejoined
// (the batch norm follows the max: a negative gamma does not commute with it).
template <bool PRE>
__global__ void max_pool_kernel(const __half* __restrict__ ihi, const __half* __restrict__ ilo,
                                __half* __restrict__ ohi, __half* __restrict__ olo, int n, int h, int w, int c,
                                int ho, int wo, int k, int stride, int pad_t, int pad_l,
                                const float* __restrict__ pre_scale, const float* __restrict__ pre_bias) {
  const int cv = c >> 3;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t total = (size_t)n * ho * wo * cv;
  if (i >= total) return;
  int c8 = (int)(i % cv);
  size_t p = i / cv;
  int ox = (int)(p % wo);
  int oy = (int)((p / wo) % ho);
  int ni = (int)(p / ((size_t)wo * ho));
  float best[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) best[j] = -INFINITY;
  for (int r = 0; r < k; ++r) {
    int iy = oy * stride + r - pad_t;
    if (iy < 0 || iy >= h) continue;
    for (int s = 0; s < k; ++s) {
      int ix = ox * stride + s - pad_l;
      if (ix < 0 || ix >= w) continue;
      size_t off = (((size_t)ni * h + iy) * w + ix) * c + (size_t)c8 * 8;
      uint4 vh = *reinterpret_cast<const uint4*>(ihi + off);
      uint4 vl = *reinterpret_cast<const uint4*>(ilo + off);
      const __half* ph = reinterpret_cast<const __half*>(&vh);
      const __half* pl = reinterpret_cast<const __half*>(&vl);
#pragma unroll
      for (int j = 0; j < 8; ++j) best[j] = fmaxf(best[j], join_f16(ph[j], pl[j]));
    }
  }
  uint4 oh, ol;
  __half* qh = reinterpret_cast<__half*>(&oh);
  __half* ql = reinterpret_cast<__half*>(&ol);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    split_f32(best[j], qh[j], ql[j]);
    if constexpr (PRE) {
      const int ch = c8 * 8 + j;
      split_f32(fmaxf(fmaf(join_f16(qh[j], ql[j]), pre_scale[ch], pre_bias[ch]), 0.f), qh[j], ql[j]);
    }
  }
  size_t ooff = p * c + (size_t)c8 * 8;
  *reinterpret_cast<uint4*>(ohi + ooff) = oh;
  *reinterpret_cast<uint4*>(olo + ooff) = ol;
}
void launch_max_pool(Act in, Act out, int k, int stride, int pad_t, int pad_l, cudaStream_t st,
                     const float* pre_scale, const float* pre_bias) {
  LUMI_REQUIRE(in.c % 8 == 0 && in.c == out.c && in.n == out.n, "max_pool: C must be a multiple of 8");
  LUMI_REQUIRE(!pre_scale == !pre_bias, "max_pool: pre_scale and pre_bias go together");
  size_t total = (size_t)out.n * out.h * out.w * (out.c / 8);
  if (!total) return;
  if (pre_scale)
    max_pool_kernel<true><<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(
        in.hi, in.lo, out.hi, out.lo, in.n, in.h, in.w, in.c, out.h, out.w, k, stride, pad_t, pad_l, pre_scale, pre_bias);
  else
    max_pool_kernel<false><<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(
        in.hi, in.lo, out.hi, out.lo, in.n, in.h, in.w, in.c, out.h, out.w, k, stride, pad_t, pad_l, nullptr, nullptr);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
}

// tf.nn.l2_normalize over channels x gamma (ssd/feature_extractor.py:62-76): one warp per pixel.
__global__ void l2norm_scale_kernel(const __half* __restrict__ ihi, const __half* __restrict__ ilo,
                                    __half* __restrict__ ohi, __half* __restrict__ olo,
                                    const float* __restrict__ gamma, size_t pixels, int c, float eps) {
  size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (warp >= pixels) return;
  const __half* ph = ihi + warp * c;
  const __half* pl = ilo + warp * c;
  float ss = 0.f;
  for (int j = lane; j < c; j += 32) { float v = join_f16(ph[j], pl[j]); ss = fmaf(v, v, ss); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  float inv = __frcp_rn(__fsqrt_rn(fmaxf(ss, eps)));
  for (int j = lane; j < c; j += 32) {
    float v = __fmul_rn(__fmul_rn(join_f16(ph[j], pl[j]), inv), gamma[j]);
    __half h, l;
    split_f32(v, h, l);
    ohi[warp * c + j] = h; olo[warp * c + j] = l;
  }
}
void launch_l2norm_scale(Act in, Act out, const float* gamma, float eps, cudaStream_t st) {
  size_t pixels = (size_t)in.n * in.h * in.w;
  if (!pixels) return;
  l2norm_scale_kernel<<<(unsigned)cdiv64(pixels * 32, 256), 256, 0, st>>>(in.hi, in.lo, out.hi, out.lo, gamma, pixels,
                                                                         in.c, eps);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
}

// tf.reduce_mean(features, [1, 2]) (rcnn.py:188)
__global__ void spatial_mean_kernel(const __half* __restrict__ ihi, const __half* __restrict__ ilo,
                                    __half* __restrict__ ohi, __half* __restrict__ olo, int rows, int hw, int c) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)rows * c) return;
  int ch = (int)(i % c);
  size_t r = i / c;
  const __half* ph = ihi + r * hw * c + ch;
  const __half* pl = ilo + r * hw * c + ch;
  float s = 0.f;
  for (int p = 0; p < hw; ++p) s += join_f16(ph[(size_t)p * c], pl[(size_t)p * c]);
  float v = __fdiv_rn(s, (float)hw);
  __half h, l;
  split_f32(v, h, l);
  ohi[i] = h; olo[i] = l;
}
void launch_spatial_mean(Act in, Act out, cudaStream_t st) {
  size_t total = (size_t)in.n * in.c;
  if (!total) return;
  spatial_mean_kernel<<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(in.hi, in.lo, out.hi, out.lo, in.n, in.h * in.w,
                                                                    in.c);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
}

// tf.nn.softmax over the first `cols` entries of each row: one warp per row.
__global__ void softmax_rows_kernel(const float* __restrict__ x, float* __restrict__ y, int rows, int cols,
                                    int in_stride) {
  int warp = (int)(((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  int lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const float* xr = x + (size_t)warp * in_stride;
  float m = -INFINITY;
  for (int j = lane; j < cols; j += 32) m = fmaxf(m, xr[j]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  float s = 0.f;
  for (int j = lane; j < cols; j += 32) s += expf(xr[j] - m);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  for (int j = lane; j < cols; j += 32) y[(size_t)warp * cols + j] = __fdiv_rn(expf(xr[j] - m), s);
}
void launch_softmax_rows(const float* x, float* y, int rows, int cols, int in_stride, cudaStream_t st) {
  if (!rows) return;
  softmax_rows_kernel<<<(unsigned)cdiv64((size_t)rows * 32, 256), 256, 0, st>>>(x, y, rows, cols, in_stride);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
}

// fasterrcnn.py:261-308 anchors: int32 reference (truncated, quirk Q1) + int32 shifts, cast to float
// where decode() needs them (bbox_transform_tf.py:6 `tf.cast(bboxes, tf.float32)`).
__global__ void frcnn_anchors_kernel(const int* __restrict__ ref, int A, int fh, int fw, int stride,
                                     float* __restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  int total = fh * fw * A;
  if (i >= total) return;
  int a = i % A;
  int cell = i / A;
  int sx = (cell % fw) * stride, sy = (cell / fw) * stride;
  float4 v = make_float4((float)(ref[a * 4 + 0] + sx), (float)(ref[a * 4 + 1] + sy), (float)(ref[a * 4 + 2] + sx),
                         (float)(ref[a * 4 + 3] + sy));
  reinterpret_cast<float4*>(out)[i] = v;
}
void launch_frcnn_anchors(const int* ref, int A, int fh, int fw, int stride, float* out, cudaStream_t st) {
  int total = fh * fw * A;
  if (!total) return;
  frcnn_anchors_kernel<<<cdiv(total, 256), 256, 0, st>>>(ref, A, fh, fw, stride, out);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
}

}  // namespace lumi
