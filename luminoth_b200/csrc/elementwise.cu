// HBM-bound elementwise / pooling / normalisation kernels (vectorised NHWC).
#include "ops.cuh"
#include <cstdint>
#include <type_traits>

namespace lumi {

void check_pixel_format(int format, bool f32, int h, int w, const std::string& who) {
  LUMI_REQUIRE(format >= PIX_RGB && format <= PIX_I420, who + ": unknown pixel format " + std::to_string(format) +
                                                            " (0 RGB, 1 BGR, 2 NV12, 3 I420)");
  if (!pix_yuv(format)) return;
  const char* name = format == PIX_NV12 ? "NV12" : "I420";
  LUMI_REQUIRE(!f32, who + ": " + name + " images are uint8");
  LUMI_REQUIRE(h % 2 == 0 && w % 2 == 0, who + ": " + name + " needs an even height and width, the image is " +
                                             std::to_string(h) + " x " + std::to_string(w));
}

// cv::cvtColor(COLOR_YUV2RGB_NV12 / _I420): BT.601 limited range in 20-bit fixed point, integer only.
__device__ __forceinline__ void yuv_to_rgb(int Y, int U, int V, float (&v)[3]) {
  const int uu = U - 128, vv = V - 128, yy = max(0, Y - 16) * 1220542 + (1 << 19);
  v[0] = (float)min(max((yy + 1673527 * vv) >> 20, 0), 255);
  v[1] = (float)min(max((yy - 852492 * vv - 409993 * uu) >> 20, 0), 255);
  v[2] = (float)min(max((yy + 2116026 * uu) >> 20, 0), 255);
}

// The RGB value of pixel (row, col) of the image at p in format FMT: RGB / BGR rows start `pitch` pixels apart; a YUV
// image's Y plane is plane_h rows of `pitch` bytes, its chroma planes follow (pitch and plane_h even).
template <int FMT, typename PIX>
__device__ __forceinline__ void load_pixel(const PIX* __restrict__ p, int pitch, int plane_h, int row, int col,
                                           float (&v)[3]) {
  if constexpr (FMT == PIX_RGB || FMT == PIX_BGR) {
    const PIX* q = p + ((size_t)row * pitch + col) * 3;
    const int r = FMT == PIX_RGB ? 0 : 2;
    v[0] = (float)q[r]; v[1] = (float)q[1]; v[2] = (float)q[2 - r];
  } else {
    static_assert(sizeof(PIX) == 1, "YUV pixels are uint8");
    const PIX* chroma = p + (size_t)plane_h * pitch;
    const size_t half = (size_t)(row >> 1) * (pitch >> 1) + (col >> 1);
    int u, v_;
    if constexpr (FMT == PIX_NV12) {
      u = chroma[2 * half]; v_ = chroma[2 * half + 1];
    } else {
      u = chroma[half]; v_ = chroma[(size_t)(plane_h >> 1) * (pitch >> 1) + half];
    }
    yuv_to_rgb(p[(size_t)row * pitch + col], u, v_, v);
  }
}

// tf.image.resize_images(BILINEAR) of TF 1.x (legacy kernel: align_corners=False, src = dst * (in / out), no
// half-pixel offset) -- luminoth/utils/image.py:94-97,139-142.  Same float32 operation order as the oracle
// (tf_ops.resize_bilinear), no FMA contraction, so the result is bit-identical to it.  Pixel (y, x) of the h x w
// output of the h0 x w0 image that starts at (oy, ox) of the image at src (load_pixel's pitch and plane_h), hs = h0 / h
// and ws = w0 / w in float32.  The taps are RGB values, so a converted format resizes like its RGB image.
template <int FMT, typename PIX>
__device__ __forceinline__ void bilinear_sample(const PIX* __restrict__ src, int h0, int w0, int pitch, int plane_h,
                                                int oy, int ox, float hs, float ws, int y, int x, float (&v)[3]) {
  const float fy = __fmul_rn((float)y, hs), fx = __fmul_rn((float)x, ws);
  const int y0 = (int)floorf(fy), x0 = (int)floorf(fx);
  const int y1 = min(y0 + 1, h0 - 1), x1 = min(x0 + 1, w0 - 1);
  const float yl = __fsub_rn(fy, (float)y0), xl = __fsub_rn(fx, (float)x0);
  float tl[3], tr[3], bl[3], br[3];
  load_pixel<FMT>(src, pitch, plane_h, oy + y0, ox + x0, tl);
  load_pixel<FMT>(src, pitch, plane_h, oy + y0, ox + x1, tr);
  load_pixel<FMT>(src, pitch, plane_h, oy + y1, ox + x0, bl);
  load_pixel<FMT>(src, pitch, plane_h, oy + y1, ox + x1, br);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float top = __fadd_rn(tl[c], __fmul_rn(__fsub_rn(tr[c], tl[c]), xl));
    const float bot = __fadd_rn(bl[c], __fmul_rn(__fsub_rn(br[c], bl[c]), xl));
    v[c] = __fadd_rn(top, __fmul_rn(__fsub_rn(bot, top), yl));
  }
}

template <typename PIX>
__global__ void resize_bilinear_kernel(const PIX* __restrict__ src, int h0, int w0, float* __restrict__ dst, int h, int w,
                                       float hs, float ws) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)h * w) return;
  float v[3];
  bilinear_sample<PIX_RGB>(src, h0, w0, w0, h0, 0, 0, hs, ws, (int)(i / w), (int)(i % w), v);
  dst[i * 3] = v[0]; dst[i * 3 + 1] = v[1]; dst[i * 3 + 2] = v[2];
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

// Pixel sources of the input staging kernels: pixel (y, x) of image ni of the h x w batch the network sees.
// DirectPixels: the batch itself, n images of h x w in format FMT one after the other.
template <typename PIX, int FMT>
struct DirectPixels {
  const PIX* img;
  int h, w;
  __device__ __forceinline__ bool inside(int, int, int) const { return true; }
  __device__ __forceinline__ void load(int ni, int y, int x, float (&v)[3]) const {
    const size_t image = pix_yuv(FMT) ? (size_t)h * w * 3 / 2 : (size_t)h * w * 3;
    load_pixel<FMT>(img + ni * image, w, h, y, x, v);
  }
};
// ResizedPixels: image ni is the source table[ni] locates in `base`, resized to its target on the fly -- the values
// launch_resize_bilinear writes, so a fused staging is bit-identical to resize-then-stage.  PACKED: the batch is a
// canvas, and only the pixels inside image ni's target th x tw are the image's.
template <typename PIX, bool PACKED, int FMT>
struct ResizedPixels {
  const uint8_t* base;
  const ResizeSrc* table;
  __device__ __forceinline__ bool inside(int ni, int y, int x) const {
    return !PACKED || (y < table[ni].th && x < table[ni].tw);
  }
  __device__ __forceinline__ void load(int ni, int y, int x, float (&v)[3]) const {
    const ResizeSrc t = table[ni];
    bilinear_sample<FMT>(reinterpret_cast<const PIX*>(base + t.off), t.h0, t.w0, t.pitch, t.plane_h, t.oy, t.ox, t.hs,
                         t.ws, y, x, v);
  }
};
// Calls f(format constant, pixel type) for the formats the readers are built for: RGB / BGR uint8 and float32, YUV
// uint8.  Every caller has run check_pixel_format, which refuses the rest with its own message.
template <typename F>
void with_format(int format, bool f32, F&& f) {
  using std::integral_constant;
  LUMI_REQUIRE(format >= PIX_RGB && format <= PIX_I420 && !(f32 && pix_yuv(format)),
               "with_format: unchecked pixel format " + std::to_string(format) + " (internal)");
  switch (format) {
    case PIX_RGB:
      if (f32) f(integral_constant<int, PIX_RGB>{}, float{});
      else f(integral_constant<int, PIX_RGB>{}, uint8_t{});
      break;
    case PIX_BGR:
      if (f32) f(integral_constant<int, PIX_BGR>{}, float{});
      else f(integral_constant<int, PIX_BGR>{}, uint8_t{});
      break;
    case PIX_NV12: f(integral_constant<int, PIX_NV12>{}, uint8_t{}); break;
    case PIX_I420: f(integral_constant<int, PIX_I420>{}, uint8_t{}); break;
  }
}
// Calls launch(pixels) with the source policy `src` describes.
template <typename F>
void with_pixels(const ImgSrc& src, int h, int w, F&& launch) {
  with_format(src.format, src.f32, [&](auto fmt, auto pix) {
    using PIX = decltype(pix);
    constexpr int FMT = decltype(fmt)::value;
    if (src.table) {
      const uint8_t* base = static_cast<const uint8_t*>(src.img);
      if (src.packed) launch(ResizedPixels<PIX, true, FMT>{base, src.table});
      else launch(ResizedPixels<PIX, false, FMT>{base, src.table});
    } else {
      launch(DirectPixels<PIX, FMT>{static_cast<const PIX*>(src.img), h, w});
    }
  });
}

// One image in any format -> [h][w][3] RGB of its dtype, through DirectPixels (the staging kernels' reader).
template <typename PIX, int FMT>
__global__ void pixels_to_rgb_kernel(DirectPixels<PIX, FMT> src, PIX* __restrict__ dst) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)src.h * src.w) return;
  float v[3];
  src.load(0, (int)(i / src.w), (int)(i % src.w), v);
  dst[i * 3] = (PIX)v[0]; dst[i * 3 + 1] = (PIX)v[1]; dst[i * 3 + 2] = (PIX)v[2];     // exact: v holds PIX values
}
void launch_pixels_to_rgb(const void* src, int format, bool f32, int h, int w, void* dst, cudaStream_t st) {
  check_pixel_format(format, f32, h, w, "pixels_to_rgb");
  const size_t total = (size_t)h * w;
  if (!total) return;
  with_format(format, f32, [&](auto fmt, auto pix) {
    using PIX = decltype(pix);
    const DirectPixels<PIX, decltype(fmt)::value> px{static_cast<const PIX*>(src), h, w};
    pixels_to_rgb_kernel<<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(px, static_cast<PIX*>(dst));
  });
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
}

// RGB image -> (optionally mean-subtracted) fp16x2 planes, one pixel per thread.
// base_network.py:153-177 (`inputs - [means]`, only for resnet*/vgg* architectures).
template <typename SRC>
__global__ void u8_to_act_kernel(SRC src, __half* __restrict__ hi, __half* __restrict__ lo, int n, int h, int w,
                                 float m0, float m1, float m2) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)n * h * w) return;
  const int x = (int)(i % w), y = (int)((i / w) % h), ni = (int)(i / ((size_t)w * h));
  if (!src.inside(ni, y, x)) {                    // canvas padding: the image's zero padding after mean subtraction
    const __half z = __float2half_rn(0.f);
    hi[i * 3] = hi[i * 3 + 1] = hi[i * 3 + 2] = z;
    lo[i * 3] = lo[i * 3 + 1] = lo[i * 3 + 2] = z;
    return;
  }
  float v[3];
  src.load(ni, y, x, v);
  split_f32(__fsub_rn(v[0], m0), hi[i * 3], lo[i * 3]);
  split_f32(__fsub_rn(v[1], m1), hi[i * 3 + 1], lo[i * 3 + 1]);
  split_f32(__fsub_rn(v[2], m2), hi[i * 3 + 2], lo[i * 3 + 2]);
}
void launch_u8_to_act(ImgSrc src, Act out, const float* means, cudaStream_t st) {
  LUMI_REQUIRE(out.c == 3, "u8_to_act: the staged image has 3 channels");
  const size_t total = (size_t)out.n * out.h * out.w;
  if (!total) return;
  const float m0 = means ? means[0] : 0.f, m1 = means ? means[1] : 0.f, m2 = means ? means[2] : 0.f;
  with_pixels(src, out.h, out.w, [&](auto px) {
    u8_to_act_kernel<<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(px, out.hi, out.lo, out.n, out.h, out.w, m0, m1, m2);
  });
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
}

// Space-to-depth staging of the 7x7/2 stem (slim conv2d_same: zero pad 3/3 AFTER mean subtraction):
// X2[n][Y][X][dy*6 + dx*3 + c] = xp[2Y+dy][2X+dx][c], xp = padded (image - mean); channels 12..15 = 0.
// The stem then is a 4x4/1 VALID conv over X2 that the tensor-core kernel runs as 4 taps of K = 64.
template <typename SRC>
__global__ void stem_s2d_kernel(SRC src, __half* __restrict__ hi, __half* __restrict__ lo, int n, int h, int w, int h2,
                                int w2, float m0, float m1, float m2) {
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
      if (py >= 0 && py < h && px >= 0 && px < w && src.inside(ni, py, px)) {
        float p[3];
        src.load(ni, py, px, p);
        const float v0 = __fsub_rn(p[0], m0), v1 = __fsub_rn(p[1], m1), v2 = __fsub_rn(p[2], m2);
        const int o = dy * 6 + dx * 3;
        split_f32(v0, ph[o], pl[o]); split_f32(v1, ph[o + 1], pl[o + 1]); split_f32(v2, ph[o + 2], pl[o + 2]);
      }
    }
  uint4* oh = reinterpret_cast<uint4*>(hi + i * 16);
  uint4* ol = reinterpret_cast<uint4*>(lo + i * 16);
  oh[0] = vh[0]; oh[1] = vh[1]; ol[0] = vl[0]; ol[1] = vl[1];
}
void launch_stem_s2d(ImgSrc src, int n, int h, int w, Act x2, const float* means, cudaStream_t st) {
  size_t total = (size_t)n * x2.h * x2.w;
  if (!total) return;
  with_pixels(src, h, w, [&](auto px) {
    stem_s2d_kernel<<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(px, x2.hi, x2.lo, n, h, w, x2.h, x2.w, means[0],
                                                                  means[1], means[2]);
  });
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
}

// SSD conv1_1 (3x3, C_in = 3) staging for the tensor-core path: zero-padded image with 16-channel
// pixels (3 real), so that the 64 contiguous fp16 starting at pixel (y, x) are the filter-row window
// x-1 .. x+2 of row y-1 (the 4th pixel meets zero weights).  uint8 values are exact in fp16: lo = 0.
template <typename SRC>
__global__ void pack_c3_kernel(SRC src, __half* __restrict__ hi, __half* __restrict__ lo, int n, int h, int w, int h2,
                               int w2) {
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
  if (py >= 0 && py < h && px >= 0 && px < w && src.inside(ni, py, px)) {
    float p[3];
    src.load(ni, py, px, p);
    // uint8 pixels are exact in fp16 (lo = 0); resized float pixels keep their low part
    split_f32(p[0], ph[0], pl[0]); split_f32(p[1], ph[1], pl[1]); split_f32(p[2], ph[2], pl[2]);
  }
  uint4* oh = reinterpret_cast<uint4*>(hi + i * 16);
  uint4* ol = reinterpret_cast<uint4*>(lo + i * 16);
  oh[0] = vh[0]; oh[1] = vh[1];
  ol[0] = vl[0]; ol[1] = vl[1];
}
void launch_pack_c3(ImgSrc src, int n, int h, int w, Act x2, cudaStream_t st) {
  size_t total = (size_t)n * x2.h * x2.w;
  if (!total) return;
  with_pixels(src, h, w, [&](auto px) {
    pack_c3_kernel<<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(px, x2.hi, x2.lo, n, h, w, x2.h, x2.w);
  });
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
// PACKED: image ni of a canvas batch -- its own input extent and SAME front padding (tab, in_stride), and 0 past its
// own output extent.
template <bool PRE, bool PACKED>
__global__ void max_pool_kernel(const __half* __restrict__ ihi, const __half* __restrict__ ilo,
                                __half* __restrict__ ohi, __half* __restrict__ olo, int n, int h, int w, int c,
                                int ho, int wo, int k, int stride, int pad_t, int pad_l,
                                const float* __restrict__ pre_scale, const float* __restrict__ pre_bias,
                                const ResizeSrc* __restrict__ tab, int in_stride) {
  const int cv = c >> 3;
  const int hc = h, wc = w;                       // the input's layout; h x w: the extent the window may read
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t total = (size_t)n * ho * wo * cv;
  if (i >= total) return;
  int c8 = (int)(i % cv);
  size_t p = i / cv;
  int ox = (int)(p % wo);
  int oy = (int)((p / wo) % ho);
  int ni = (int)(p / ((size_t)wo * ho));
  if constexpr (PACKED) {
    const int th = tab[ni].th, tw = tab[ni].tw;
    h = (th + in_stride - 1) / in_stride;
    w = (tw + in_stride - 1) / in_stride;
    const int oh = (h + stride - 1) / stride, ow = (w + stride - 1) / stride;
    if (oy >= oh || ox >= ow) {
      const size_t ooff = p * c + (size_t)c8 * 8;
      *reinterpret_cast<uint4*>(ohi + ooff) = make_uint4(0u, 0u, 0u, 0u);
      *reinterpret_cast<uint4*>(olo + ooff) = make_uint4(0u, 0u, 0u, 0u);
      return;
    }
    pad_t = max((oh - 1) * stride + k - h, 0) / 2;
    pad_l = max((ow - 1) * stride + k - w, 0) / 2;
  }
  float best[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) best[j] = -INFINITY;
  for (int r = 0; r < k; ++r) {
    int iy = oy * stride + r - pad_t;
    if (iy < 0 || iy >= h) continue;
    for (int s = 0; s < k; ++s) {
      int ix = ox * stride + s - pad_l;
      if (ix < 0 || ix >= w) continue;
      size_t off = (((size_t)ni * hc + iy) * wc + ix) * c + (size_t)c8 * 8;
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
                     const float* pre_scale, const float* pre_bias, const ResizeSrc* tab, int in_stride) {
  LUMI_REQUIRE(in.c % 8 == 0 && in.c == out.c && in.n == out.n, "max_pool: C must be a multiple of 8");
  LUMI_REQUIRE(!pre_scale == !pre_bias, "max_pool: pre_scale and pre_bias go together");
  LUMI_REQUIRE(!tab || in_stride > 0, "max_pool: a packed batch needs the input stride");
  size_t total = (size_t)out.n * out.h * out.w * (out.c / 8);
  if (!total) return;
  const unsigned grid = (unsigned)cdiv64(total, 256);
  auto go = [&](auto kernel) {
    kernel<<<grid, 256, 0, st>>>(in.hi, in.lo, out.hi, out.lo, in.n, in.h, in.w, in.c, out.h, out.w, k, stride, pad_t,
                                 pad_l, pre_scale, pre_bias, tab, in_stride);
  };
  if (tab) {
    if (pre_scale) go(max_pool_kernel<true, true>);
    else go(max_pool_kernel<false, true>);
  } else {
    if (pre_scale) go(max_pool_kernel<true, false>);
    else go(max_pool_kernel<false, false>);
  }
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
}

// Band clear of a packed batch: along each axis, image ni's valid outputs of the conv read input cells up to
// max_read = (out - 1) * stride - pad + k_eff - 1, out = ceil(ext / stride) (SAME and conv2d_same alike), ext = the
// image's extent ceil(t / in_stride).  Cells [ext, min(max_read + 1, canvas)) are the zero padding the image has alone;
// the canvas holds other values there.  Grid (., n): the first bh * w pixels are the candidate rows ext .. ext+bh-1, the
// next h * bw the candidate columns; 8 channels per thread.
__global__ void band_clear_kernel(__half* __restrict__ hi, __half* __restrict__ lo, int h, int w, int c,
                                  const ResizeSrc* __restrict__ tab, int in_stride, int keff_h, int keff_w, int stride,
                                  int pad_t, int pad_l, int bh, int bw) {
  const int ni = blockIdx.y, cv = c >> 3;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t rows = (size_t)bh * w * cv;
  if (i >= rows + (size_t)h * bw * cv) return;
  const int ext_h = (tab[ni].th + in_stride - 1) / in_stride, ext_w = (tab[ni].tw + in_stride - 1) / in_stride;
  const int end_h = min(((ext_h + stride - 1) / stride - 1) * stride - pad_t + keff_h, h);
  const int end_w = min(((ext_w + stride - 1) / stride - 1) * stride - pad_l + keff_w, w);
  const int c8 = (int)(i % cv);
  int y, x;
  if (i < rows) { const size_t p = i / cv; y = ext_h + (int)(p / w); x = (int)(p % w); if (y >= end_h) return; }
  else { const size_t p = (i - rows) / cv; y = (int)(p / bw); x = ext_w + (int)(p % bw); if (x >= end_w) return; }
  const size_t off = (((size_t)ni * h + y) * w + x) * c + (size_t)c8 * 8;
  *reinterpret_cast<uint4*>(hi + off) = make_uint4(0u, 0u, 0u, 0u);
  *reinterpret_cast<uint4*>(lo + off) = make_uint4(0u, 0u, 0u, 0u);
}
void launch_band_clear(Act a, const ResizeSrc* tab, int in_stride, int kh, int kw, int stride, int rate, int pad_t,
                       int pad_l, cudaStream_t st) {
  LUMI_REQUIRE(a.c % 8 == 0 && tab && in_stride > 0, "band_clear: C must be a multiple of 8 (internal)");
  const int keff_h = kh + (kh - 1) * (rate - 1), keff_w = kw + (kw - 1) * (rate - 1);
  // (out - 1) * stride <= ext - 1, so the band is at most k_eff - 1 - pad cells wide
  const int bh = keff_h - 1 - pad_t > 0 ? keff_h - 1 - pad_t : 0, bw = keff_w - 1 - pad_l > 0 ? keff_w - 1 - pad_l : 0;
  const size_t total = ((size_t)bh * a.w + (size_t)a.h * bw) * (a.c / 8);
  if (!total || !a.n) return;
  band_clear_kernel<<<dim3((unsigned)cdiv64(total, 256), a.n), 256, 0, st>>>(a.hi, a.lo, a.h, a.w, a.c, tab, in_stride,
                                                                             keff_h, keff_w, stride, pad_t, pad_l, bh, bw);
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
