// ROI crop (bilinear, tf.image.crop_and_resize) fused with the 2x2/2 max pool
// -- luminoth/models/fasterrcnn/roi_pool.py:37-95 (quirks Q3/Q4: boxes are
// normalised by the IMAGE size, crop size is [2*pooled_width, 2*pooled_height]).
//
// One CTA = one ROI x 256-channel slice; 8 warps walk the pooled cells, a lane owns 8 channels.
// The gather reads an fp32 copy of the feature map (made once per forward) so a tap costs two 16 B
// loads and no conversions; taps shared by the 2x2 samples of a cell are loaded once.  The kernel is
// instruction / L1-bound (12.8 G bilinear taps per batch at R = 2000), not HBM-bound.
#include "ops.cuh"
#include <cstdlib>
#include <string>

namespace lumi {

struct RoiArgs {
  const float* fmap;         // fp32 NHWC copy of the feature map (one-off conversion; saves 3 instr / element / tap)
  int n, fh, fw, c;
  const float* rois; const int* counts; int rmax;
  float im_h, im_w;
  const ResizeSrc* tab;      // packed batch: image i is tab[i].th x tw on a ceil(th / feat_stride) x ... grid, or nullptr
  int feat_stride;
  int crop_h, crop_w;        // 2*pw, 2*ph  (sic)
  __half* ohi; __half* olo;  // (n*rmax, crop_h/2, crop_w/2, c) or nullptr (mean only)
  __half* mhi; __half* mlo;  // optional fused tf.reduce_mean over the pooled cells: (n*rmax, c)
};

struct Samp { int lo, hi; float lerp; int ok; };    // one crop sample coordinate along y or x

// The image size the rois of image img are normalised by, and its feature grid (D - 1 is the crop's last cell): the
// batch's, or in a packed batch the image's own -- the map's row pitch stays a.fw.
__device__ __forceinline__ void roi_geometry(const RoiArgs& a, int img, bool is_y, float& im, int& D) {
  if (a.tab) {
    const int t = is_y ? a.tab[img].th : a.tab[img].tw;
    im = (float)t;
    D = (t + a.feat_stride - 1) / a.feat_stride;
  } else {
    im = is_y ? a.im_h : a.im_w;
    D = is_y ? a.fh : a.fw;
  }
}

template <int CPL>
__device__ __forceinline__ void load8f(const float* f, size_t off, float (&v)[CPL]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(f + off));
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
  if (CPL == 8) {
    const float4 b = __ldg(reinterpret_cast<const float4*>(f + off) + 1);
    v[CPL - 4] = b.x; v[CPL - 3] = b.y; v[CPL - 2] = b.z; v[CPL - 1] = b.w;
  }
}

// horizontal lerp of one feature row at the two x samples of a pooled cell; column loads are shared
// between the two samples whenever they hit the same feature cell (all indices are warp-uniform).
template <int CPL>
__device__ __forceinline__ void lerp8(const float (&l)[CPL], const float (&r)[CPL], float t, float (&h)[CPL]) {
#pragma unroll
  for (int j = 0; j < CPL; ++j) h[j] = fmaf(r[j] - l[j], t, l[j]);     // left + (right - left) * lerp
}
// Every re-use case names its source registers statically, so sharing a column costs no register moves (copying the
// shared values into l1 / r1 first measured 2.48 ms vs 2.38 ms per step).  The same treatment of the row-level sharing
// in the caller is register-neutral on its own (2.40 ms) but spills when combined with this one (3.43 ms): not done.
template <int CPL>
__device__ __forceinline__ void row_interp(const float* f, size_t rowbase, int c, int c0, const Samp& s0,
                                           const Samp& s1, float (&h0)[CPL], float (&h1)[CPL]) {
  float l0[CPL], r0[CPL], l1[CPL], r1[CPL];
  const float* row = f + rowbase * c + c0;
  load8f<CPL>(row, (size_t)s0.lo * c, l0);
  const bool r0_is_l0 = s0.hi == s0.lo;
  if (!r0_is_l0) { load8f<CPL>(row, (size_t)s0.hi * c, r0); lerp8<CPL>(l0, r0, s0.lerp, h0); }
  else lerp8<CPL>(l0, l0, s0.lerp, h0);
  if (s1.lo == s0.lo) {                                        // left1 = left0
    if (s1.hi == s0.hi) { if (r0_is_l0) lerp8<CPL>(l0, l0, s1.lerp, h1); else lerp8<CPL>(l0, r0, s1.lerp, h1); }
    else if (s1.hi == s1.lo) lerp8<CPL>(l0, l0, s1.lerp, h1);
    else { load8f<CPL>(row, (size_t)s1.hi * c, r1); lerp8<CPL>(l0, r1, s1.lerp, h1); }
  } else if (s1.lo == s0.hi) {                                 // left1 = right0 (r0 is loaded: s0.hi != s0.lo here)
    if (s1.hi == s0.hi || s1.hi == s1.lo) lerp8<CPL>(r0, r0, s1.lerp, h1);
    else { load8f<CPL>(row, (size_t)s1.hi * c, r1); lerp8<CPL>(r0, r1, s1.lerp, h1); }
  } else {
    load8f<CPL>(row, (size_t)s1.lo * c, l1);
    if (s1.hi == s0.hi) { if (r0_is_l0) lerp8<CPL>(l1, l0, s1.lerp, h1); else lerp8<CPL>(l1, r0, s1.lerp, h1); }
    else if (s1.hi == s1.lo) lerp8<CPL>(l1, l1, s1.lerp, h1);
    else { load8f<CPL>(row, (size_t)s1.hi * c, r1); lerp8<CPL>(l1, r1, s1.lerp, h1); }
  }
}

// RB consecutive ROIs per CTA: their RB*49 pooled cells are dealt round-robin to the 8 warps.  With one ROI per
// CTA, 49 cells on 8 warps leave seven warps idle for 1/8 of the CTA's life (ncu: 10 % of all samples stalled at the
// final barrier); with four ROIs the imbalance is 196 = 8*24 + 4 -> 2 %.
template <int CPL, int RB, int NW>
__global__ void __launch_bounds__(32 * NW, (CPL == 8 ? 2 : 3) * (8 / NW)) roi_pool_kernel(const RoiArgs a) {
  constexpr int SLICE = 32 * CPL;             // channels per CTA (one warp-wide vector of CPL channels per lane)
  const int row0 = blockIdx.x * RB;           // first global roi row (= img*rmax + r) of this CTA
  const int rows_total = a.n * a.rmax;
  const int cslice = blockIdx.y * SLICE;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c0 = cslice + lane * CPL;
  const int oh = a.crop_h >> 1, ow = a.crop_w >> 1;
  const int ncell = oh * ow;

  // sample tables: crop_h y-samples then crop_w x-samples (TF crop_and_resize arithmetic, once per CTA and ROI)
  __shared__ Samp samp_all[RB][64];
  const int nsamp = a.crop_h + a.crop_w;
  if ((int)threadIdx.x < RB * nsamp && row0 + (int)threadIdx.x / nsamp < rows_total) {
    const int rl_ = threadIdx.x / nsamp, ts = threadIdx.x % nsamp;
    const int row = row0 + rl_;
    const bool is_y = ts < a.crop_h;
    const int k = is_y ? ts : ts - a.crop_h;
    const float* rb = a.rois + (size_t)row * 4;
    float im; int D;
    roi_geometry(a, row / a.rmax, is_y, im, D);
    // normalised box, TF order (y1,x1,y2,x2): divided by the IMAGE size (quirk Q3)
    const float lo_n = __fdiv_rn(is_y ? rb[1] : rb[0], im);
    const float hi_n = __fdiv_rn(is_y ? rb[3] : rb[2], im);
    const int crop = is_y ? a.crop_h : a.crop_w;
    const float Dm1 = (float)(D - 1);
    const float step = crop > 1 ? __fdiv_rn(__fmul_rn(__fsub_rn(hi_n, lo_n), Dm1), (float)(crop - 1)) : 0.f;
    const float in = crop > 1 ? __fadd_rn(__fmul_rn(lo_n, Dm1), __fmul_rn((float)k, step))
                              : __fmul_rn(__fmul_rn(0.5f, __fadd_rn(lo_n, hi_n)), Dm1);
    Samp s;
    s.ok = !(in < 0.f || in > Dm1);
    s.lo = s.ok ? (int)floorf(in) : 0;
    s.hi = s.ok ? (int)ceilf(in) : 0;
    s.lerp = __fsub_rn(in, (float)s.lo);
    samp_all[rl_][ts] = s;
  }
  __syncthreads();

  __shared__ float part[RB][NW][SLICE];       // per-warp partial sums of the fused spatial mean
  float msum[CPL];
#pragma unroll
  for (int j = 0; j < CPL; ++j) msum[j] = 0.f;
  for (int rl = 0; rl < RB; ++rl) {
    const int row = row0 + rl;
    if (row >= rows_total) break;
    const int img = row / a.rmax, r = row - img * a.rmax;
    const bool live = (a.counts == nullptr || r < a.counts[img]) && c0 < a.c;
    const size_t obase = (size_t)row * ncell * a.c;
    const float* f = a.fmap + (size_t)img * a.fh * a.fw * a.c;
    const Samp* samp = samp_all[rl];
    // the RB*ncell cells of the CTA are dealt round-robin: this warp's first cell inside ROI rl
    const int first = (((warp - rl * ncell) % NW) + NW) % NW;
  for (int cell = first; cell < ncell; cell += NW) {
    if (c0 >= a.c) break;
    const int py = cell / ow, px = cell % ow;
    float best[CPL];
#pragma unroll
    for (int j = 0; j < CPL; ++j) best[j] = live ? -INFINITY : 0.f;
    if (live) {
      const Samp y0 = samp[py * 2], y1 = samp[py * 2 + 1];
      const Samp x0 = samp[a.crop_h + px * 2], x1 = samp[a.crop_h + px * 2 + 1];
      // row-interpolated values, shared between the two y samples when they touch the same feature rows
      float t0[2][CPL], b0[2][CPL];          // sample row 0: top / bottom feature row, [sx][ch]
      row_interp<CPL>(f, (size_t)y0.lo * a.fw, a.c, c0, x0, x1, t0[0], t0[1]);
      if (y0.hi != y0.lo) row_interp<CPL>(f, (size_t)y0.hi * a.fw, a.c, c0, x0, x1, b0[0], b0[1]);
      else {
#pragma unroll
        for (int j = 0; j < CPL; ++j) { b0[0][j] = t0[0][j]; b0[1][j] = t0[1][j]; }
      }
#pragma unroll
      for (int sx = 0; sx < 2; ++sx) {
        const bool ok = y0.ok && (sx ? x1.ok : x0.ok);          // warp-uniform
        if (ok) {
#pragma unroll
          for (int j = 0; j < CPL; ++j) best[j] = fmaxf(best[j], fmaf(b0[sx][j] - t0[sx][j], y0.lerp, t0[sx][j]));
        } else {
#pragma unroll
          for (int j = 0; j < CPL; ++j) best[j] = fmaxf(best[j], 0.f);              // extrapolation_value = 0
        }
      }
      float t1[2][CPL], b1[2][CPL];
      if (y1.lo == y0.lo) {
#pragma unroll
        for (int j = 0; j < CPL; ++j) { t1[0][j] = t0[0][j]; t1[1][j] = t0[1][j]; }
      } else if (y1.lo == y0.hi) {
#pragma unroll
        for (int j = 0; j < CPL; ++j) { t1[0][j] = b0[0][j]; t1[1][j] = b0[1][j]; }
      } else {
        row_interp<CPL>(f, (size_t)y1.lo * a.fw, a.c, c0, x0, x1, t1[0], t1[1]);
      }
      if (y1.hi == y0.hi) {
#pragma unroll
        for (int j = 0; j < CPL; ++j) { b1[0][j] = b0[0][j]; b1[1][j] = b0[1][j]; }
      } else if (y1.hi == y1.lo) {
#pragma unroll
        for (int j = 0; j < CPL; ++j) { b1[0][j] = t1[0][j]; b1[1][j] = t1[1][j]; }
      } else {
        row_interp<CPL>(f, (size_t)y1.hi * a.fw, a.c, c0, x0, x1, b1[0], b1[1]);
      }
#pragma unroll
      for (int sx = 0; sx < 2; ++sx) {
        const bool ok = y1.ok && (sx ? x1.ok : x0.ok);
        if (ok) {
#pragma unroll
          for (int j = 0; j < CPL; ++j) best[j] = fmaxf(best[j], fmaf(b1[sx][j] - t1[sx][j], y1.lerp, t1[sx][j]));
        } else {
#pragma unroll
          for (int j = 0; j < CPL; ++j) best[j] = fmaxf(best[j], 0.f);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < CPL; ++j) msum[j] += best[j];
    if (a.ohi) {
      uint4 vh, vl;
      __half* qh = reinterpret_cast<__half*>(&vh);
      __half* ql = reinterpret_cast<__half*>(&vl);
#pragma unroll
      for (int j = 0; j < CPL; ++j) split_f32(best[j], qh[j], ql[j]);
      const size_t off = obase + (size_t)cell * a.c + c0;
      if (CPL == 8) {
        *reinterpret_cast<uint4*>(a.ohi + off) = vh;
        *reinterpret_cast<uint4*>(a.olo + off) = vl;
      } else {
        *reinterpret_cast<uint2*>(a.ohi + off) = make_uint2(vh.x, vh.y);
        *reinterpret_cast<uint2*>(a.olo + off) = make_uint2(vl.x, vl.y);
      }
    }
  }
    if (a.mhi) {          // this warp's share of ROI rl
#pragma unroll
      for (int j = 0; j < CPL; ++j) { part[rl][warp][lane * CPL + j] = msum[j]; msum[j] = 0.f; }
    }
  }
  if (a.mhi) {            // fused spatial mean (rcnn.py:188): warp partials -> fixed-order sum -> / cells
    __syncthreads();
    for (int i = threadIdx.x; i < SLICE; i += 32 * NW) {
      const int ch = cslice + i;
      if (ch >= a.c) break;
      for (int rl = 0; rl < RB && row0 + rl < rows_total; ++rl) {
        float s = 0.f;
#pragma unroll
        for (int w8 = 0; w8 < NW; ++w8) s += part[rl][w8][i];
        const float v = __fdiv_rn(s, (float)ncell);
        __half h, l;
        split_f32(v, h, l);
        a.mhi[(size_t)(row0 + rl) * a.c + ch] = h;
        a.mlo[(size_t)(row0 + rl) * a.c + ch] = l;
      }
    }
  }
}


// =====================================================================================================================
// Column-walk kernel (round 2).  One WARP = one ROI x one channel slice (32 lanes x CPL channels); no shared memory,
// no CTA-level synchronisation.  For each pooled column q the warp walks the 2*oh sample rows top to bottom and keeps
// the horizontally interpolated values of the last two feature rows it touched in registers (H0 / H1, tagged with
// their row index): vertically adjacent samples -- inside a cell AND across cells -- reuse them, so each feature row
// is fetched once per pooled column instead of once per sample row (round-1 kernel: sharing inside one 2x2 cell only).
// The sample tables live in the lanes of the warp (lane t = sample t) and are broadcast with shuffles.
// =====================================================================================================================
template <int CPL> struct RoiVec { float2 p[CPL / 2]; };

template <int CPL>
__device__ __forceinline__ RoiVec<CPL> roi_load(const float* f, int off) {
  RoiVec<CPL> v;
  const float4 a = __ldg(reinterpret_cast<const float4*>(f + off));
  v.p[0] = make_float2(a.x, a.y); v.p[1] = make_float2(a.z, a.w);
  if (CPL == 8) {
    const float4 b = __ldg(reinterpret_cast<const float4*>(f + off) + 1);
    v.p[CPL / 2 - 2] = make_float2(b.x, b.y); v.p[CPL / 2 - 1] = make_float2(b.z, b.w);
  }
  return v;
}
// l + (r - l) * t   (TF: top_left + (top_right - top_left) * x_lerp; the multiply-add is contracted like the
// round-1 kernel and like any -O2 CPU build with FMA)
template <int CPL>
__device__ __forceinline__ RoiVec<CPL> roi_lerp(const RoiVec<CPL>& l, const RoiVec<CPL>& r, float t) {
  RoiVec<CPL> h;
#pragma unroll
  for (int j = 0; j < CPL / 2; ++j)
    h.p[j] = make_float2(__fmaf_rn(__fsub_rn(r.p[j].x, l.p[j].x), t, l.p[j].x),
                         __fmaf_rn(__fsub_rn(r.p[j].y, l.p[j].y), t, l.p[j].y));
  return h;
}
struct RoiX { int lo, hi; float t; int ok; };   // lo / hi: ELEMENT offsets of the two feature columns (x * C)
// horizontal interpolation of feature row `rowoff` (element offset of its first pixel) at the two x samples of a
// pooled column; loads shared between the two samples are issued once (all indices are warp-uniform)
template <int CPL>
__device__ __forceinline__ void roi_row(const float* f, int rowoff, const RoiX& s0, const RoiX& s1,
                                        RoiVec<CPL>& h0, RoiVec<CPL>& h1) {
  constexpr int c = 1;                                  // offsets are already in elements (32-bit: one IMAD.WIDE per load)
  const RoiVec<CPL> l0 = roi_load<CPL>(f, rowoff + s0.lo * c);
  const bool r0_is_l0 = s0.hi == s0.lo;
  RoiVec<CPL> r0 = l0;
  if (!r0_is_l0) r0 = roi_load<CPL>(f, rowoff + s0.hi * c);
  h0 = roi_lerp<CPL>(l0, r0, s0.t);
  if (s1.lo == s0.lo) {
    if (s1.hi == s0.hi) h1 = roi_lerp<CPL>(l0, r0, s1.t);
    else if (s1.hi == s1.lo) h1 = roi_lerp<CPL>(l0, l0, s1.t);
    else { const RoiVec<CPL> r1 = roi_load<CPL>(f, rowoff + s1.hi * c); h1 = roi_lerp<CPL>(l0, r1, s1.t); }
  } else if (s1.lo == s0.hi) {
    if (s1.hi == s1.lo) h1 = roi_lerp<CPL>(r0, r0, s1.t);
    else { const RoiVec<CPL> r1 = roi_load<CPL>(f, rowoff + s1.hi * c); h1 = roi_lerp<CPL>(r0, r1, s1.t); }
  } else {
    const RoiVec<CPL> l1 = roi_load<CPL>(f, rowoff + s1.lo * c);
    if (s1.hi == s1.lo) h1 = roi_lerp<CPL>(l1, l1, s1.t);
    else { const RoiVec<CPL> r1 = roi_load<CPL>(f, rowoff + s1.hi * c); h1 = roi_lerp<CPL>(l1, r1, s1.t); }
  }
}

template <int CPL>
__device__ __forceinline__ void roi_max_sample(RoiVec<CPL>& best, const RoiVec<CPL>& top, const RoiVec<CPL>& bot,
                                               float ly, bool ok) {
  if (ok) {
    const RoiVec<CPL> v = roi_lerp<CPL>(top, bot, ly);
#pragma unroll
    for (int j = 0; j < CPL / 2; ++j) { best.p[j].x = fmaxf(best.p[j].x, v.p[j].x); best.p[j].y = fmaxf(best.p[j].y, v.p[j].y); }
  } else {                                              // extrapolation_value = 0
#pragma unroll
    for (int j = 0; j < CPL / 2; ++j) { best.p[j].x = fmaxf(best.p[j].x, 0.f); best.p[j].y = fmaxf(best.p[j].y, 0.f); }
  }
}

// one sample row: (re)compute the rows that are not resident, then the two bilinear samples of the pooled column.
// HT / HB are the register sets currently playing "top" / "bottom" (the caller dispatches on the role parity).
template <int CPL>
__device__ __forceinline__ void roi_step(const float* f, int rowstride, int ylo, int yhi, float ly, bool need_top,
                                         bool need_bot, const RoiX& x0, const RoiX& x1, RoiVec<CPL> (&HT)[2],
                                         RoiVec<CPL> (&HB)[2], RoiVec<CPL>& best) {
  if (need_top) roi_row<CPL>(f, ylo * rowstride, x0, x1, HT[0], HT[1]);
  if (need_bot) roi_row<CPL>(f, yhi * rowstride, x0, x1, HB[0], HB[1]);
  if (yhi == ylo) {
    roi_max_sample<CPL>(best, HT[0], HT[0], ly, x0.ok != 0);
    roi_max_sample<CPL>(best, HT[1], HT[1], ly, x1.ok != 0);
  } else {
    roi_max_sample<CPL>(best, HT[0], HB[0], ly, x0.ok != 0);
    roi_max_sample<CPL>(best, HT[1], HB[1], ly, x1.ok != 0);
  }
}

template <int CPL, int WARPS>
__global__ void __launch_bounds__(32 * WARPS) roi_pool_cols_kernel(const RoiArgs a) {
  constexpr int SLICE = 32 * CPL;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x;                                   // global roi row = img * rmax + r
  const int slice = blockIdx.y * WARPS + warp;
  if (slice * SLICE >= a.c) return;                             // whole warp
  const int c0 = slice * SLICE + lane * CPL;
  const bool lane_ok = c0 < a.c;
  const int img = row / a.rmax, r = row - img * a.rmax;
  const int oh = a.crop_h >> 1, ow = a.crop_w >> 1;
  const int ncell = oh * ow;
  const bool live = (a.counts == nullptr || r < a.counts[img]);
  if (!live) {                                                  // padded row: zeros (the heads read every row)
    if (lane_ok) {
      if (a.ohi)
        for (int cell = 0; cell < ncell; ++cell) {
          const size_t off = ((size_t)row * ncell + cell) * a.c + c0;
#pragma unroll
          for (int j = 0; j < CPL; ++j) { a.ohi[off + j] = __float2half_rn(0.f); a.olo[off + j] = __float2half_rn(0.f); }
        }
      if (a.mhi)
#pragma unroll
        for (int j = 0; j < CPL; ++j) { a.mhi[(size_t)row * a.c + c0 + j] = __float2half_rn(0.f); a.mlo[(size_t)row * a.c + c0 + j] = __float2half_rn(0.f); }
    }
    return;
  }
  // ---- sample table: lane t < crop_h holds y sample t, lanes crop_h .. crop_h+crop_w-1 the x samples (TF
  // crop_and_resize arithmetic in the reference's operation order; boxes normalised by the IMAGE size, quirk Q3)
  int s_lo = 0, s_hi = 0, s_ok = 0;
  float s_t = 0.f;
  {
    const int nsamp = a.crop_h + a.crop_w;                      // <= 32 (checked by the launcher)
    if (lane < nsamp) {
      const bool is_y = lane < a.crop_h;
      const int k = is_y ? lane : lane - a.crop_h;
      const float* rb = a.rois + (size_t)row * 4;
      float im; int D;
      roi_geometry(a, img, is_y, im, D);
      const float lo_n = __fdiv_rn(is_y ? rb[1] : rb[0], im);
      const float hi_n = __fdiv_rn(is_y ? rb[3] : rb[2], im);
      const int crop = is_y ? a.crop_h : a.crop_w;
      const float Dm1 = (float)(D - 1);
      const float step = crop > 1 ? __fdiv_rn(__fmul_rn(__fsub_rn(hi_n, lo_n), Dm1), (float)(crop - 1)) : 0.f;
      const float in = crop > 1 ? __fadd_rn(__fmul_rn(lo_n, Dm1), __fmul_rn((float)k, step))
                                : __fmul_rn(__fmul_rn(0.5f, __fadd_rn(lo_n, hi_n)), Dm1);
      s_ok = !(in < 0.f || in > Dm1);
      s_lo = s_ok ? (int)floorf(in) : 0;
      s_hi = s_ok ? (int)ceilf(in) : 0;
      s_t = __fsub_rn(in, (float)s_lo);
    }
  }
  const float* f = a.fmap + (size_t)img * a.fh * a.fw * a.c + (lane_ok ? c0 : 0);
  asm volatile("" : "+l"(f));     // keep ONE per-lane base pointer: every tap address is then base + 32-bit offset
  const int rowstride = a.fw * a.c;
  RoiVec<CPL> msum;
#pragma unroll
  for (int j = 0; j < CPL / 2; ++j) msum.p[j] = make_float2(0.f, 0.f);
  constexpr unsigned FULL = 0xffffffffu;
  for (int q = 0; q < ow; ++q) {
    RoiX x0, x1;
    const int lx = a.crop_h + 2 * q;
    x0.lo = __shfl_sync(FULL, s_lo, lx) * a.c; x0.hi = __shfl_sync(FULL, s_hi, lx) * a.c;
    x0.t = __shfl_sync(FULL, s_t, lx); x0.ok = __shfl_sync(FULL, s_ok, lx);
    x1.lo = __shfl_sync(FULL, s_lo, lx + 1) * a.c; x1.hi = __shfl_sync(FULL, s_hi, lx + 1) * a.c;
    x1.t = __shfl_sync(FULL, s_t, lx + 1); x1.ok = __shfl_sync(FULL, s_ok, lx + 1);
    RoiVec<CPL> H0[2], H1[2];
#pragma unroll
    for (int j = 0; j < CPL / 2; ++j) { H0[0].p[j] = H0[1].p[j] = H1[0].p[j] = H1[1].p[j] = make_float2(0.f, 0.f); }
    int tag_top = -1, tag_bot = -1, parity = 0;               // parity 0: H0 plays "top", H1 "bottom"
    for (int py = 0; py < oh; ++py) {
      RoiVec<CPL> best;
#pragma unroll
      for (int j = 0; j < CPL / 2; ++j) best.p[j] = make_float2(-INFINITY, -INFINITY);
#pragma unroll
      for (int sy = 0; sy < 2; ++sy) {
        const int i = 2 * py + sy;
        const int ylo = __shfl_sync(FULL, s_lo, i), yhi = __shfl_sync(FULL, s_hi, i);
        const float ly = __shfl_sync(FULL, s_t, i);
        const int yok = __shfl_sync(FULL, s_ok, i);
        if (!yok) {
#pragma unroll
          for (int j = 0; j < CPL / 2; ++j) { best.p[j].x = fmaxf(best.p[j].x, 0.f); best.p[j].y = fmaxf(best.p[j].y, 0.f); }
          continue;
        }
        bool need_top = false;
        if (ylo != tag_top) {
          if (ylo == tag_bot) { const int t = tag_top; tag_top = tag_bot; tag_bot = t; parity ^= 1; }
          else { need_top = true; tag_top = ylo; }
        }
        const bool need_bot = (yhi != ylo) && (yhi != tag_bot);
        if (need_bot) tag_bot = yhi;
        if (parity == 0) roi_step<CPL>(f, rowstride, ylo, yhi, ly, need_top, need_bot, x0, x1, H0, H1, best);
        else             roi_step<CPL>(f, rowstride, ylo, yhi, ly, need_top, need_bot, x0, x1, H1, H0, best);
      }
#pragma unroll
      for (int j = 0; j < CPL / 2; ++j) { msum.p[j].x += best.p[j].x; msum.p[j].y += best.p[j].y; }
      if (a.ohi && lane_ok) {
        const size_t off = ((size_t)row * ncell + (size_t)py * ow + q) * a.c + c0;
        __half2 vh[CPL / 2], vl[CPL / 2];
#pragma unroll
        for (int j = 0; j < CPL / 2; ++j) split2_f32(best.p[j].x, best.p[j].y, vh[j], vl[j]);
        if (CPL == 8) {
          *reinterpret_cast<uint4*>(a.ohi + off) = *reinterpret_cast<const uint4*>(vh);
          *reinterpret_cast<uint4*>(a.olo + off) = *reinterpret_cast<const uint4*>(vl);
        } else {
          *reinterpret_cast<uint2*>(a.ohi + off) = *reinterpret_cast<const uint2*>(vh);
          *reinterpret_cast<uint2*>(a.olo + off) = *reinterpret_cast<const uint2*>(vl);
        }
      }
    }
  }
  if (a.mhi && lane_ok) {            // fused tf.reduce_mean over the pooled cells (rcnn.py:188)
    __half2 vh[CPL / 2], vl[CPL / 2];
#pragma unroll
    for (int j = 0; j < CPL / 2; ++j)
      split2_f32(__fdiv_rn(msum.p[j].x, (float)ncell), __fdiv_rn(msum.p[j].y, (float)ncell), vh[j], vl[j]);
    const size_t off = (size_t)row * a.c + c0;
    if (CPL == 8) {
      *reinterpret_cast<uint4*>(a.mhi + off) = *reinterpret_cast<const uint4*>(vh);
      *reinterpret_cast<uint4*>(a.mlo + off) = *reinterpret_cast<const uint4*>(vl);
    } else {
      *reinterpret_cast<uint2*>(a.mhi + off) = *reinterpret_cast<const uint2*>(vh);
      *reinterpret_cast<uint2*>(a.mlo + off) = *reinterpret_cast<const uint2*>(vl);
    }
  }
}


// =====================================================================================================================
// Row-walk kernel (round 2, second pass over the design).  A profile of the column-walk kernel above: only
// 28 % of its 1.12 G warp instructions were lerps / maxima / loads -- the rest was the warp-uniform bookkeeping of tap
// sharing (compares, branches, register moves) -- and its L1 hit rate was 6 %: every tap is an L2 hit, so sharing
// taps across samples does not save memory traffic that L1 would not merge anyway.  This kernel drops all
// data-dependent sharing logic:
//  * a sample's right / bottom tap is ALWAYS the next cell (offset +C / +row, or +0 on the last cell): when the
//    coordinate is an exact integer TF uses floor == ceil, but its lerp weight is then 0, so the value is identical;
//  * four sample columns (two pooled columns) per pass instead of two: half the passes over the rows;
//  * the row plan (which sample rows reuse / shift / reload the two resident feature rows) is computed ONCE per warp
//    into a 2-bit-per-row mask instead of being re-derived with compares in every pass;
//  * 3 maxima per pooled cell instead of 4.
// One warp = one ROI x 128 channels (4 per lane, LDG.128), no shared memory, no CTA barriers.
// =====================================================================================================================
template <int NC>
__device__ __forceinline__ void roi_hrow(const float* f, int rowoff, const int (&xo)[NC], const int (&xd)[NC],
                                         const float (&xt)[NC], RoiVec<4> (&H)[NC]) {
  RoiVec<4> l[NC], r[NC];
#pragma unroll
  for (int j = 0; j < NC; ++j) l[j] = roi_load<4>(f, rowoff + xo[j]);
#pragma unroll
  for (int j = 0; j < NC; ++j) r[j] = roi_load<4>(f, rowoff + xo[j] + xd[j]);
#pragma unroll
  for (int j = 0; j < NC; ++j) H[j] = roi_lerp<4>(l[j], r[j], xt[j]);
}

__device__ __forceinline__ RoiVec<4> roi_vmax(const RoiVec<4>& a, const RoiVec<4>& b) {
  RoiVec<4> m;
#pragma unroll
  for (int j = 0; j < 2; ++j) { m.p[j].x = fmaxf(a.p[j].x, b.p[j].x); m.p[j].y = fmaxf(a.p[j].y, b.p[j].y); }
  return m;
}

// One pass: sample columns [col0, col0 + NC) of the crop, all sample rows.  s_* are the lane-resident sample tables
// (lane i < crop_h: y sample i; lane crop_h + j: x sample j): off = element offset of the low tap (row * fw*C or
// col * C), dlt = distance to the high tap (one row / one pixel, 0 on the last cell), t = lerp weight, ok = inside.
template <int NC>
__device__ __forceinline__ void roi_rows_pass(const float* f, const RoiArgs& a, int col0, int s_off, int s_dlt, float s_t,
                                              int s_ok, unsigned plan, int row, int c0, bool lane_ok, RoiVec<4>& msum) {
  constexpr unsigned FULL = 0xffffffffu;
  const int oh = a.crop_h >> 1, ow = a.crop_w >> 1;
  int xo[NC], xd[NC], xk[NC];
  float xt[NC];
#pragma unroll
  for (int j = 0; j < NC; ++j) {
    const int ln = a.crop_h + col0 + j;
    xo[j] = __shfl_sync(FULL, s_off, ln); xd[j] = __shfl_sync(FULL, s_dlt, ln);
    xt[j] = __shfl_sync(FULL, s_t, ln); xk[j] = __shfl_sync(FULL, s_ok, ln);
  }
  // H0 / H1 hold the two resident feature rows; `parity` says which one currently plays "top".  A one-row advance
  // (the common case: the crop's row step is below one cell for ROIs under 14 cells tall) flips the parity and
  // overwrites the old top with the new bottom -- no register copies.
  RoiVec<4> H0[NC], H1[NC], best[NC / 2];
#pragma unroll
  for (int j = 0; j < NC; ++j)
#pragma unroll
    for (int k = 0; k < 2; ++k) H0[j].p[k] = H1[j].p[k] = make_float2(0.f, 0.f);
  int parity = 0;
  for (int py = 0; py < oh; ++py) {
#pragma unroll
    for (int sy = 0; sy < 2; ++sy) {
      const int i = 2 * py + sy;
      const unsigned act = (plan >> (2 * i)) & 3u;                  // 0 reuse, 1 advance one row, 2 load both, 3 outside
      const int yo = __shfl_sync(FULL, s_off, i), yd = __shfl_sync(FULL, s_dlt, i);
      const float ly = __shfl_sync(FULL, s_t, i);
      if (act == 1u) parity ^= 1;
      auto step = [&](RoiVec<4> (&T)[NC], RoiVec<4> (&B)[NC]) {
        if (act == 1u) {
          roi_hrow<NC>(f, yo + yd, xo, xd, xt, B);
        } else if (act == 2u) {
          roi_hrow<NC>(f, yo, xo, xd, xt, T);
          roi_hrow<NC>(f, yo + yd, xo, xd, xt, B);
        }
        RoiVec<4> v[NC];
#pragma unroll
        for (int j = 0; j < NC; ++j) {
          if (act != 3u && xk[j]) v[j] = roi_lerp<4>(T[j], B[j], ly);
          else { v[j].p[0] = make_float2(0.f, 0.f); v[j].p[1] = make_float2(0.f, 0.f); }    // extrapolation_value = 0
        }
#pragma unroll
        for (int m = 0; m < NC / 2; ++m) {
          const RoiVec<4> mh = roi_vmax(v[2 * m], v[2 * m + 1]);
          best[m] = sy == 0 ? mh : roi_vmax(best[m], mh);
        }
      };
      if (parity == 0) step(H0, H1); else step(H1, H0);
    }
#pragma unroll
    for (int m = 0; m < NC / 2; ++m) {
#pragma unroll
      for (int k = 0; k < 2; ++k) { msum.p[k].x += best[m].p[k].x; msum.p[k].y += best[m].p[k].y; }
      if (a.ohi && lane_ok) {
        const int q = (col0 >> 1) + m;
        const size_t off = ((size_t)row * (oh * ow) + (size_t)py * ow + q) * a.c + c0;
        __half2 vh[2], vl[2];
#pragma unroll
        for (int k = 0; k < 2; ++k) split2_f32(best[m].p[k].x, best[m].p[k].y, vh[k], vl[k]);
        *reinterpret_cast<uint2*>(a.ohi + off) = *reinterpret_cast<const uint2*>(vh);
        *reinterpret_cast<uint2*>(a.olo + off) = *reinterpret_cast<const uint2*>(vl);
      }
    }
  }
}

template <int WARPS, int MINB>
__global__ void __launch_bounds__(32 * WARPS, MINB) roi_pool_rows_kernel(const RoiArgs a) {
  constexpr int CPL = 4, SLICE = 32 * CPL;
  constexpr unsigned FULL = 0xffffffffu;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x;                                   // global roi row = img * rmax + r
  const int slice = blockIdx.y * WARPS + warp;
  if (slice * SLICE >= a.c) return;                             // whole warp
  const int c0 = slice * SLICE + lane * CPL;
  const bool lane_ok = c0 < a.c;
  const int img = row / a.rmax, r = row - img * a.rmax;
  const int oh = a.crop_h >> 1, ow = a.crop_w >> 1;
  const int ncell = oh * ow;
  const bool live = (a.counts == nullptr || r < a.counts[img]);
  if (!live) {                                                  // padded row: zeros (the heads read every row)
    if (lane_ok) {
      const uint2 z = make_uint2(0u, 0u);
      if (a.ohi)
        for (int cell = 0; cell < ncell; ++cell) {
          const size_t off = ((size_t)row * ncell + cell) * a.c + c0;
          *reinterpret_cast<uint2*>(a.ohi + off) = z; *reinterpret_cast<uint2*>(a.olo + off) = z;
        }
      if (a.mhi) {
        *reinterpret_cast<uint2*>(a.mhi + (size_t)row * a.c + c0) = z;
        *reinterpret_cast<uint2*>(a.mlo + (size_t)row * a.c + c0) = z;
      }
    }
    return;
  }
  // ---- sample tables (TF crop_and_resize arithmetic in the reference's operation order, quirk Q3)
  const int rowstride = a.fw * a.c;
  int s_off = 0, s_dlt = 0, s_ok = 0, s_cell = 0;
  float s_t = 0.f;
  if (lane < a.crop_h + a.crop_w) {
    const bool is_y = lane < a.crop_h;
    const int k = is_y ? lane : lane - a.crop_h;
    const float* rb = a.rois + (size_t)row * 4;
    float im; int D;
    roi_geometry(a, img, is_y, im, D);
    const float lo_n = __fdiv_rn(is_y ? rb[1] : rb[0], im);
    const float hi_n = __fdiv_rn(is_y ? rb[3] : rb[2], im);
    const int crop = is_y ? a.crop_h : a.crop_w;
    const float Dm1 = (float)(D - 1);
    const float step = crop > 1 ? __fdiv_rn(__fmul_rn(__fsub_rn(hi_n, lo_n), Dm1), (float)(crop - 1)) : 0.f;
    const float in = crop > 1 ? __fadd_rn(__fmul_rn(lo_n, Dm1), __fmul_rn((float)k, step))
                              : __fmul_rn(__fmul_rn(0.5f, __fadd_rn(lo_n, hi_n)), Dm1);
    s_ok = !(in < 0.f || in > Dm1);
    s_cell = s_ok ? (int)floorf(in) : 0;
    s_t = __fsub_rn(in, (float)s_cell);            // == 0 exactly when in is an integer: the high tap's value is unused
    const int unit = is_y ? rowstride : a.c;
    s_off = s_cell * unit;
    s_dlt = (s_cell < D - 1) ? unit : 0;
  }
  // ---- row plan, once per warp: which of the two resident feature rows each sample row can reuse
  unsigned plan = 0u;
  {
    int cur_top = -1, cur_bot = -1;
    for (int i = 0; i < a.crop_h; ++i) {
      const int cell = __shfl_sync(FULL, s_cell, i), ok = __shfl_sync(FULL, s_ok, i), dl = __shfl_sync(FULL, s_dlt, i);
      unsigned act;
      if (!ok) act = 3u;
      else {
        const int lo = cell, hi = cell + (dl != 0);
        if (lo == cur_top && hi == cur_bot) act = 0u;
        else if (lo == cur_bot && cur_bot != cur_top) { act = 1u; cur_top = lo; cur_bot = hi; }
        else { act = 2u; cur_top = lo; cur_bot = hi; }
      }
      plan |= act << (2 * i);
    }
  }
  const float* f = a.fmap + (size_t)img * a.fh * a.fw * a.c + (lane_ok ? c0 : 0);
  asm volatile("" : "+l"(f));     // keep ONE per-lane base pointer: every tap address is then base + 32-bit offset
  RoiVec<4> msum;
  msum.p[0] = msum.p[1] = make_float2(0.f, 0.f);
  int col0 = 0;
  for (; col0 + 4 <= a.crop_w; col0 += 4) roi_rows_pass<4>(f, a, col0, s_off, s_dlt, s_t, s_ok, plan, row, c0, lane_ok, msum);
  if (col0 < a.crop_w) roi_rows_pass<2>(f, a, col0, s_off, s_dlt, s_t, s_ok, plan, row, c0, lane_ok, msum);
  if (a.mhi && lane_ok) {            // fused tf.reduce_mean over the pooled cells (rcnn.py:188)
    __half2 vh[2], vl[2];
#pragma unroll
    for (int k = 0; k < 2; ++k)
      split2_f32(__fdiv_rn(msum.p[k].x, (float)ncell), __fdiv_rn(msum.p[k].y, (float)ncell), vh[k], vl[k]);
    const size_t off = (size_t)row * a.c + c0;
    *reinterpret_cast<uint2*>(a.mhi + off) = *reinterpret_cast<const uint2*>(vh);
    *reinterpret_cast<uint2*>(a.mlo + off) = *reinterpret_cast<const uint2*>(vl);
  }
}

// Shape preconditions of each instance (crop_h = 2*pw, crop_w = 2*ph, both even): the row-walk kernel keeps the
// crop_h + crop_w sample tables in the lanes of one warp and a 2-bit plan per sample row in 32 bits; the column-walk
// kernel keeps the tables in the lanes; the cell kernel keeps RB tables of up to 64 samples in shared memory and fills
// them with one thread per sample.
static bool roi_kernel_fits(int k, int c, int ph, int pw) {
  if (c % 8 != 0 || ph < 1 || pw < 1 || 2 * (ph + pw) > 64) return false;
  const int crop_h = 2 * pw, nsamp = 2 * (ph + pw);
  switch (k) {
    case ROI_ROWS_MINB6: case ROI_ROWS_MINB5: case ROI_ROWS_MINB4: return crop_h <= 16 && nsamp <= 32;
    case ROI_COLS_CPL4: case ROI_COLS_CPL8: return nsamp <= 32;
    case ROI_CELLS_8_4_4: return 4 * nsamp <= 128;
    case ROI_CELLS_8_4_8: return 4 * nsamp <= 256;
    case ROI_CELLS_8_1_8: case ROI_CELLS_4_1_8: return true;
    default: return false;
  }
}

int roi_kernel(int c, int ph, int pw) {
  if (!roi_kernel_fits(ROI_CELLS_8_1_8, c, ph, pw)) return -1;
  // LUMI_ROI_KERNEL: "rows" (default, round-2 row-walk kernel) | "cols" (round-2 first design) | "cells" (round-1 kernel);
  // the older ones are kept for A/B measurement
  static const int variant = [] {
    const char* e = getenv("LUMI_ROI_KERNEL");
    if (e && e[0] == 'c' && e[1] == 'e') return 0;
    if (e && e[0] == 'c' && e[1] == 'o') return 1;
    return 2;
  }();
  // occupancy: 4 / 5 / 6 resident CTAs per SM (<= 128 / 102 / 80 registers) measured 1.308 / 1.269 / 1.241 ms per step: 6
  static const int minb = [] { const char* e = getenv("LUMI_ROI_MINB"); const int v = e ? atoi(e) : 6; return (v == 4 || v == 5) ? v : 6; }();
  if (variant == 2 && roi_kernel_fits(ROI_ROWS_MINB6, c, ph, pw))
    return minb == 5 ? ROI_ROWS_MINB5 : minb == 4 ? ROI_ROWS_MINB4 : ROI_ROWS_MINB6;
  static const int cols_cpl = [] { const char* e = getenv("LUMI_ROI_COLS_CPL"); return (e && atoi(e) == 8) ? 8 : 4; }();
  if (variant == 1 && roi_kernel_fits(ROI_COLS_CPL4, c, ph, pw)) return cols_cpl == 8 ? ROI_COLS_CPL8 : ROI_COLS_CPL4;
  static const int cpl = [] { const char* e = getenv("LUMI_ROI_CPL"); return (e && atoi(e) == 4) ? 4 : 8; }();
  // (measured alternatives at R = 2000, batch 8: 4 channels/lane 3.1 ms, straight-line 16-tap loads
  //  without sharing 3.0 ms, this kernel 2.7 ms)
  static const int rb = [] { const char* e = getenv("LUMI_ROI_RB"); return (e && atoi(e) == 1) ? 1 : 4; }();
  // 4 warps x 4 ROIs: 196 cells = 49 per warp, no tail at all (measured 2.49 vs 2.51 ms with 8 warps, 2.73 ms with
  // one ROI per CTA)
  static const int nw = [] { const char* e = getenv("LUMI_ROI_NW"); return (e && atoi(e) == 8) ? 8 : 4; }();
  if (cpl == 4) return ROI_CELLS_4_1_8;  // 4 channels per lane: half the registers (measured slower: 3.1 vs 2.7 ms at R = 2000)
  if (rb == 4 && nw == 4 && roi_kernel_fits(ROI_CELLS_8_4_4, c, ph, pw)) return ROI_CELLS_8_4_4;
  if (rb == 4 && roi_kernel_fits(ROI_CELLS_8_4_8, c, ph, pw)) return ROI_CELLS_8_4_8;
  return ROI_CELLS_8_1_8;
}

void launch_roi_pool(const float* fmap_f32, int n, int fh, int fw, int c, const float* rois, const int* counts, int rmax,
                     float im_h, float im_w, int ph, int pw, Act out, Act mean, cudaStream_t st, int kernel,
                     const ResizeSrc* tab, int feat_stride) {
  LUMI_REQUIRE(c % 8 == 0, "roi_pool: C must be a multiple of 8");
  LUMI_REQUIRE(ph >= 1 && pw >= 1 && 2 * (ph + pw) <= 64, "roi_pool: pooled size must be >= 1 with 2 * (ph + pw) <= 64");
  LUMI_REQUIRE(kernel >= -1 && kernel < ROI_KERNEL_COUNT, "roi_pool: kernel must be -1 or one of the codes 0-8");
  const int k = kernel < 0 ? roi_kernel(c, ph, pw) : kernel;
  LUMI_REQUIRE(roi_kernel_fits(k, c, ph, pw), "roi_pool: kernel " + std::to_string(k) + " does not take C = " +
                                                  std::to_string(c) + " at " + std::to_string(ph) + " x " +
                                                  std::to_string(pw));
  RoiArgs a;
  a.fmap = fmap_f32; a.n = n; a.fh = fh; a.fw = fw; a.c = c;
  a.rois = rois; a.counts = counts; a.rmax = rmax; a.im_h = im_h; a.im_w = im_w;
  LUMI_REQUIRE(!tab || feat_stride > 0, "roi_pool: a packed batch needs the feature stride");
  a.tab = tab; a.feat_stride = feat_stride;
  a.crop_h = pw * 2; a.crop_w = ph * 2;      // roi_pool.py:77 passes [pooled_width*2, pooled_height*2]
  a.ohi = out.hi; a.olo = out.lo;
  a.mhi = mean.hi; a.mlo = mean.lo;
  LUMI_REQUIRE(out.hi || mean.hi, "roi_pool: no output requested");
  long rows = (long)n * rmax;
  if (!rows) return;
  constexpr int W = 4;
  switch (k) {
    case ROI_ROWS_MINB6: case ROI_ROWS_MINB5: case ROI_ROWS_MINB4: {
      dim3 grid((unsigned)rows, (unsigned)cdiv(c, 128 * W));
      if (k == ROI_ROWS_MINB5) roi_pool_rows_kernel<W, 5><<<grid, 32 * W, 0, st>>>(a);
      else if (k == ROI_ROWS_MINB4) roi_pool_rows_kernel<W, 4><<<grid, 32 * W, 0, st>>>(a);
      else roi_pool_rows_kernel<W, 6><<<grid, 32 * W, 0, st>>>(a);
      break;
    }
    case ROI_COLS_CPL8: {
      dim3 grid((unsigned)rows, (unsigned)cdiv(c, 256 * W));
      roi_pool_cols_kernel<8, W><<<grid, 32 * W, 0, st>>>(a);
      break;
    }
    case ROI_COLS_CPL4: {
      dim3 grid((unsigned)rows, (unsigned)cdiv(c, 128 * W));
      roi_pool_cols_kernel<4, W><<<grid, 32 * W, 0, st>>>(a);
      break;
    }
    case ROI_CELLS_8_4_4: {
      dim3 grid((unsigned)cdiv64(rows, 4), (unsigned)cdiv(c, 256));
      roi_pool_kernel<8, 4, 4><<<grid, 128, 0, st>>>(a);
      break;
    }
    case ROI_CELLS_8_4_8: {
      dim3 grid((unsigned)cdiv64(rows, 4), (unsigned)cdiv(c, 256));
      roi_pool_kernel<8, 4, 8><<<grid, 256, 0, st>>>(a);
      break;
    }
    case ROI_CELLS_8_1_8: {
      dim3 grid((unsigned)rows, (unsigned)cdiv(c, 256));
      roi_pool_kernel<8, 1, 8><<<grid, 256, 0, st>>>(a);
      break;
    }
    default: {
      dim3 grid((unsigned)rows, (unsigned)cdiv(c, 128));
      roi_pool_kernel<4, 1, 8><<<grid, 256, 0, st>>>(a);
      break;
    }
  }
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
}

}  // namespace lumi
