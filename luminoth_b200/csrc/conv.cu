// Convolution kernels of the backbone / RPN / head stack.
//
//  * conv_simt_kernel : fp32 implicit GEMM on CUDA cores. Handles every shape
//    (C_in = 3 stem, stride 2, FC layers); also the on-GPU cross-check of the
//    tensor-core kernel.
//  * conv_tc_kernel   : wgmma (sm_90a) implicit GEMM, stride 1 or 2, C_in % 64 == 0.
//    Activations and weights are fp16 (hi, lo) split planes; each K=16 slice
//    issues three wgmma  Ahi*Bhi + Ahi*Blo + Alo*Bhi  into fp32 register
//    accumulators that are folded into an fp32 running sum once per 64-deep
//    K slice (fp32-class accuracy, DESIGN section 3).  im2col is fused: a TMA
//    producer thread issues one 4-D box {64 ch, tw, th, nb} per filter tap at
//    shifted (possibly negative) coordinates; out-of-bounds elements are
//    zero-filled by TMA, which IS the TF SAME zero padding.  Persistent CTAs
//    (whole tiles or stream-K) of one producer and two or four consumer
//    warpgroups, mbarrier operand ring; split-plane outputs leave through shared-memory
//    epilogue slots (TMA residual prefetch, TMA stores).  Variants: 128 x 256 tiles for the
//    long-K layers with C_out >= 256, 2-CTA clusters that multicast the weight tile, and halo-patch kernels for 3x3
//    layers.
//
// Replaces slim conv2d+batch_norm+relu (luminoth/models/base/base_network.py:143-151),
// snt.Conv2D (models/fasterrcnn/rpn.py:69-90, models/ssd/ssd.py:83-96,
// models/ssd/feature_extractor.py:28-37) and snt.Linear (models/fasterrcnn/rcnn.py:74-98).
#include "conv.cuh"
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <tuple>

namespace lumi {

thread_local int g_launch_count = 0;

// =====================================================================================
// SIMT fp32 implicit GEMM
// =====================================================================================
struct SimtArgs {
  const __half* in_hi; const __half* in_lo;
  int n, h, w, cin;
  const float* wgt; const float* scale; const float* bias;
  int kh, kw, stride, rate, pad_t, pad_l, ho, wo, cout, act;
  __half* out_hi; __half* out_lo; float* out_f32;
  const __half* res_hi; const __half* res_lo; int res_h, res_w, res_stride;
  int* overflow;
  const float* pre_scale; const float* pre_bias; __half* pre_hi; __half* pre_lo;   // PRE: see ConvIO::pre
};

constexpr int SM_BM = 128, SM_BN = 64, SM_BK = 16;

// PRE: the layer also writes the pre-activation output p (out_hi == nullptr: p only)
template <bool PRE>
__global__ void __launch_bounds__(256) conv_simt_kernel(const SimtArgs a) {
  __shared__ float As[SM_BK][SM_BM + 4];
  __shared__ float Bs[SM_BK][SM_BN + 4];
  const int tid = threadIdx.x;
  const int M = a.n * a.ho * a.wo;
  const int K = a.kh * a.kw * a.cin;
  const int m0 = blockIdx.x * SM_BM, n0 = blockIdx.y * SM_BN;

  // A loader coordinates: one output pixel row, 8 consecutive k
  const int arow = tid >> 1, akseg = (tid & 1) * 8;
  const int am = m0 + arow;
  const bool am_ok = am < M;
  int a_n = 0, a_oy = 0, a_ox = 0;
  if (am_ok) { a_n = am / (a.ho * a.wo); int r = am % (a.ho * a.wo); a_oy = r / a.wo; a_ox = r % a.wo; }
  const bool vec_a = (a.cin % 8) == 0;
  // B loader coordinates
  const int bkk = tid >> 4, bnn = (tid & 15) * 4;

  const int ty = tid >> 4, tx = tid & 15;
  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < K; k0 += SM_BK) {
    // ---- A tile
    float av[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) av[j] = 0.f;
    const int kbase = k0 + akseg;
    if (am_ok && kbase < K) {
      if (vec_a) {
        int tap = kbase / a.cin, c = kbase % a.cin;
        int r = tap / a.kw, s = tap % a.kw;
        int iy = a_oy * a.stride + r * a.rate - a.pad_t, ix = a_ox * a.stride + s * a.rate - a.pad_l;
        if (iy >= 0 && iy < a.h && ix >= 0 && ix < a.w) {
          size_t off = (((size_t)a_n * a.h + iy) * a.w + ix) * a.cin + c;
          uint4 vh = *reinterpret_cast<const uint4*>(a.in_hi + off);
          uint4 vl = *reinterpret_cast<const uint4*>(a.in_lo + off);
          const __half* ph = reinterpret_cast<const __half*>(&vh);
          const __half* pl = reinterpret_cast<const __half*>(&vl);
#pragma unroll
          for (int j = 0; j < 8; ++j) av[j] = join_f16(ph[j], pl[j]);
        }
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          int k = kbase + j;
          if (k < K) {
            int tap = k / a.cin, c = k % a.cin;
            int r = tap / a.kw, s = tap % a.kw;
            int iy = a_oy * a.stride + r * a.rate - a.pad_t, ix = a_ox * a.stride + s * a.rate - a.pad_l;
            if (iy >= 0 && iy < a.h && ix >= 0 && ix < a.w) {
              size_t off = (((size_t)a_n * a.h + iy) * a.w + ix) * a.cin + c;
              av[j] = join_f16(a.in_hi[off], a.in_lo[off]);
            }
          }
        }
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) As[akseg + j][arow] = av[j];
    // ---- B tile
    {
      int k = k0 + bkk;
      float bv[4] = {0.f, 0.f, 0.f, 0.f};
      if (k < K) {
        const float* wp = a.wgt + (size_t)k * a.cout + n0 + bnn;
        if ((a.cout % 4) == 0 && n0 + bnn + 3 < a.cout) {
          float4 t = *reinterpret_cast<const float4*>(wp);
          bv[0] = t.x; bv[1] = t.y; bv[2] = t.z; bv[3] = t.w;
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (n0 + bnn + j < a.cout) bv[j] = wp[j];
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) Bs[bkk][bnn + j] = bv[j];
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < SM_BK; ++kk) {
      float ar[8], br[4];
#pragma unroll
      for (int i = 0; i < 8; ++i) ar[i] = As[kk][ty * 8 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) br[j] = Bs[kk][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ar[i], br[j], acc[i][j]);
    }
    __syncthreads();
  }

  // ---- epilogue
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int m = m0 + ty * 8 + i;
    if (m >= M) continue;
    int n_img = m / (a.ho * a.wo);
    int r = m % (a.ho * a.wo);
    int oy = r / a.wo, ox = r % a.wo;
    size_t obase = (size_t)m * a.cout;
    size_t rbase = 0;
    if (a.res_hi)
      rbase = (((size_t)n_img * a.res_h + (size_t)oy * a.res_stride) * a.res_w + (size_t)ox * a.res_stride) * a.cout;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int c = n0 + tx * 4 + j;
      if (c >= a.cout) continue;
      float sc = a.scale ? a.scale[c] : 1.f;
      float bi = a.bias ? a.bias[c] : 0.f;
      float v = fmaf(acc[i][j], sc, bi);
      if (a.res_hi) v += join_f16(a.res_hi[rbase + c], a.res_lo[rbase + c]);
      v = apply_act(v, a.act);
      if (a.out_f32) {
        a.out_f32[obase + c] = v;
      } else {
        if (split_overflows(v) && a.overflow) atomicOr(a.overflow, 1);
        __half hi, lo;
        split_f32(v, hi, lo);
        if (!PRE || a.out_hi) {
          a.out_hi[obase + c] = hi;
          a.out_lo[obase + c] = lo;
        }
        if constexpr (PRE) {
          const float p = fmaxf(fmaf(join_f16(hi, lo), a.pre_scale[c], a.pre_bias[c]), 0.f);
          if (split_overflows(p) && a.overflow) atomicOr(a.overflow, 1);
          split_f32(p, hi, lo);
          a.pre_hi[obase + c] = hi;
          a.pre_lo[obase + c] = lo;
        }
      }
    }
  }
}

void launch_conv_simt(const ConvLayer& L, const ConvIO& io, cudaStream_t st) {
  SimtArgs a;
  a.in_hi = io.in.hi; a.in_lo = io.in.lo;
  a.n = io.in.n; a.h = io.in.h; a.w = io.in.w; a.cin = io.in.c;
  LUMI_REQUIRE(io.in.c == L.cin, "conv_simt: channel mismatch");
  a.wgt = L.w_f32; a.scale = L.scale; a.bias = L.bias;
  a.kh = L.kh; a.kw = L.kw; a.stride = L.stride; a.rate = L.rate;
  a.pad_t = io.pad_t; a.pad_l = io.pad_l; a.ho = io.ho; a.wo = io.wo; a.cout = L.cout; a.act = L.act;
  a.out_hi = io.out.hi; a.out_lo = io.out.lo; a.out_f32 = io.out_f32;
  a.res_hi = io.res.hi; a.res_lo = io.res.lo; a.res_h = io.res.h; a.res_w = io.res.w; a.res_stride = io.res_stride;
  a.overflow = io.overflow_flag;
  a.pre_scale = io.pre_scale; a.pre_bias = io.pre_bias; a.pre_hi = io.pre.hi; a.pre_lo = io.pre.lo;
  LUMI_REQUIRE(!io.pre.hi || (!io.out_f32 && io.pre_scale && io.pre_bias), "conv_simt: bad pre-activation output");
  long M = (long)a.n * a.ho * a.wo;
  if (M == 0) return;
  dim3 grid((unsigned)cdiv64(M, SM_BM), (unsigned)cdiv(L.cout, SM_BN));
  if (io.pre.hi) conv_simt_kernel<true><<<grid, 256, 0, st>>>(a);
  else conv_simt_kernel<false><<<grid, 256, 0, st>>>(a);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
}

// =====================================================================================
// wgmma implicit GEMM (fp16x2 split operands, fp32 register accumulators)
// =====================================================================================
struct TcArgs {
  CUtensorMap tm_a_hi, tm_a_lo, tm_b_hi, tm_b_lo;
  // slot epilogue (SLOTS > 0): output and residual planes as boxes {64 ch, tw, th, nb} (residual with the traversal
  // stride res_stride)
  CUtensorMap tm_o_hi, tm_o_lo, tm_r_hi, tm_r_lo;
  // PRE: the pre-activation planes (ConvIO::pre) as store boxes; with p only (out_hi == nullptr) tm_o_* describe them
  CUtensorMap tm_p_hi, tm_p_lo;
  const float* pre_scale; const float* pre_bias;
  __half* pre_hi; __half* pre_lo;
  const float* scale; const float* bias;
  __half* out_hi; __half* out_lo; float* out_f32;
  const __half* res_hi; const __half* res_lo;
  int res_h, res_w, res_stride;
  int n, ho, wo, cin, cout;
  int kh, kw, rate, pad_t, pad_l, act;
  int nb, th, tw;                  // M tile = nb images x th rows x tw cols (<= 128 pixels)
  int tiles_w, tiles_h, tiles_n;   // M tiles per row / column / image groups
  int n_tiles;                     // C_out tiles (cout_pad / BN)
  int stride;                      // TMA traversal stride of the activation map (1 or 2)
  int* overflow;
  // stream-K (sk_mode != 0): the K loops of all tiles form one unit sequence that is cut into gridDim.x equal
  // contiguous ranges; a CTA that starts in the middle of a tile writes its partial accumulators to
  // sk_partials[blockIdx.x] and publishes sk_flags[blockIdx.x] = sk_epoch, the CTA holding the tile's first
  // K iteration adds them (in CTA order -- deterministic) and runs the epilogue.
  int sk_mode;
  float* sk_partials;              // [gridDim.x][BN columns][128 rows] fp32
  int* sk_flags;                   // [gridDim.x]
  int sk_epoch;
};

// One unit of work of a persistent CTA: K iterations [k0, k1) of output tile `tile`.
struct TcItem { int tile, k0, k1; };
struct TcSched {
  int mode, total_tiles, n_iters, t, bid, nblk;
  long long u, u_end;
  __device__ TcSched(int mode_, int total_tiles_, int n_iters_, int bid_, int nblk_)
      : mode(mode_), total_tiles(total_tiles_), n_iters(n_iters_), bid(bid_), nblk(nblk_) {
    t = bid;
    const long long U = (long long)total_tiles * n_iters;
    u = U * bid / nblk;
    u_end = U * (bid + 1) / nblk;
  }
  __device__ static long long range_end(int unit, int total_tiles, int n_iters, int nblk_) {
    return (long long)total_tiles * n_iters * (unit + 1) / nblk_;
  }
  __device__ bool next(TcItem& it) {
    if (!mode) {                   // round robin over whole tiles
      if (t >= total_tiles) return false;
      it.tile = t; it.k0 = 0; it.k1 = n_iters;
      t += nblk;
      return true;
    }
    if (u >= u_end) return false;
    it.tile = (int)(u / n_iters);
    it.k0 = (int)(u - (long long)it.tile * n_iters);
    const long long rem = u_end - u;
    it.k1 = (rem < (long long)(n_iters - it.k0)) ? it.k0 + (int)rem : n_iters;
    u += it.k1 - it.k0;
    return true;
  }
};

constexpr int TC_A_BYTES = 128 * 128;       // 128 pixel rows x 64 fp16 (one 128 B swizzle row each)
constexpr int TC_BN_MAX = 256;              // widest N tile: sizes the stream-K partial-sum slots
// HALO (3x3, stride 1, rate 1): the nine taps of a 64-channel slice read the SAME input pixels, shifted.  The HALO
// kernels fetch the (th + 2) x (8 + 2)-pixel patch of the slice ONCE (one TMA box per patch row and plane, zero-filled
// outside the image = SAME padding) and hand the tensor core nine shifted VIEWS of it: M tile = th rows x 8 pixels,
// 8-row group g = image row g, so a view is the K-major SWIZZLE_128B matrix that starts at patch pixel (r, s) with a
// group stride of one patch row.  The tensor core applies the 128 B swizzle to the absolute shared-memory address,
// as TMA does when it writes the patch, so a view may start at any 128 B row; patch rows sit 2048 B apart so that every
// row starts at the same phase of the pattern.  Only the weights stream per tap.
constexpr int TC_HALO_TW = 8;                              // tile width: one 8-row group per image row
constexpr int TC_HALO_PITCH = 2048;                        // bytes per patch row (10 pixels x 128 B, padded)
constexpr int TC_HALO_ROWS = 16 + 2;                       // th <= 16
constexpr int TC_HALO_PLANE_BYTES = TC_HALO_ROWS * TC_HALO_PITCH;

// NCWG consumer warpgroups: 2 (each 64 rows x BN columns) or 4 (64 rows x BN / 2 columns each; sixteen epilogue warps
// with half the accumulator registers each, for the short-K layers whose time is mostly epilogue).
// PAIR: a 2-CTA cluster shares one N tile between two M tiles; each CTA loads HALF of the weight tile and multicasts
// it into both CTAs' shared memory, halving the weight traffic from L2.
// SLOTS > 0: split-plane outputs leave through a ring of SLOTS epilogue slots (one 64-column group of the tile, hi and
// lo plane, in the SWIZZLE_128B layout of a box {64 ch, tw, th, nb}): the producer prefetches the residual into the
// slot, the consumers overwrite it with the result in place and one thread TMA-stores it.  0: register epilogue.
// BN = 256 (wide tile): two consumer warpgroups of 64 rows x 256 columns, slot epilogue; see conv_tc_kernel.
template <int BN, int STAGES, int NCWG = 2, bool PAIR = false, bool HALO = false, int SLOTS = 0>
struct TcCfg {
  static_assert(NCWG == 2 || NCWG == 4, "two or four consumer warpgroups");
  static_assert(!PAIR || BN == 128, "the cluster pair exists for BN = 128");
  static_assert(BN != 256 || (NCWG == 2 && !HALO && SLOTS > 0), "the wide tile: generic kernel, two consumers, slots");
  static constexpr int WN = BN * 2 / NCWG;                         // columns per consumer warpgroup
  static_assert(SLOTS == 0 || (!PAIR && !HALO && WN % 64 == 0), "slot epilogue: generic kernel, whole column groups");
  // four warpgroups: each column group's pair waits only on its own groups' slot phases, so every slot must carry
  // the same column group (a waiter two phases behind would read the other parity as complete)
  static_assert(NCWG == 2 || SLOTS % 2 == 0, "four warpgroups: an even slot count");
  static constexpr int B_BYTES = BN * 128;                         // BN weight rows x 64 fp16
  static constexpr int A_STAGE_BYTES = HALO ? 0 : 2 * TC_A_BYTES;  // HALO: A lives in the patch buffers
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + 2 * B_BYTES;  // A hi, A lo, B hi, B lo
  static constexpr int PATCH_BYTES = HALO ? 2 * TC_HALO_PLANE_BYTES : 0;   // one patch buffer: hi + lo plane
  static constexpr int SLOT_BYTES = 2 * TC_A_BYTES;                // 128 rows x 64 fp16, hi + lo plane
  static constexpr int SMEM_BYTES = 2 * PATCH_BYTES + STAGES * STAGE_BYTES + SLOTS * SLOT_BYTES + 1024 /*align slack*/ +
                                    256 /*barriers*/;
  static_assert(SMEM_BYTES <= 232448, "shared memory per CTA");
  static constexpr int THREADS = (1 + NCWG) * 128;   // warpgroup 0: TMA producer (one thread), then the consumers
  // register split: the producer warpgroup keeps the minimum and hands the rest to the consumers.  setmaxnreg.inc
  // can only take what the CTA's own warpgroups released, so the total stays within the launch allocation (the
  // per-thread count __launch_bounds__ allows, rounded down to a multiple of 8, times THREADS)
  static constexpr int LAUNCH_REGS = (65536 / THREADS) / 8 * 8;
  static constexpr int PRODUCER_REGS = NCWG == 2 ? 40 : 24;
  static constexpr int CONSUMER_REGS = NCWG == 2 ? 232 : 112;
  static_assert(128 * (PRODUCER_REGS + NCWG * CONSUMER_REGS) <= THREADS * LAUNCH_REGS, "register budget of the CTA");
};

// Operand descriptors of one K slice, with the ring stage and (HALO) patch buffer it occupies.
struct TcSlice { uint64_t ahi, alo, bhi, blo; uint32_t st, pb; };

// The 12 wgmma of one 64-deep K slice into a fresh accumulator tile d, committed as one group.  The 2^-11-times-smaller
// cross terms come first, the hi*hi products last: each MMA's addition into the chain can cost up to one ulp of the
// value held, so only the last four additions act on the full-size partial sum.
template <int WN>
__device__ __forceinline__ void tc_slice_mma(float (&d)[WN / 2], const TcSlice& s) {
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    const uint64_t ko = (uint64_t)(kk * 2);           // 16 fp16 = 32 B = 2 x 16 B descriptor units
    if constexpr (WN == 128) {
      wgmma_m64n128k16_f16(d, s.ahi + ko, s.blo + ko, kk > 0 ? 1u : 0u);
      wgmma_m64n128k16_f16(d, s.alo + ko, s.bhi + ko, 1u);
    } else {
      wgmma_m64n64k16_f16(d, s.ahi + ko, s.blo + ko, kk > 0 ? 1u : 0u);
      wgmma_m64n64k16_f16(d, s.alo + ko, s.bhi + ko, 1u);
    }
  }
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    const uint64_t ko = (uint64_t)(kk * 2);
    if constexpr (WN == 128) wgmma_m64n128k16_f16(d, s.ahi + ko, s.bhi + ko, 1u);
    else wgmma_m64n64k16_f16(d, s.ahi + ko, s.bhi + ko, 1u);
  }
  wgmma_commit();
}

// The pre-activation output of a column pair, in place: (h2, l2) holding x as split become p = relu(fmaf(x^, s, b)) as
// split.  Returns whether p leaves the split range.
__device__ __forceinline__ bool tc_preact(__half2& h2, __half2& l2, const float* s, const float* b, int c0) {
  const float2 sc = __ldg(reinterpret_cast<const float2*>(s + c0));
  const float2 bi = __ldg(reinterpret_cast<const float2*>(b + c0));
  const float p0 = fmaxf(fmaf(__low2float(h2) + __low2float(l2), sc.x, bi.x), 0.f);
  const float p1 = fmaxf(fmaf(__high2float(h2) + __high2float(l2), sc.y, bi.y), 0.f);
  split2_f32(p0, p1, h2, l2);
  return split_overflows(p0) || split_overflows(p1);
}

// Persistent: grid = min(#tiles, #SMs) (or #SMs for stream-K); every CTA (or CTA pair) walks its schedule.  One
// producer thread keeps a ring of STAGES (tap, 64-channel) K slices in flight with TMA: im2col is fused -- one 4-D box
// {64 ch, tw, th, nb} per filter tap at shifted (possibly negative) coordinates, zero-filled outside the map, which IS
// the TF SAME zero padding.  Per K slice each consumer warpgroup issues, for each K = 16 step, the three products
// Ahi*Blo + Alo*Bhi + Ahi*Bhi  into a fresh fp32 register tile (the lo*lo term is below fp32 resolution) and adds the
// tile into the running fp32 sum with round-to-nearest adds once the tensor core is done with it: the tensor core's
// own accumulation chain never spans more than one 64-deep slice, which keeps fp32-class accuracy at K = 9216
// (DESIGN section 3).
// PIPE: two slice tiles d0 / d1 alternate, so slice k + 1's wgmma run while slice k is waited for, released and
// folded; without it every slice drains the warpgroup's wgmma queue before the fold.  Both orders fold the same tiles
// in ascending k, so the results are bit-identical.
// BN = 256 (wide tile, for C_out >= 256 on long K): the A tile of a stage serves twice the columns, a quarter less
// L2 -> shared-memory operand traffic per FLOP than BN = 128.  A 128 x 256 register tile d next to the 128-register
// running sum does not fit, so each slice runs as two 128-column halves: the BN = 128 slice chain on the B descriptors
// of one half into a 64-register d, waited for and folded into that half of the running sum before the next half is
// issued.  Every output element gets the BN = 128 kernel's MMA chain and fold order, so the results are bit-identical.
// Epilogue: scale/bias (folded BN) -> +residual -> relu/relu6 -> fp32 or hi/lo split.
// SLOTS > 0 (split outputs): per 64-column group of a tile, in order, the slot ring carries
//   producer: wait slot empty -> TMA-load the residual boxes (hi, lo) into it, or arrive without bytes;
//   consumers of those columns: wait slot full -> read the residual -> the same arithmetic as the register epilogue ->
//     write hi / lo over it in place -> fence.proxy.async -> named barrier -> one thread TMA-stores both boxes;
//   that thread frees the slot once cp.async.bulk.wait_group.read shows the store has read it.
// TMA zero-fills the out-of-range part of a residual box and clips it on the store, so edge tiles need no masking.
// PRE (split outputs only): the layer also writes the pre-activation output p = relu(fmaf(x^, pre_scale, pre_bias)) of
// ConvIO::pre.  The register epilogue writes its planes next to x's.  The slot epilogue has no room for a second slot
// ring (four consumers: 2 x 64 KB stages + 2 x 32 KB slots already), so p reuses the slot: x is stored, the issuer
// waits until that store has read the slot and releases the column group's warpgroups, each thread rewrites the
// values it wrote with p and a second store follows; the slot is freed after the second store has read it.  With
// p only (out_hi == nullptr) the slot carries p in the first place and one store (through tm_o_*) suffices.
template <int BN, int STAGES, int NCWG, bool PAIR, bool HALO, bool PIPE, int SLOTS, bool PRE>
__global__ void __launch_bounds__(TcCfg<BN, STAGES, NCWG, PAIR, HALO, SLOTS>::THREADS, 1)
conv_tc_kernel(const __grid_constant__ TcArgs a) {
  using Cfg = TcCfg<BN, STAGES, NCWG, PAIR, HALO, SLOTS>;
  static_assert(!PRE || !HALO, "pre-activation outputs: generic and 2-CTA kernels");
  static_assert(BN != 256 || (!PIPE && !PRE), "the wide tile: single-buffered, no pre-activation output");
  constexpr int WN = Cfg::WN;
  constexpr int NR = WN / 2;                          // accumulator registers per thread (64 rows x WN / 128 threads)
  constexpr int NGT = BN / 64;                        // 64-column groups (slots) per tile
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* patch = smem;                              // HALO: [2 buffers][hi, lo][18 rows x 2048 B]
  uint8_t* stages = smem + 2 * Cfg::PATCH_BYTES;
  uint8_t* slots = stages + STAGES * Cfg::STAGE_BYTES;   // [SLOTS][hi, lo][128 rows x 128 B]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(slots + SLOTS * Cfg::SLOT_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* patch_full_bar = empty_bar + STAGES;      // [2]
  uint64_t* patch_empty_bar = patch_full_bar + 2;     // [2]
  uint64_t* slot_full_bar = patch_empty_bar + 2;      // [SLOTS]
  uint64_t* slot_empty_bar = slot_full_bar + SLOTS;   // [SLOTS]

  // PAIR: rank in the cluster; the scheduling unit is the pair, whose CTAs take M tiles 2 m and 2 m + 1 of one N tile
  const int rank = PAIR ? (int)cluster_ctarank() : 0;
  const int sched_id = PAIR ? (int)(blockIdx.x >> 1) : (int)blockIdx.x;
  const int sched_n = PAIR ? (int)(gridDim.x >> 1) : (int)gridDim.x;
  const int wg = threadIdx.x >> 7;
  const int m_tiles = a.tiles_w * a.tiles_h * a.tiles_n;
  const int total_tiles = (PAIR ? (m_tiles + 1) / 2 : m_tiles) * a.n_tiles;
  const int rows_valid = a.nb * a.th * a.tw;
  const int cchunks = a.cin >> 6;
  const int n_iters = a.kh * a.kw * cchunks;

  if (threadIdx.x == 0) {
    // empty: one arrival per consumer warpgroup of every CTA whose shared memory the stage's copies write
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], (PAIR ? 2 : 1) * NCWG); }
    for (int s = 0; s < 2; ++s) { mbar_init(&patch_full_bar[s], 1); mbar_init(&patch_empty_bar[s], NCWG); }
    for (int s = 0; s < SLOTS; ++s) { mbar_init(&slot_full_bar[s], 1); mbar_init(&slot_empty_bar[s], 1); }
    fence_mbar_init();
    tma_prefetch_desc(&a.tm_a_hi); tma_prefetch_desc(&a.tm_a_lo);
    tma_prefetch_desc(&a.tm_b_hi); tma_prefetch_desc(&a.tm_b_lo);
    if (SLOTS) {
      tma_prefetch_desc(&a.tm_o_hi); tma_prefetch_desc(&a.tm_o_lo);
      if (a.res_hi) { tma_prefetch_desc(&a.tm_r_hi); tma_prefetch_desc(&a.tm_r_lo); }
      if (PRE && a.out_hi) { tma_prefetch_desc(&a.tm_p_hi); tma_prefetch_desc(&a.tm_p_lo); }
    }
  }
  if (PAIR) cluster_sync_all();        // both CTAs' barriers exist before either multicasts into the other
  else __syncthreads();

  if (wg == 0) {
    setmaxnreg_dec<Cfg::PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      // ---------------- TMA producer: one (tap, 64-channel) slice per stage
      const uint32_t stage_tx = (HALO ? 0u : 2u * (uint32_t)rows_valid * 128u) + 2u * (uint32_t)Cfg::B_BYTES;
      const uint32_t patch_tx = 2u * (uint32_t)(a.th + 2) * (uint32_t)((TC_HALO_TW + 2) * 128);
      const uint32_t res_tx = 2u * (uint32_t)rows_valid * 128u;
      uint32_t git = 0, gpatch = 0, gslot = 0;
      TcSched sched(a.sk_mode, total_tiles, n_iters, sched_id, sched_n);
      TcItem item;
      while (sched.next(item)) {
        const int t = item.tile;
        const int nt = t % a.n_tiles, mt = PAIR ? 2 * (t / a.n_tiles) + rank : t / a.n_tiles;
        const int x0 = (mt % a.tiles_w) * a.tw, y0 = ((mt / a.tiles_w) % a.tiles_h) * a.th;
        const int img0 = (mt / (a.tiles_w * a.tiles_h)) * a.nb, n0 = nt * BN;
        int patch_cc = -1;
        for (int k = item.k0; k < item.k1; ++k, ++git) {
          // K order: tap-major for the im2col kernels, 64-channel-slice-major for HALO (nine taps share one patch)
          const int tap = HALO ? k % 9 : k / cchunks, cc = HALO ? k / 9 : k - tap * cchunks;
          const int r = tap / a.kw, s = tap % a.kw;
          const int iy = y0 * a.stride + r * a.rate - a.pad_t, ix = x0 * a.stride + s * a.rate - a.pad_l;
          if (HALO && cc != patch_cc) {
            patch_cc = cc;
            const uint32_t pb = gpatch & 1u;
            mbar_wait(&patch_empty_bar[pb], ((gpatch >> 1) & 1u) ^ 1u);
            uint8_t* pbase = patch + pb * Cfg::PATCH_BYTES;
            mbar_arrive_expect_tx(&patch_full_bar[pb], patch_tx);
            for (int i = 0; i < a.th + 2; ++i) {
              tma_load_4d(pbase + i * TC_HALO_PITCH, &a.tm_a_hi, &patch_full_bar[pb], cc * 64, x0 - a.pad_l,
                          y0 - a.pad_t + i, img0);
              tma_load_4d(pbase + TC_HALO_PLANE_BYTES + i * TC_HALO_PITCH, &a.tm_a_lo, &patch_full_bar[pb], cc * 64,
                          x0 - a.pad_l, y0 - a.pad_t + i, img0);
            }
            ++gpatch;
          }
          const uint32_t st = git % STAGES, ph = (git / STAGES) & 1u;
          mbar_wait(&empty_bar[st], ph ^ 1u);
          uint8_t* sbase = stages + st * Cfg::STAGE_BYTES;
          const int kcol = tap * a.cin + cc * 64;
          mbar_arrive_expect_tx(&full_bar[st], stage_tx);
          if (!HALO) {
            tma_load_4d(sbase, &a.tm_a_hi, &full_bar[st], cc * 64, ix, iy, img0);
            tma_load_4d(sbase + TC_A_BYTES, &a.tm_a_lo, &full_bar[st], cc * 64, ix, iy, img0);
          }
          uint8_t* bbase = sbase + Cfg::A_STAGE_BYTES;
          if (PAIR) {          // this CTA's half of the weight rows, into the same offset of both CTAs
            const int off = rank * (BN / 2);
            tma_load_2d_mc(bbase + off * 128, &a.tm_b_hi, &full_bar[st], kcol, n0 + off, 0x3);
            tma_load_2d_mc(bbase + Cfg::B_BYTES + off * 128, &a.tm_b_lo, &full_bar[st], kcol, n0 + off, 0x3);
          } else {
            tma_load_2d(bbase, &a.tm_b_hi, &full_bar[st], kcol, n0);
            tma_load_2d(bbase + Cfg::B_BYTES, &a.tm_b_lo, &full_bar[st], kcol, n0);
          }
        }
        // the tile's slots, after its K slices (which need no slot): the CTA holding the head of the tile runs the
        // epilogue.  The residual lands while the consumers work through those slices.
        if constexpr (SLOTS > 0) {
          for (int g = 0; g < NGT && item.k0 == 0; ++g, ++gslot) {
            const uint32_t sl = gslot % SLOTS;
            mbar_wait(&slot_empty_bar[sl], ((gslot / SLOTS) & 1u) ^ 1u);
            if (a.res_hi) {
              uint8_t* sb = slots + sl * Cfg::SLOT_BYTES;
              mbar_arrive_expect_tx(&slot_full_bar[sl], res_tx);
              tma_load_4d(sb, &a.tm_r_hi, &slot_full_bar[sl], n0 + g * 64, x0 * a.res_stride, y0 * a.res_stride, img0);
              tma_load_4d(sb + TC_A_BYTES, &a.tm_r_lo, &slot_full_bar[sl], n0 + g * 64, x0 * a.res_stride,
                          y0 * a.res_stride, img0);
            } else {
              mbar_arrive(&slot_full_bar[sl]);
            }
          }
        }
      }
    }
  } else {
    // ---------------- consumer warpgroups: rows wrow .. wrow + 63, columns wcol .. wcol + WN - 1 of the tile
    setmaxnreg_inc<Cfg::CONSUMER_REGS>();
    const int c = wg - 1;
    const int ctid = threadIdx.x - 128;               // 0 .. 128 NCWG - 1 over the consumer warpgroups
    const int wrow = (c & 1) * 64, wcol = (c >> 1) * WN;
    const int lrow = ((threadIdx.x & 127) >> 5) * 16 + ((threadIdx.x & 31) >> 2);   // + 8 for the odd register pairs
    const int lcol = 2 * (threadIdx.x & 3);
    uint32_t git = 0, gpatch = 0;
    // slot epilogue: the slot sequence of the producer, and the stores of this warpgroup pair's columns are issued
    // (and their slots freed, in order from `rel`) by thread 0 of the row-0 warpgroup
    uint32_t gslot = 0, rel = 0;
    const bool slot_issuer = (threadIdx.x & 127) == 0 && (c & 1) == 0;
    TcSched sched(a.sk_mode, total_tiles, n_iters, sched_id, sched_n);
    TcItem item;
    while (sched.next(item)) {
      const int t = item.tile;
      const int nt = t % a.n_tiles, mt = PAIR ? 2 * (t / a.n_tiles) + rank : t / a.n_tiles;
      const int x0 = (mt % a.tiles_w) * a.tw, y0 = ((mt / a.tiles_w) % a.tiles_h) * a.th;
      const int img0 = (mt / (a.tiles_w * a.tiles_h)) * a.nb;
      const int n0 = nt * BN + wcol;

      float racc[NR];
#pragma unroll
      for (int j = 0; j < NR; ++j) racc[j] = 0.f;
      int patch_cc = -1;
      uint32_t pb = 0;
      // waits until slice k (ring position g) has landed and returns its operand descriptors
      auto acquire = [&](int k, uint32_t g) {
        TcSlice s;
        s.st = g % STAGES;
        if (HALO) {
          const int cc = k / 9, tap = k - cc * 9;
          if (cc != patch_cc) {
            patch_cc = cc;
            pb = gpatch & 1u;
            mbar_wait(&patch_full_bar[pb], (gpatch >> 1) & 1u);
            ++gpatch;
          }
          // view of the patch shifted by tap (r, s): row 8 g + j of the operand = patch pixel (g + r, j + s)
          const int r = tap / 3, c3 = tap - r * 3;
          const uint32_t pa = smem_u32(patch + pb * Cfg::PATCH_BYTES) + (uint32_t)(((wrow >> 3) + r) * TC_HALO_PITCH + c3 * 128);
          s.ahi = make_sw128_kmajor_desc(pa, TC_HALO_PITCH);
          s.alo = make_sw128_kmajor_desc(pa + TC_HALO_PLANE_BYTES, TC_HALO_PITCH);
        }
        s.pb = pb;
        mbar_wait(&full_bar[s.st], (g / STAGES) & 1u);
        const uint32_t sa = smem_u32(stages + s.st * Cfg::STAGE_BYTES);
        if (!HALO) {
          s.ahi = make_sw128_kmajor_desc(sa + wrow * 128);
          s.alo = make_sw128_kmajor_desc(sa + TC_A_BYTES + wrow * 128);
        }
        s.bhi = make_sw128_kmajor_desc(sa + Cfg::A_STAGE_BYTES + wcol * 128);
        s.blo = make_sw128_kmajor_desc(sa + Cfg::A_STAGE_BYTES + Cfg::B_BYTES + wcol * 128);
        return s;
      };
      // the wgmma of slice k have completed: free its stage (pair: in both CTAs) and, after the last tap of a channel
      // slice, its patch buffer -- the buffer of the slice retired, not of one issued since
      auto release = [&](int k, const TcSlice& s) {
        if ((threadIdx.x & 127) == 0) {
          mbar_arrive(&empty_bar[s.st]);
          if (PAIR) mbar_arrive_cluster(&empty_bar[s.st], (uint32_t)(rank ^ 1));
          if (HALO && (k + 1 == item.k1 || (k + 1) % 9 == 0)) mbar_arrive(&patch_empty_bar[s.pb]);
        }
      };
      auto fold = [&](float (&d)[NR]) {
        wgmma_fence_operand(d);
#pragma unroll
        for (int j = 0; j < NR; ++j) racc[j] = __fadd_rn(racc[j], d[j]);
      };
      if constexpr (BN == 256) {
        // two 128-column halves per slice (see above); the stage is freed once the second half has read it
        constexpr uint64_t HALF_B = (128 * 128) >> 4;   // 128 weight rows, in 16 B descriptor units
        for (int k = item.k0; k < item.k1; ++k, ++git) {
          const TcSlice s = acquire(k, git);
          float d[NR / 2];
          tc_slice_mma<128>(d, s);
          wgmma_wait0();
          wgmma_fence_operand(d);
#pragma unroll
          for (int j = 0; j < NR / 2; ++j) racc[j] = __fadd_rn(racc[j], d[j]);
          TcSlice s1 = s;
          s1.bhi += HALF_B;
          s1.blo += HALF_B;
          tc_slice_mma<128>(d, s1);
          wgmma_wait0();
          release(k, s);
          wgmma_fence_operand(d);
#pragma unroll
          for (int j = 0; j < NR / 2; ++j) racc[NR / 2 + j] = __fadd_rn(racc[NR / 2 + j], d[j]);
        }
      } else if constexpr (PIPE) {
        // slices alternate between d0 and d1 at compile-time-known places (a run-time choice of the tile serialises
        // the wgmma); the loop runs two slices per trip, the tail finishes one or two
        const int k1 = item.k1;
        int k = item.k0;
        float d0[NR], d1[NR];
        TcSlice s0 = acquire(k, git), s1;
        tc_slice_mma<WN>(d0, s0);
        for (; k + 2 < k1; k += 2, git += 2) {
          s1 = acquire(k + 1, git + 1);
          tc_slice_mma<WN>(d1, s1);
          wgmma_wait1();                              // slice k done, k + 1 in flight
          release(k, s0);
          fold(d0);
          s0 = acquire(k + 2, git + 2);
          tc_slice_mma<WN>(d0, s0);
          wgmma_wait1();
          release(k + 1, s1);
          fold(d1);
        }
        if (k + 1 < k1) {
          s1 = acquire(k + 1, git + 1);
          tc_slice_mma<WN>(d1, s1);
          wgmma_wait1();
          release(k, s0);
          fold(d0);
          wgmma_wait0();
          release(k + 1, s1);
          fold(d1);
          git += 2;
        } else {
          wgmma_wait0();
          release(k, s0);
          fold(d0);
          git += 1;
        }
      } else {
        for (int k = item.k0; k < item.k1; ++k, ++git) {
          const TcSlice s = acquire(k, git);
          float d[NR];
          tc_slice_mma<WN>(d, s);
          wgmma_wait0();
          release(k, s);
          fold(d);
        }
      }

      // ---- stream-K fix-up.  Partial-sum layout [column][row] of the 128 x BN tile, one slot per CTA.
      if (item.k0 != 0) {
        // this CTA continued a tile somebody else started: publish the partial sums, no epilogue
        float* wsp = a.sk_partials + (size_t)blockIdx.x * (128 * BN);
#pragma unroll
        for (int j = 0; j < NR; ++j) {
          const int row = wrow + lrow + ((j & 2) ? 8 : 0), col = wcol + (j >> 2) * 8 + lcol + (j & 1);
          wsp[col * 128 + row] = racc[j];
        }
        __threadfence();
        named_bar_sync(1, 128 * NCWG);                 // all consumer threads have written and fenced
        if (ctid == 0)
          asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(a.sk_flags + blockIdx.x), "r"(a.sk_epoch) : "memory");
        continue;
      }
      if (item.k1 != n_iters) {
        // this CTA holds the head of the tile: the following units hold the rest (they computed it first thing); in a
        // pair the partner in unit u is the CTA of the same rank, slot 2 u + rank
        const long long tile_end = (long long)(item.tile + 1) * n_iters;
        int last_unit = sched_id;
        for (int unit = sched_id + 1;; ++unit) {
          const int cta = PAIR ? 2 * unit + rank : unit;
          int seen;
          do {
            asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(seen) : "l"(a.sk_flags + cta) : "memory");
          } while (seen != a.sk_epoch);
          const float* wsp = a.sk_partials + (size_t)cta * (128 * BN);
#pragma unroll
          for (int j = 0; j < NR; ++j) {
            const int row = wrow + lrow + ((j & 2) ? 8 : 0), col = wcol + (j >> 2) * 8 + lcol + (j & 1);
            racc[j] = __fadd_rn(racc[j], __ldcg(wsp + col * 128 + row));
          }
          last_unit = unit;
          if (TcSched::range_end(unit, total_tiles, n_iters, sched_n) >= tile_end) break;
        }
        // every flag is consumed by exactly one CTA (the one holding the tile's head): clear it once all
        // consumer threads are past their polls, so a REPLAY of this launch with the same epoch (CUDA graph) starts clean
        named_bar_sync(1, 128 * NCWG);
        if (ctid == 0)
          for (int unit = sched_id + 1; unit <= last_unit; ++unit)
            asm volatile("st.relaxed.gpu.global.s32 [%0], %1;" ::"l"(a.sk_flags + (PAIR ? 2 * unit + rank : unit)), "r"(0) : "memory");
      }

      if constexpr (SLOTS > 0) {
        // ---- slot epilogue, one 64-column group at a time (the arithmetic of the register epilogue below)
        bool row_ok[2];                                 // the overflow flag counts real output elements only
#pragma unroll
        for (int hrow = 0; hrow < 2; ++hrow) {
          const int row = wrow + lrow + hrow * 8;
          bool valid = row < rows_valid;
          if (valid) {
            const int nl = row / (a.th * a.tw), rem = row % (a.th * a.tw);
            valid = img0 + nl < a.n && y0 + rem / a.tw < a.ho && x0 + rem % a.tw < a.wo;
          }
          row_ok[hrow] = valid;
        }
        bool ovf = false;
        const bool p_only = PRE && a.out_hi == nullptr;
#pragma unroll
        for (int i = 0; i < WN / 64; ++i) {
          const int cg = wcol / 64 + i;
          const uint32_t gs = gslot + cg, sl = gs % SLOTS;
          uint8_t* sb = slots + sl * Cfg::SLOT_BYTES;
          const int oc = n0 - wcol + cg * 64;
          mbar_wait(&slot_full_bar[sl], (gs / SLOTS) & 1u);
#pragma unroll
          for (int jl = 0; jl < 8; ++jl) {
            const int jb = i * 8 + jl;
            const int c0 = n0 + jb * 8 + lcol;
            const float2 sc = __ldg(reinterpret_cast<const float2*>(a.scale + c0));
            const float2 bi = __ldg(reinterpret_cast<const float2*>(a.bias + c0));
#pragma unroll
            for (int hrow = 0; hrow < 2; ++hrow) {
              // row r of the box, 16 B chunk (column / 8) ^ (r % 8): a warp's 8 rows x 16 B hit all 32 banks once
              const int row = wrow + lrow + hrow * 8;
              const int off = row * 128 + ((jl ^ (row & 7)) << 4) + lcol * 2;
              __half2* ph = reinterpret_cast<__half2*>(sb + off);
              __half2* pl = reinterpret_cast<__half2*>(sb + TC_A_BYTES + off);
              float v0 = fmaf(racc[jb * 4 + hrow * 2 + 0], sc.x, bi.x);
              float v1 = fmaf(racc[jb * 4 + hrow * 2 + 1], sc.y, bi.y);
              if (a.res_hi) {
                const __half2 h2 = *ph, l2 = *pl;
                v0 = add_f16_pair(v0, __low2half(h2), __low2half(l2));
                v1 = add_f16_pair(v1, __high2half(h2), __high2half(l2));
              }
              v0 = apply_act(v0, a.act);
              v1 = apply_act(v1, a.act);
              __half2 h2, l2;
              split2_f32(v0, v1, h2, l2);
              // bitwise, not short-circuit: a branch per column pair would cost the epilogue its straight-line code
              ovf |= row_ok[hrow] & (c0 < a.cout) & (split_overflows(v0) | split_overflows(v1));
              if (p_only) ovf |= row_ok[hrow] && c0 < a.cout && tc_preact(h2, l2, a.pre_scale, a.pre_bias, c0);
              *ph = h2;                                 // in place: each thread rewrites only what it read
              *pl = l2;
            }
          }
          fence_proxy_async();                          // the generic-proxy writes, before the TMA store reads them
          named_bar_sync(2 + cg, 256);                  // the two warpgroups that own rows 0-63 / 64-127 of these columns
          if (slot_issuer) {
            tma_store_4d(&a.tm_o_hi, sb, oc, x0, y0, img0);
            tma_store_4d(&a.tm_o_lo, sb + TC_A_BYTES, oc, x0, y0, img0);
            bulk_commit_group();
          }
          if (PRE && !p_only) {
            // x + p: once the store of x has read the slot, every thread turns the x^ it wrote into p in place
            if (slot_issuer) bulk_wait_group_read<0>();
            named_bar_sync(2 + cg, 256);
#pragma unroll
            for (int jl = 0; jl < 8; ++jl) {
              const int c0 = n0 + (i * 8 + jl) * 8 + lcol;
#pragma unroll
              for (int hrow = 0; hrow < 2; ++hrow) {
                const int row = wrow + lrow + hrow * 8;
                const int off = row * 128 + ((jl ^ (row & 7)) << 4) + lcol * 2;
                __half2* ph = reinterpret_cast<__half2*>(sb + off);
                __half2* pl = reinterpret_cast<__half2*>(sb + TC_A_BYTES + off);
                __half2 h2 = *ph, l2 = *pl;
                ovf |= row_ok[hrow] && c0 < a.cout && tc_preact(h2, l2, a.pre_scale, a.pre_bias, c0);
                *ph = h2;
                *pl = l2;
              }
            }
            fence_proxy_async();
            named_bar_sync(2 + cg, 256);
            if (slot_issuer) {
              tma_store_4d(&a.tm_p_hi, sb, oc, x0, y0, img0);
              tma_store_4d(&a.tm_p_lo, sb + TC_A_BYTES, oc, x0, y0, img0);
              bulk_commit_group();
            }
          }
          if (slot_issuer) {
            if constexpr (NCWG == 4) {                  // one issuer per column group, one slot each (SLOTS == 2)
              bulk_wait_group_read<0>();
              mbar_arrive(&slot_empty_bar[sl]);
            } else if (i + 1 == NGT || SLOTS < NGT) {
              // free the slots whose stores have read them: before the tile's next group when it needs this slot,
              // else at the end of the tile; with a spare slot in the ring the newest store stays in flight
              constexpr int KEEP = SLOTS > NGT ? 1 : 0;
              const bool last = i + 1 == NGT;
              if (last) bulk_wait_group_read<KEEP>();
              else bulk_wait_group_read<0>();
              for (const uint32_t upto = gs + 1 - (last ? KEEP : 0); rel < upto; ++rel)
                mbar_arrive(&slot_empty_bar[rel % SLOTS]);
            }
          }
        }
        gslot += NGT;
        if (ovf && a.overflow) atomicOr(a.overflow, 1);
      } else {
        // ---- scale/bias (folded BN) -> +residual -> activation -> store; two rows per thread, column pairs
#pragma unroll
        for (int hrow = 0; hrow < 2; ++hrow) {
          const int row = wrow + lrow + hrow * 8;
          bool valid = row < rows_valid;
          int n_img = 0, oy = 0, ox = 0;
          if (valid) {
            const int nl = row / (a.th * a.tw);
            const int rem = row % (a.th * a.tw);
            n_img = img0 + nl; oy = y0 + rem / a.tw; ox = x0 + rem % a.tw;
            valid = n_img < a.n && oy < a.ho && ox < a.wo;
          }
          const size_t opix = ((size_t)n_img * a.ho + oy) * a.wo + ox;
          size_t rpix = 0;
          if (a.res_hi)
            rpix = ((size_t)n_img * a.res_h + (size_t)oy * a.res_stride) * a.res_w + (size_t)ox * a.res_stride;
          bool ovf = false;
#pragma unroll
          for (int jb = 0; jb < WN / 8; ++jb) {
            const int c0 = n0 + jb * 8 + lcol;
            if (!valid || c0 >= a.cout) continue;
            // scale / bias vectors are padded to cout_pad (even): 8 B loads are always in bounds
            const float2 sc = __ldg(reinterpret_cast<const float2*>(a.scale + c0));
            const float2 bi = __ldg(reinterpret_cast<const float2*>(a.bias + c0));
            float v0 = fmaf(racc[jb * 4 + hrow * 2 + 0], sc.x, bi.x);
            float v1 = fmaf(racc[jb * 4 + hrow * 2 + 1], sc.y, bi.y);
            if (a.res_hi) {              // residual tensors always have cout % 32 == 0 channels
              const __half2 h2 = *reinterpret_cast<const __half2*>(a.res_hi + rpix * a.cout + c0);
              const __half2 l2 = *reinterpret_cast<const __half2*>(a.res_lo + rpix * a.cout + c0);
              v0 = add_f16_pair(v0, __low2half(h2), __low2half(l2));
              v1 = add_f16_pair(v1, __high2half(h2), __high2half(l2));
            }
            v0 = apply_act(v0, a.act);
            v1 = apply_act(v1, a.act);
            if (a.out_f32) {
              float* op = a.out_f32 + opix * a.cout + c0;
              if ((a.cout & 1) == 0) {
                *reinterpret_cast<float2*>(op) = make_float2(v0, v1);
              } else {
                op[0] = v0;
                if (c0 + 1 < a.cout) op[1] = v1;
              }
            } else {                     // split outputs always have cout % 32 == 0
              // packed split: hi = rn16(v), lo = rn16(v - hi)
              __half2 h2, l2;
              split2_f32(v0, v1, h2, l2);
              ovf |= split_overflows(v0) || split_overflows(v1);
              if (!PRE || a.out_hi) {
                *reinterpret_cast<__half2*>(a.out_hi + opix * a.cout + c0) = h2;
                *reinterpret_cast<__half2*>(a.out_lo + opix * a.cout + c0) = l2;
              }
              if constexpr (PRE) {
                ovf |= tc_preact(h2, l2, a.pre_scale, a.pre_bias, c0);
                *reinterpret_cast<__half2*>(a.pre_hi + opix * a.cout + c0) = h2;
                *reinterpret_cast<__half2*>(a.pre_lo + opix * a.cout + c0) = l2;
              }
            }
          }
          if (ovf && a.overflow) atomicOr(a.overflow, 1);
        }
      }
    }
    if (SLOTS && slot_issuer) bulk_wait_group0();     // the stores are complete before the CTA (and its smem) ends
  }
  // PAIR: the peer's shared memory and barriers must stay alive until both CTAs are done with them
  if (PAIR) cluster_sync_all();
}

// ---------------------------------------------------------------- host: TMA descriptors
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  if (!fn) throw Error(-2, "cuTensorMapEncodeTiled not available from the driver");
  return fn;
}

// `stride` > 1 (strided conv): TMA traversal stride along W and H -- the box spans tw*stride x th*stride
// input pixels and every stride-th one is copied, so smem still receives tw x th rows.
static CUtensorMap make_map_act(const __half* base, int n, int h, int w, int c, int nb, int th, int tw, int stride,
                                long pix_pitch, long row_pitch, long img_pitch) {
  CUtensorMap m;
  if (!pix_pitch) pix_pitch = c;
  if (!row_pitch) row_pitch = (long)w * c;
  if (!img_pitch) img_pitch = (long)h * w * c;
  cuuint64_t dims[4] = {(cuuint64_t)c, (cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)n};
  cuuint64_t strides[3] = {(cuuint64_t)pix_pitch * 2, (cuuint64_t)row_pitch * 2, (cuuint64_t)img_pitch * 2};
  cuuint32_t box[4] = {64, (cuuint32_t)(tw * stride), (cuuint32_t)(th * stride), (cuuint32_t)nb};
  cuuint32_t es[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
  CUresult r = get_encode_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, (void*)base, dims, strides, box, es,
                               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                               CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw Error(-2, "cuTensorMapEncodeTiled(activation) failed: " + std::to_string((int)r));
  return m;
}

static CUtensorMap make_map_wgt(const __half* base, int rows, int kdim, int bn) {
  CUtensorMap m;
  cuuint64_t dims[2] = {(cuuint64_t)kdim, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)kdim * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)bn};
  cuuint32_t es[2] = {1, 1};
  CUresult r = get_encode_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)base, dims, strides, box, es,
                               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                               CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw Error(-2, "cuTensorMapEncodeTiled(weights) failed: " + std::to_string((int)r));
  return m;
}

// descriptor cache: engine buffers are static, so every (pointer, geometry) repeats each predict call.
// `kind` keeps the maps of different uses of one pointer apart (an epilogue store map never stands in for a load map).
enum MapKind { MAP_LOAD = 0, MAP_STORE = 1 };
struct MapKey {
  const void* p; int a, b, c, d, e, f, g, kind;
  bool operator<(const MapKey& o) const {
    return std::tie(p, a, b, c, d, e, f, g, kind) < std::tie(o.p, o.a, o.b, o.c, o.d, o.e, o.f, o.g, o.kind);
  }
};
static std::map<MapKey, CUtensorMap> g_map_cache;
static std::mutex g_map_mutex;

static CUtensorMap cached_act_map(const __half* base, int n, int h, int w, int c, int nb, int th, int tw, int stride,
                                  long pix_pitch, long row_pitch, long img_pitch, MapKind kind = MAP_LOAD) {
  std::lock_guard<std::mutex> lk(g_map_mutex);
  MapKey k{base, n, h, w, c + (int)(pix_pitch << 12), nb, th * 16 + stride, tw, kind};
  auto it = g_map_cache.find(k);
  if (it != g_map_cache.end()) return it->second;
  if (g_map_cache.size() > 4096) g_map_cache.clear();
  CUtensorMap m = make_map_act(base, n, h, w, c, nb, th, tw, stride, pix_pitch, row_pitch, img_pitch);
  g_map_cache[k] = m;
  return m;
}
static CUtensorMap cached_wgt_map(const __half* base, int rows, int kdim, int bn) {
  std::lock_guard<std::mutex> lk(g_map_mutex);
  MapKey k{base, rows, kdim, bn, -1, -1, -1, -1, MAP_LOAD};
  auto it = g_map_cache.find(k);
  if (it != g_map_cache.end()) return it->second;
  CUtensorMap m = make_map_wgt(base, rows, kdim, bn);
  g_map_cache[k] = m;
  return m;
}

// M-tile geometry: (nb, th, tw) with nb*th*tw <= 128 maximising useful rows per tile.
static void pick_tile(int n, int ho, int wo, int& nb, int& th, int& tw) {
  double best = -1.0;
  nb = 1; th = 1; tw = 1;
  for (int w_ = 1; w_ <= 128 && w_ <= wo; ++w_) {
    int hmax = 128 / w_;
    if (hmax > ho) hmax = ho;
    for (int h_ = 1; h_ <= hmax; ++h_) {
      int b_ = 1;
      if (h_ == ho && w_ == wo) { b_ = 128 / (h_ * w_); if (b_ > n) b_ = n; if (b_ < 1) b_ = 1; }
      long tiles = (long)cdiv(n, b_) * cdiv(ho, h_) * cdiv(wo, w_);
      double eff = (double)n * ho * wo / ((double)tiles * 128.0);
      // prefer wide tiles on ties (longer contiguous TMA rows)
      if (eff > best + 1e-9 || (eff > best - 1e-9 && w_ > tw)) { best = eff; nb = b_; th = h_; tw = w_; }
    }
  }
}

bool conv_tc_supported(const ConvLayer& L, const ConvIO& io) {
  if (!L.tc_ready) return false;
  if (L.stride != 1 && L.stride != 2) return false;
  if (L.stride == 2 && L.rate != 1) return false;
  if (L.cin % 64 != 0) return false;
  if (io.out_f32 == nullptr && (L.cout % 32) != 0) return false;
  if (io.res.hi && (L.cout % 32) != 0) return false;
  if (io.pre.hi && (io.out_f32 || !io.pre_scale || !io.pre_bias)) return false;
  return true;
}

// SMs a persistent conv launch may occupy.  While the engine runs its two-stream pipeline it leaves
// io.sm_reserve SMs free so the few-CTA latency-bound kernels (sort, NMS scan) of the other half-batch
// run concurrently instead of waiting behind a persistent grid that fills every SM.
// The count is cached per DEVICE (an engine may live on any device of the process).
int device_sm_count() {
  static int n[LUMI_MAX_DEVICES] = {0};
  int dev = 0;
  LUMI_CUDA_CHECK(cudaGetDevice(&dev));
  if (dev < 0 || dev >= LUMI_MAX_DEVICES) {
    int v = 0;
    LUMI_CUDA_CHECK(cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev));
    return v;
  }
  int v = __atomic_load_n(&n[dev], __ATOMIC_RELAXED);
  if (!v) {
    LUMI_CUDA_CHECK(cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev));
    __atomic_store_n(&n[dev], v, __ATOMIC_RELAXED);
  }
  return v;
}
int sm_budget(int reserve, int limit) {
  int n = device_sm_count();
  if (limit > 0 && limit < n) n = limit;
  return (reserve > 0 && reserve < n) ? n - reserve : n;
}

void conv_workspace_create(ConvWorkspace& w) {
  int dev = 0, n = 0;
  LUMI_CUDA_CHECK(cudaGetDevice(&dev));
  LUMI_CUDA_CHECK(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
  w.ctas = n;
  LUMI_CUDA_CHECK(cudaMalloc(&w.partials, (size_t)n * 128 * TC_BN_MAX * sizeof(float)));
  LUMI_CUDA_CHECK(cudaMalloc(&w.flags, (size_t)n * sizeof(int)));
  LUMI_CUDA_CHECK(cudaMemset(w.flags, 0, (size_t)n * sizeof(int)));
  w.epoch = 0;
}
void conv_workspace_free(ConvWorkspace& w) {
  cudaFree(w.partials); cudaFree(w.flags);
  w.partials = nullptr; w.flags = nullptr; w.ctas = 0;
}

template <int BN, int STAGES, int NCWG, bool PAIR, bool HALO, bool PIPE, int SLOTS, bool PRE>
static void launch_tc_cfg(const TcArgs& a, ConvWorkspace* sk, int streamk, int sms, cudaStream_t st) {
  using Cfg = TcCfg<BN, STAGES, NCWG, PAIR, HALO, SLOTS>;
  auto kernel = conv_tc_kernel<BN, STAGES, NCWG, PAIR, HALO, PIPE, SLOTS, PRE>;
  // cudaFuncSetAttribute is per device: one flag per (kernel instance, device)
  static bool attr_set[LUMI_MAX_DEVICES] = {false};
  int dev = 0;
  LUMI_CUDA_CHECK(cudaGetDevice(&dev));
  if (dev < 0 || dev >= LUMI_MAX_DEVICES || !__atomic_load_n(&attr_set[dev], __ATOMIC_ACQUIRE)) {
    LUMI_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    if (dev >= 0 && dev < LUMI_MAX_DEVICES) __atomic_store_n(&attr_set[dev], true, __ATOMIC_RELEASE);
  }
  const long m_tiles = (long)a.tiles_w * a.tiles_h * a.tiles_n;
  const long total = (PAIR ? (m_tiles + 1) / 2 : m_tiles) * a.n_tiles;      // scheduling units (tiles or tile pairs)
  int units_max = PAIR ? sms / 2 : sms;
  if (PAIR) {
    LUMI_REQUIRE(units_max >= 1, "conv_tc: the 2-CTA cluster kernel needs a budget of at least 2 SMs, got " +
                                     std::to_string(sms));
    // stream-K needs every cluster of the grid resident at once: never launch more pairs than can be co-scheduled
    static int max_clusters[LUMI_MAX_DEVICES] = {0};
    int mc = (dev >= 0 && dev < LUMI_MAX_DEVICES) ? __atomic_load_n(&max_clusters[dev], __ATOMIC_RELAXED) : 0;
    if (!mc) {
      cudaLaunchConfig_t cfg;
      std::memset(&cfg, 0, sizeof(cfg));
      cfg.gridDim = dim3(2 * units_max, 1, 1);
      cfg.blockDim = dim3(Cfg::THREADS, 1, 1);
      cfg.dynamicSmemBytes = Cfg::SMEM_BYTES;
      cudaLaunchAttribute at[1];
      at[0].id = cudaLaunchAttributeClusterDimension;
      at[0].val.clusterDim.x = 2; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
      cfg.attrs = at;
      cfg.numAttrs = 1;
      LUMI_CUDA_CHECK(cudaOccupancyMaxActiveClusters(&mc, kernel, &cfg));
      LUMI_REQUIRE(mc > 0, "conv_tc: the 2-CTA cluster kernel cannot be scheduled on this device");
      if (dev >= 0 && dev < LUMI_MAX_DEVICES) __atomic_store_n(&max_clusters[dev], mc, __ATOMIC_RELAXED);
    }
    if (units_max > mc) units_max = mc;
  }
  TcArgs args = a;
  args.sk_mode = 0;
  int units = (int)(total < units_max ? total : units_max);             // persistent: one CTA (pair) per SM (pair)
  if (sk && sk->partials && streamk > 0 && sms <= sk->ctas) {
    // stream-K when whole-tile scheduling would leave SMs idle in the last wave (or has fewer tiles than SMs).
    // It balances K iterations, not epilogues, and every CTA pays one partial-tile write and one read, so it is
    // kept to the long-K layers (3x3 with C_in >= 128, 1x1 with C_in >= 1024, the RPN conv).
    const long n_iters = (long)a.kh * a.kw * (a.cin >> 6);
    const double waves = (double)total / units_max;
    const double eff = waves / std::ceil(waves);
    const long units_per_cta = total * n_iters / units_max;
    const bool forced = streamk >= 2 && units_per_cta >= 3;
    if (forced || (eff < 0.92 && n_iters >= 12 && units_per_cta >= 12)) {
      args.sk_mode = 1;
      args.sk_partials = sk->partials;
      args.sk_flags = sk->flags;
      args.sk_epoch = (int)(++sk->epoch & 0x7fffffff);
      units = units_max;
    }
  }
  if (PAIR) {
    cudaLaunchConfig_t cfg;
    std::memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(2 * units, 1, 1);
    cfg.blockDim = dim3(Cfg::THREADS, 1, 1);
    cfg.dynamicSmemBytes = Cfg::SMEM_BYTES;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = 2; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    LUMI_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kernel, args));
  } else {
    kernel<<<units, Cfg::THREADS, Cfg::SMEM_BYTES, st>>>(args);
  }
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
}

// io.pipe selects the double-buffered slice accumulators (the single-buffered loop is kept for A/B runs); a
// pre-activation output selects the PRE instances, which exist for the non-halo kernels only
template <int BN, int STAGES, int NCWG = 2, bool PAIR = false, bool HALO = false, int SLOTS = 0>
static void launch_tc(const TcArgs& a, const ConvIO& io, cudaStream_t st) {
  const int sms = sm_budget(io.sm_reserve, io.sm_limit);
  if constexpr (!HALO) {
    if (io.pre.hi) {
      if (io.pipe) launch_tc_cfg<BN, STAGES, NCWG, PAIR, HALO, true, SLOTS, true>(a, io.sk, io.streamk, sms, st);
      else launch_tc_cfg<BN, STAGES, NCWG, PAIR, HALO, false, SLOTS, true>(a, io.sk, io.streamk, sms, st);
      return;
    }
  }
  if (io.pipe) launch_tc_cfg<BN, STAGES, NCWG, PAIR, HALO, true, SLOTS, false>(a, io.sk, io.streamk, sms, st);
  else launch_tc_cfg<BN, STAGES, NCWG, PAIR, HALO, false, SLOTS, false>(a, io.sk, io.streamk, sms, st);
}

void launch_conv_tc(const ConvLayer& L, const ConvIO& io, cudaStream_t st) {
  LUMI_REQUIRE(conv_tc_supported(L, io), "conv_tc: layer not supported by the tensor-core kernel");
  LUMI_REQUIRE(io.in.c == L.cin, "conv_tc: channel mismatch");
  if ((long)io.in.n * io.ho * io.wo == 0) return;
  TcArgs a;
  std::memset(&a, 0, sizeof(a));
  int nb, th, tw;
  pick_tile(io.in.n, io.ho, io.wo, nb, th, tw);
  const long n_iters_all = (long)L.kh * L.kw * (L.cin >> 6);
  // 128 x 256 tiles (slot epilogue, no pre-activation output) on the layers with at least io.wide K slices and enough
  // of those tiles for io.wide_sm_pct % of the SMs: on SSD's small extra layers (1-64 tiles) they measured up to 1.8x
  // slower (DESIGN 7.1).  They are never halo or cluster-pair layers.
  const long wide_tiles = (long)cdiv(io.in.n, nb) * cdiv(io.ho, th) * cdiv(io.wo, tw) * (L.cout_pad / 256);
  const bool wide = io.wide && L.cout_pad % 256 == 0 && n_iters_all >= io.wide && !io.out_f32 && io.epi_tma &&
                    !io.pre.hi && wide_tiles * 100 >= (long)sm_budget(io.sm_reserve, io.sm_limit) * io.wide_sm_pct;
  const int bn = wide ? 256 : (L.cout_pad % 128 == 0) ? 128 : 64;
  // halo-patch kernels (3x3, stride 1, rate 1, SAME): tiles of th x 8 pixels of one image, th <= 16 chosen so that the
  // rows of the map split evenly.  They trade M-tile occupancy (th * 8 <= 128 rows, and the weights stream once per
  // tile) for ~6x less activation traffic, so they are used while the tile count stays within io.halo_tiles_pct of the
  // generic one.
  bool halo = false;
  if (io.halo && !wide && L.kh == 3 && L.kw == 3 && L.stride == 1 && L.rate == 1 && io.pad_t == 1 && io.pad_l == 1 &&
      !io.res.hi && !io.out_f32 && !io.pre.hi && !io.in_pix_pitch && !io.in_row_pitch && !io.in_img_pitch) {
    const int h_tiles = cdiv(io.ho, 16), h_th = cdiv(io.ho, h_tiles);
    const long std_tiles = (long)cdiv(io.in.n, nb) * cdiv(io.ho, th) * cdiv(io.wo, tw);
    const long halo_tiles = (long)io.in.n * h_tiles * cdiv(io.wo, TC_HALO_TW);
    if (halo_tiles * 100 <= std_tiles * io.halo_tiles_pct) { halo = true; nb = 1; th = h_th; tw = TC_HALO_TW; }
  }
  if (halo) {            // the activation maps describe one patch row: box {64 ch, 10, 1, 1}
    a.tm_a_hi = cached_act_map(io.in.hi, io.in.n, io.in.h, io.in.w, io.in.c, 1, 1, TC_HALO_TW + 2, 1, 0, 0, 0);
    a.tm_a_lo = cached_act_map(io.in.lo, io.in.n, io.in.h, io.in.w, io.in.c, 1, 1, TC_HALO_TW + 2, 1, 0, 0, 0);
  } else {
    a.tm_a_hi = cached_act_map(io.in.hi, io.in.n, io.in.h, io.in.w, io.in.c, nb, th, tw, L.stride, io.in_pix_pitch,
                               io.in_row_pitch, io.in_img_pitch);
    a.tm_a_lo = cached_act_map(io.in.lo, io.in.n, io.in.h, io.in.w, io.in.c, nb, th, tw, L.stride, io.in_pix_pitch,
                               io.in_row_pitch, io.in_img_pitch);
  }
  // CTA pairs on the long-K layers: each CTA of a pair loads (and multicasts) 64 of the 128 weight rows
  const bool pair = io.cta2 && bn == 128 && !io.out_f32 && n_iters_all >= io.cta2;
  const int kdim = L.kh * L.kw * L.cin;
  a.tm_b_hi = cached_wgt_map(L.w_hi, L.cout_pad, kdim, pair ? bn / 2 : bn);
  a.tm_b_lo = cached_wgt_map(L.w_lo, L.cout_pad, kdim, pair ? bn / 2 : bn);
  a.scale = L.scale_tc; a.bias = L.bias;
  a.out_hi = io.out.hi; a.out_lo = io.out.lo; a.out_f32 = io.out_f32;
  a.res_hi = io.res.hi; a.res_lo = io.res.lo; a.res_h = io.res.h; a.res_w = io.res.w; a.res_stride = io.res_stride;
  a.n = io.in.n; a.ho = io.ho; a.wo = io.wo; a.cin = L.cin; a.cout = L.cout;
  a.kh = L.kh; a.kw = L.kw; a.rate = L.rate; a.pad_t = io.pad_t; a.pad_l = io.pad_l; a.act = L.act;
  a.nb = nb; a.th = th; a.tw = tw;
  a.tiles_w = cdiv(io.wo, tw); a.tiles_h = cdiv(io.ho, th); a.tiles_n = cdiv(io.in.n, nb);
  a.n_tiles = L.cout_pad / bn;
  a.stride = L.stride;
  a.overflow = io.overflow_flag;
  a.pre_scale = io.pre_scale; a.pre_bias = io.pre_bias; a.pre_hi = io.pre.hi; a.pre_lo = io.pre.lo;
  // operands per stage: 64 KB (BN = 128) or 48 KB (BN = 64), B only for HALO (next to two 72 KB patch buffers)
  if (halo) {
    if (pair) launch_tc<128, 2, 2, true, true>(a, io, st);
    else if (bn == 128) launch_tc<128, 2, 2, false, true>(a, io, st);
    else launch_tc<64, 4, 2, false, true>(a, io, st);
    return;
  }
  // four consumer warpgroups (sixteen epilogue warps) for the shortest-K layers (io.epi16 = largest K-slice count)
  const bool epi16 = io.epi16 && bn == 128 && !io.out_f32 && n_iters_all <= io.epi16;
  if (pair) { launch_tc<128, 3, 2, true>(a, io, st); return; }
  // split outputs leave through the slot epilogue: on an H100 it was faster on every split-output layer of the R50
  // step, 1x1 and 3x3, short and long K (DESIGN 7.1).  Per instance, the slot count that measured best: two (one per
  // column group) with four consumers, one next to three operand stages for BN = 128 (the 36-slice 3x3 layers want
  // the third stage), two next to three stages for BN = 64.
  if (!io.out_f32 && io.epi_tma) {
    if (io.pre.hi) {
      a.tm_p_hi = cached_act_map(io.pre.hi, io.in.n, io.ho, io.wo, L.cout, nb, th, tw, 1, 0, 0, 0, MAP_STORE);
      a.tm_p_lo = cached_act_map(io.pre.lo, io.in.n, io.ho, io.wo, L.cout, nb, th, tw, 1, 0, 0, 0, MAP_STORE);
    }
    if (io.out.hi) {
      a.tm_o_hi = cached_act_map(io.out.hi, io.in.n, io.ho, io.wo, L.cout, nb, th, tw, 1, 0, 0, 0, MAP_STORE);
      a.tm_o_lo = cached_act_map(io.out.lo, io.in.n, io.ho, io.wo, L.cout, nb, th, tw, 1, 0, 0, 0, MAP_STORE);
    } else {                                     // p only: the slot's one store carries p
      a.tm_o_hi = a.tm_p_hi;
      a.tm_o_lo = a.tm_p_lo;
    }
    if (io.res.hi) {
      a.tm_r_hi = cached_act_map(io.res.hi, io.res.n, io.res.h, io.res.w, io.res.c, nb, th, tw, io.res_stride, 0, 0, 0);
      a.tm_r_lo = cached_act_map(io.res.lo, io.res.n, io.res.h, io.res.w, io.res.c, nb, th, tw, io.res_stride, 0, 0, 0);
    }
    // the wide tile: 2 x 96 KB stages + one slot (224 KB); a slice is twice the MMA work of a BN = 128 slice, so two
    // stages keep as much of it in flight as four do there
    if (wide)
      launch_tc_cfg<256, 2, 2, false, false, false, 1, false>(a, io.sk, io.streamk,
                                                              sm_budget(io.sm_reserve, io.sm_limit), st);
    else if (epi16) launch_tc<128, 2, 4, false, false, 2>(a, io, st);
    else if (bn == 128) launch_tc<128, 3, 2, false, false, 1>(a, io, st);
    else launch_tc<64, 3, 2, false, false, 2>(a, io, st);
    return;
  }
  if (epi16) launch_tc<128, 3, 4>(a, io, st);
  else if (bn == 128) launch_tc<128, 3>(a, io, st);
  else launch_tc<64, 4>(a, io, st);
}

// ---------------------------------------------------------------- host: weight packing
void pack_conv_weights(const float* w, size_t kdim, int cout, const float* scale, __half* hi, __half* lo,
                       float* scale_tc) {
  for (int c = 0; c < cout; ++c) {
    float mx = 0.f;
    for (size_t k = 0; k < kdim; ++k) mx = std::fmax(mx, std::fabs(w[k * cout + c]));
    int e = 0;
    if (mx > 0.f && std::isfinite(mx)) {
      int ex;
      std::frexp(mx, &ex);            // mx = f * 2^ex, f in [0.5,1)
      e = 14 - ex;                    // mx * 2^e in [2^13, 2^14)
      e = std::min(std::max(e, -CONV_PACK_EXP_MAX), CONV_PACK_EXP_MAX);
    }
    const float up = std::ldexp(1.f, e);
    for (size_t k = 0; k < kdim; ++k) {
      float v = w[k * cout + c] * up;
      __half h = __float2half_rn(v);
      __half l = __float2half_rn(v - __half2float(h));
      hi[(size_t)c * kdim + k] = h;
      lo[(size_t)c * kdim + k] = l;
    }
    // exact in double; one rounding to fp32 (a subnormal scale_tc only for a clamped column and |scale| < 1)
    scale_tc[c] = (float)((scale ? (double)scale[c] : 1.0) * std::ldexp(1.0, -e));
  }
}

void conv_layer_upload(ConvLayer& L, const float* w, const float* scale, const float* bias) {
  const size_t kdim = (size_t)L.kh * L.kw * L.cin;
  const size_t nw = kdim * L.cout;
  LUMI_CUDA_CHECK(cudaMalloc(&L.w_f32, nw * sizeof(float)));
  LUMI_CUDA_CHECK(cudaMemcpy(L.w_f32, w, nw * sizeof(float), cudaMemcpyHostToDevice));
  const int cpad = cdiv(L.cout, 128) * 128;        // vectors padded so the tensor-core epilogue can use vector loads
  std::vector<float> sc(cpad, 1.f), bi(cpad, 0.f);
  if (scale) std::memcpy(sc.data(), scale, L.cout * sizeof(float));
  if (bias) std::memcpy(bi.data(), bias, L.cout * sizeof(float));
  LUMI_CUDA_CHECK(cudaMalloc(&L.scale, cpad * sizeof(float)));
  LUMI_CUDA_CHECK(cudaMalloc(&L.bias, cpad * sizeof(float)));
  LUMI_CUDA_CHECK(cudaMemcpy(L.scale, sc.data(), cpad * sizeof(float), cudaMemcpyHostToDevice));
  LUMI_CUDA_CHECK(cudaMemcpy(L.bias, bi.data(), cpad * sizeof(float), cudaMemcpyHostToDevice));
  L.tc_ready = false;
  if (L.cin % 64 == 0 && (L.stride == 1 || L.stride == 2)) {
    // [cout_pad][kdim] fp16 hi/lo of w * 2^e[c], zero rows for the padding channels
    L.cout_pad = cdiv(L.cout, 64) * 64;
    if (L.cout_pad > 64 && L.cout_pad % 128 != 0) L.cout_pad = cdiv(L.cout, 128) * 128;
    std::vector<__half> hi((size_t)L.cout_pad * kdim), lo((size_t)L.cout_pad * kdim);
    std::vector<float> sct(L.cout_pad, 0.f);
    std::memset(hi.data(), 0, hi.size() * sizeof(__half));
    std::memset(lo.data(), 0, lo.size() * sizeof(__half));
    pack_conv_weights(w, kdim, L.cout, sc.data(), hi.data(), lo.data(), sct.data());
    LUMI_CUDA_CHECK(cudaMalloc(&L.w_hi, hi.size() * sizeof(__half)));
    LUMI_CUDA_CHECK(cudaMalloc(&L.w_lo, lo.size() * sizeof(__half)));
    LUMI_CUDA_CHECK(cudaMemcpy(L.w_hi, hi.data(), hi.size() * sizeof(__half), cudaMemcpyHostToDevice));
    LUMI_CUDA_CHECK(cudaMemcpy(L.w_lo, lo.data(), lo.size() * sizeof(__half), cudaMemcpyHostToDevice));
    LUMI_CUDA_CHECK(cudaMalloc(&L.scale_tc, L.cout_pad * sizeof(float)));
    LUMI_CUDA_CHECK(cudaMemcpy(L.scale_tc, sct.data(), L.cout_pad * sizeof(float), cudaMemcpyHostToDevice));
    L.tc_ready = true;
  }
}

void conv_layer_free(ConvLayer& L) {
  cudaFree(L.w_f32); cudaFree(L.scale); cudaFree(L.bias);
  cudaFree(L.w_hi); cudaFree(L.w_lo); cudaFree(L.scale_tc);
  L = ConvLayer();
}

}  // namespace lumi
