// Proposal / detection post-processing chains, batched over (image) or (image, class)
// "problems":   decode+filter+clip  ->  sort (score desc, ties: lower index)  ->  gather
//            -> bitmask-matrix NMS (N x ceil(N/64) u64)  ->  serial-scan reduce  ->  gather / top-k.
//
// Replaces  luminoth/models/fasterrcnn/rpn_proposal.py:41-197,
//           luminoth/models/fasterrcnn/rcnn_proposal.py:46-164,
//           luminoth/models/ssd/proposal.py:41-171,
//           luminoth/utils/bbox_transform_tf.py:41-99 (decode / clip_boxes)
// and the TF ops they call (tf.nn.top_k, tf.image.non_max_suppression, tf.boolean_mask).
// Every float expression keeps the reference's evaluation order with explicit
// round-to-nearest intrinsics (no FMA contraction): discrete decisions
// (>=, >, iou > thr) must agree with the fp32 reference bit for bit on equal inputs.
#include "ops.cuh"
#include "conv.cuh"
#include <algorithm>
#include <cstdlib>

namespace lumi {

// ------------------------------------------------------------------ box arithmetic
__device__ __forceinline__ float4 decode_box(float4 roi, float dx, float dy, float dw, float dh, float v0, float v1) {
  const float w = __fadd_rn(__fsub_rn(roi.z, roi.x), 1.f);
  const float h = __fadd_rn(__fsub_rn(roi.w, roi.y), 1.f);
  const float urx = __fadd_rn(roi.x, __fmul_rn(.5f, w));
  const float ury = __fadd_rn(roi.y, __fmul_rn(.5f, h));
  const float px = __fadd_rn(__fmul_rn(__fmul_rn(dx, w), v0), urx);
  const float py = __fadd_rn(__fmul_rn(__fmul_rn(dy, h), v0), ury);
  const float pw = __fmul_rn(expf(__fmul_rn(dw, v1)), w);
  const float ph = __fmul_rn(expf(__fmul_rn(dh, v1)), h);
  float4 o;
  o.x = __fsub_rn(px, __fmul_rn(.5f, pw));
  o.y = __fsub_rn(py, __fmul_rn(.5f, ph));
  o.z = __fsub_rn(__fadd_rn(px, __fmul_rn(.5f, pw)), 1.f);   // "-1. extra" (bbox_transform_tf.py:59-61)
  o.w = __fsub_rn(__fadd_rn(py, __fmul_rn(.5f, ph)), 1.f);
  return o;
}
__device__ __forceinline__ float4 clip_box(float4 b, float im_h, float im_w) {
  const float mw = __fsub_rn(im_w, 1.f), mh = __fsub_rn(im_h, 1.f);
  b.x = fmaxf(fminf(b.x, mw), 0.f);
  b.z = fmaxf(fminf(b.z, mw), 0.f);
  b.y = fmaxf(fminf(b.y, mh), 0.f);
  b.w = fmaxf(fminf(b.w, mh), 0.f);
  return b;
}
__device__ __forceinline__ bool area_positive(float4 b) {
  return __fmul_rn(fmaxf(__fsub_rn(b.z, b.x), 0.f), fmaxf(__fsub_rn(b.w, b.y), 0.f)) > 0.f;
}
// tf.image.non_max_suppression's IoU test on (x1,y1,x2,y2) boxes:  iou(a, b) > thr  with
//   iou = inter / (area_a + area_b - inter)  in fp32, 0 when either area <= 0.
// Bit-identical to evaluating the division, but the IEEE divide only runs for the rare pairs whose
// ratio is within 2^-20 of the threshold (non-overlapping pairs -- the vast majority -- exit first).
__device__ __forceinline__ bool iou_gt(float4 a, float4 b, float thr) {
  const float ymin_i = fminf(a.y, a.w), xmin_i = fminf(a.x, a.z), ymax_i = fmaxf(a.y, a.w), xmax_i = fmaxf(a.x, a.z);
  const float ymin_j = fminf(b.y, b.w), xmin_j = fminf(b.x, b.z), ymax_j = fmaxf(b.y, b.w), xmax_j = fmaxf(b.x, b.z);
  const float area_i = __fmul_rn(__fsub_rn(ymax_i, ymin_i), __fsub_rn(xmax_i, xmin_i));
  const float area_j = __fmul_rn(__fsub_rn(ymax_j, ymin_j), __fsub_rn(xmax_j, xmin_j));
  if (area_i <= 0.f || area_j <= 0.f) return 0.f > thr;
  const float iy0 = fmaxf(ymin_i, ymin_j), ix0 = fmaxf(xmin_i, xmin_j);
  const float iy1 = fminf(ymax_i, ymax_j), ix1 = fminf(xmax_i, xmax_j);
  const float inter = __fmul_rn(fmaxf(__fsub_rn(iy1, iy0), 0.f), fmaxf(__fsub_rn(ix1, ix0), 0.f));
  const float uni = __fsub_rn(__fadd_rn(area_i, area_j), inter);
  if (inter == 0.f && uni > 0.f) return 0.f > thr;              // 0 / positive == +0 exactly
  if (thr > 0.f && uni > 1e-30f && uni < 1e30f && inter < 1e30f) {
    const float t = __fmul_rn(thr, uni);
    if (inter < __fmul_rn(t, 0.99999905f)) return false;        // ratio < thr (1 - 2^-20): RN(ratio) <= thr
    if (inter > __fmul_rn(t, 1.00000095f)) return true;         // ratio > thr (1 + 2^-20): RN(ratio) >  thr
  }
  return __fdiv_rn(inter, uni) > thr;
}

// ------------------------------------------------------------------ workspace
constexpr int CUT_THREADS = 256, CUT_ITEMS = 16, CUT_CHUNK = CUT_THREADS * CUT_ITEMS;   // candidates per cut CTA

// u64 words per mask row; even: mask rows stay 16 B aligned for cp.async.bulk
static int nms_words(int ncap) { return (cdiv(ncap, 64) + 1) & ~1; }

void nms_workspace_alloc(NmsWorkspace& ws, int problems, int cap, int max_out, int ncap) {
  if (ncap <= 0 || ncap > cap) ncap = cap;
  ws.problems = problems; ws.cap = cap; ws.max_out = max_out; ws.ncap = ncap;
  ws.words = nms_words(ncap);
  size_t pc = (size_t)problems * cap;
  size_t pn = (size_t)problems * ncap;
  LUMI_CUDA_CHECK(cudaMalloc(&ws.keys, pc * sizeof(float)));
  LUMI_CUDA_CHECK(cudaMalloc(&ws.boxes, pc * 4 * sizeof(float)));
  LUMI_CUDA_CHECK(cudaMalloc(&ws.order, pc * sizeof(int)));
  LUMI_CUDA_CHECK(cudaMalloc(&ws.nvalid, problems * sizeof(int)));
  LUMI_CUDA_CHECK(cudaMalloc(&ws.sboxes, pn * 4 * sizeof(float)));
  LUMI_CUDA_CHECK(cudaMalloc(&ws.sscores, pn * sizeof(float)));
  LUMI_CUDA_CHECK(cudaMalloc(&ws.mask, pn * ws.words * sizeof(unsigned long long)));
  LUMI_CUDA_CHECK(cudaMalloc(&ws.keep, (size_t)problems * max_out * sizeof(int)));
  LUMI_CUDA_CHECK(cudaMalloc(&ws.nkeep, problems * sizeof(int)));
  LUMI_CUDA_CHECK(cudaMalloc(&ws.sort_tmp, (size_t)problems * 2 * cap * sizeof(unsigned long long)));   // radix ping-pong
  if (ncap >= 4096) {                       // two-phase NMS scratch (see run_nms)
    LUMI_CUDA_CHECK(cudaMalloc(&ws.sboxes2, pn * 4 * sizeof(float)));
    LUMI_CUDA_CHECK(cudaMalloc(&ws.index_map, pn * sizeof(int)));
    LUMI_CUDA_CHECK(cudaMalloc(&ws.alive, pn));
    LUMI_CUDA_CHECK(cudaMalloc(&ws.nvalid2, problems * sizeof(int)));
  }
  if (ncap < cap) {                         // top-k cut scratch (see run_topk_cut)
    ws.cut_blocks = cdiv(cap, CUT_CHUNK);
    LUMI_CUDA_CHECK(cudaMalloc(&ws.cut_hist, (size_t)problems * 4 * 256 * sizeof(unsigned int)));
    LUMI_CUDA_CHECK(cudaMalloc(&ws.cut_counts, (size_t)problems * ws.cut_blocks * sizeof(unsigned long long)));
  }
}
void nms_workspace_free(NmsWorkspace& ws) {
  cudaFree(ws.keys); cudaFree(ws.boxes); cudaFree(ws.order); cudaFree(ws.nvalid); cudaFree(ws.sboxes);
  cudaFree(ws.sscores); cudaFree(ws.mask); cudaFree(ws.keep); cudaFree(ws.nkeep); cudaFree(ws.sort_tmp);
  cudaFree(ws.sboxes2); cudaFree(ws.index_map); cudaFree(ws.alive); cudaFree(ws.nvalid2);
  cudaFree(ws.cut_hist); cudaFree(ws.cut_counts);
  ws = NmsWorkspace();
}

// ------------------------------------------------------------------ sort keys
// key' = bits(score)+1 for valid (score >= 0), 0 for invalid / padding; order: key' desc, index asc.
__device__ __forceinline__ uint32_t score_key(float s) { return (s >= 0.f) ? (__float_as_uint(s) + 1u) : 0u; }

// ------------------------------------------------------------------ LSD radix sort (one CTA per problem)
// Stable 4 x 8-bit passes over (key', index) pairs, key' = ~score_key: ascending key' == descending
// score, stability == "ties -> lower index first" (tf.nn.top_k / NMS candidate order).  Each warp owns a
// contiguous segment and walks it 32 items at a time; 8 ballots (one per digit bit, intersected) give
// every lane the mask of its digit group (rank inside the round = popc below the lane), a per-warp
// digit table in shared memory carries the rank across rounds, and one block-wide exclusive scan in
// digit-major order yields the global offsets.  Two sweeps per pass (count, then scatter) keep register
// use independent of the problem size; data ping-pongs through L2.
// PAIRS: the input is not `keys` but n_all (~key', original index) pairs already in the first ping-pong buffer,
// in ascending index order (the output of the top-k cut); `order` then holds those original indices.
template <int NWARPS, bool PAIRS = false>
__global__ void __launch_bounds__(NWARPS * 32) sort_desc_radix_kernel(const float* __restrict__ keys, int cap,
                                                                     int n_all, const int* __restrict__ n_in,
                                                                     int topn, unsigned long long* __restrict__ tmp,
                                                                     int* __restrict__ order,
                                                                     int* __restrict__ nvalid) {
  constexpr int U = 4;                                   // rounds fetched ahead (independent loads in flight)
  constexpr int BITS = 8, BINS = 256, PASSES = 32 / BITS;
  __shared__ uint32_t hist[NWARPS][BINS];
  __shared__ uint32_t warp_tot[NWARPS];
  __shared__ int s_count;
  const int p = blockIdx.x;
  const int n = n_in ? min(n_in[p], n_all) : n_all;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t lt_mask = (1u << lane) - 1u;
  unsigned long long* bufA = tmp + (size_t)p * 2 * cap;
  unsigned long long* bufB = bufA + cap;
  const int seg = ((n + NWARPS - 1) / NWARPS + 31) & ~31;       // items per warp, multiple of 32
  const int lo = warp * seg, hi = min(n, lo + seg);
  if (threadIdx.x == 0) s_count = 0;
  __syncthreads();
  int local_valid = 0;
  // mask of the lanes (among the active ones) that hold the same digit as this lane
  auto group_mask = [&](uint32_t digit, bool act) -> uint32_t {
    uint32_t mine = __ballot_sync(0xffffffffu, act);
#pragma unroll
    for (int b = 0; b < BITS; ++b) {
      const uint32_t vote = __ballot_sync(0xffffffffu, (digit >> b) & 1u);
      mine &= ((digit >> b) & 1u) ? vote : ~vote;
    }
    return mine;
  };
  for (int pass = 0; pass < PASSES; ++pass) {
    const int shift = pass * BITS;
    const unsigned long long* src = (pass & 1) ? bufB : bufA;
    unsigned long long* dst = (pass & 1) ? bufA : bufB;
    auto fetch = [&](int i) -> unsigned long long {       // (key', index) of item i of this pass' input
      if (i >= hi) return 0ull;
      if (pass == 0 && !PAIRS) {
        const uint32_t k = score_key(keys[(size_t)p * cap + i]);
        return ((unsigned long long)(~k) << 32) | (uint32_t)i;
      }
      return src[i];
    };
    for (int d = lane; d < BINS; d += 32) hist[warp][d] = 0;
    __syncwarp();
    // ---- sweep 1: per-warp digit counts
    for (int base = lo; base < hi; base += 32 * U) {
      unsigned long long v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) v[u] = fetch(base + u * 32 + lane);
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const bool act = base + u * 32 + lane < hi;
        if (pass == 0 && act) local_valid += (uint32_t)(v[u] >> 32) != 0xFFFFFFFFu;
        const uint32_t digit = (uint32_t)(v[u] >> (32 + shift)) & (BINS - 1);
        const uint32_t peers = group_mask(digit, act);
        if (act && (peers & lt_mask) == 0) hist[warp][digit] += __popc(peers);   // leader of its digit group
        __syncwarp();
      }
    }
    __syncthreads();
    // ---- exclusive scan in digit-major order: entry j = d * NWARPS + w, EPT entries per thread
    {
      constexpr int EPT = BINS / 32;                      // BINS * NWARPS / (32 * NWARPS)
      uint32_t v[EPT], sum = 0;
#pragma unroll
      for (int e = 0; e < EPT; ++e) {
        const int j = threadIdx.x * EPT + e;
        v[e] = hist[j % NWARPS][j / NWARPS];
        sum += v[e];
      }
      uint32_t incl = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
      }
      if (lane == 31) warp_tot[warp] = incl;
      __syncthreads();
      uint32_t wbase = 0;
      for (int w = 0; w < warp; ++w) wbase += warp_tot[w];
      uint32_t run = wbase + incl - sum;
#pragma unroll
      for (int e = 0; e < EPT; ++e) {
        const int j = threadIdx.x * EPT + e;
        hist[j % NWARPS][j / NWARPS] = run;
        run += v[e];
      }
    }
    __syncthreads();
    // ---- sweep 2: stable scatter
    for (int base = lo; base < hi; base += 32 * U) {
      unsigned long long v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) v[u] = fetch(base + u * 32 + lane);
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const bool act = base + u * 32 + lane < hi;
        const uint32_t digit = (uint32_t)(v[u] >> (32 + shift)) & (BINS - 1);
        const uint32_t peers = group_mask(digit, act);
        if (act) {
          const uint32_t old = hist[warp][digit];
          const uint32_t pos = old + __popc(peers & lt_mask);
          __syncwarp(__activemask());
          if ((peers & lt_mask) == 0) hist[warp][digit] = old + __popc(peers);
          if (pass < PASSES - 1) {
            dst[pos] = v[u];
          } else if ((int)pos < topn && (uint32_t)(v[u] >> 32) != 0xFFFFFFFFu) {
            order[(size_t)p * cap + pos] = (int)(uint32_t)v[u];                 // final pass: sorted indices
          }
        }
        __syncwarp();
      }
    }
    __syncthreads();
  }
  atomicAdd(&s_count, local_valid);
  __syncthreads();
  if (threadIdx.x == 0) nvalid[p] = min(s_count, topn);
}

// keys: [problems][cap]; the first n_all (<= cap) entries of each problem are sorted
static void run_sort(const float* keys, int problems, int cap, int n_all, const int* n_in, int topn, int* order,
                     int* nvalid, unsigned long long* tmp, cudaStream_t st) {
  if (!problems || !cap || !n_all) return;
  LUMI_REQUIRE(tmp != nullptr && n_all <= cap, "sort: missing scratch");
  if (n_all > 4096)
    sort_desc_radix_kernel<32><<<problems, 1024, 0, st>>>(keys, cap, n_all, n_in, topn, tmp, order, nvalid);
  else
    sort_desc_radix_kernel<8><<<problems, 256, 0, st>>>(keys, cap, n_all, n_in, topn, tmp, order, nvalid);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
}

// ------------------------------------------------------------------ top-k cut ahead of the sort
// When a problem has many more candidates than the sort keeps (the RPN at output_stride 8 or 4 has 115 200 or
// 460 800 anchors per 600x1024 image against pre_nms_top_n = 12 000), the whole GPU first selects the k largest
// (key', index) pairs and the one-CTA sort then orders only those:
//   1. radix select, most significant 8-bit digit of key' first: in each of 4 rounds every CTA histograms those of
//      its candidates that carry the prefix selected so far.  The k-th largest key' T and the count of keys above it
//      follow from the histograms alone (cut_select, recomputed by every CTA that needs them);
//   2. stable compaction: every candidate with key' > T plus the first k - count(key' > T) with key' == T, in
//      ascending index order, written as (~key', index) pairs through per-CTA counts and an exclusive scan;
//   3. the radix sort of those k pairs.  It is stable and its input is in index order, so `order` and `nvalid` are
//      the ones the sort of all candidates gives, ties included.
// The grids depend on the candidate count only, so the chain is captured into CUDA graphs like the rest.

// Radix-select state after `rounds` digits, computed by one warp (every lane gets it): prefix = the top 8 * rounds
// bits of the k-th largest key', above = the count of keys whose top bits exceed that prefix.
__device__ __forceinline__ void cut_select(const unsigned int* __restrict__ hist, int rounds, uint32_t k,
                                           uint32_t& prefix, uint32_t& above) {
  const int lane = threadIdx.x & 31;
  prefix = 0; above = 0;
  uint32_t rem = k;                                   // rank of the wanted key among those carrying the prefix
  for (int r = 0; r < rounds; ++r) {
    uint32_t c[8], sum = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) { c[j] = hist[r * 256 + 255 - (lane * 8 + j)]; sum += c[j]; }   // digits descending
    uint32_t incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    const int src = __ffs(__ballot_sync(0xffffffffu, incl >= rem)) - 1;
    uint32_t acc = incl - sum, digit = 0;
    bool found = false;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (!found && acc + c[j] >= rem) { digit = 255 - (lane * 8 + j); found = true; }
      if (!found) acc += c[j];
    }
    digit = __shfl_sync(0xffffffffu, digit, src);
    acc = __shfl_sync(0xffffffffu, acc, src);
    rem -= acc; above += acc;
    prefix = (prefix << 8) | digit;
  }
}

// exclusive block-wide scan of v (CUT_THREADS threads); total = the sum over the block
__device__ __forceinline__ unsigned long long cut_block_scan(unsigned long long v, unsigned long long* s_warp,
                                                             unsigned long long& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  unsigned long long wbase = 0;
  total = 0;
#pragma unroll
  for (int w = 0; w < CUT_THREADS / 32; ++w) {
    if (w < warp) wbase += s_warp[w];
    total += s_warp[w];
  }
  __syncthreads();
  return wbase + incl - v;
}

// round `round` of the select: hist[p][round][d] += candidates carrying the selected prefix, by their next digit d
__global__ void __launch_bounds__(CUT_THREADS) cut_hist_kernel(const float* __restrict__ keys, int cap, int n, int k,
                                                               int round, unsigned int* __restrict__ hist) {
  __shared__ unsigned int sh[256];
  __shared__ uint32_t s_prefix;
  const int p = blockIdx.y;
  unsigned int* H = hist + (size_t)p * 4 * 256;
  sh[threadIdx.x] = 0;
  if (threadIdx.x < 32) {
    uint32_t prefix, above;
    cut_select(H, round, (uint32_t)k, prefix, above);
    if (threadIdx.x == 0) s_prefix = prefix;
  }
  __syncthreads();
  const uint32_t prefix = s_prefix;
  const int shift = 24 - 8 * round;
  const float* K = keys + (size_t)p * cap;
  const int base = blockIdx.x * CUT_CHUNK;
  const uint32_t lt_mask = (1u << (threadIdx.x & 31)) - 1u;
#pragma unroll 4
  for (int it = 0; it < CUT_ITEMS; ++it) {
    const int i = base + it * CUT_THREADS + threadIdx.x;
    const uint32_t key = i < n ? score_key(K[i]) : 0u;
    const bool match = i < n && (round == 0 || (key >> (shift + 8)) == prefix);
    const uint32_t digit = (key >> shift) & 255u;
    const uint32_t peers = __match_any_sync(0xffffffffu, match ? digit : 256u);   // one shared atomic per digit
    if (match && (peers & lt_mask) == 0) atomicAdd(&sh[digit], (unsigned int)__popc(peers));
  }
  __syncthreads();
  if (sh[threadIdx.x]) atomicAdd(&H[round * 256 + threadIdx.x], sh[threadIdx.x]);
}

// per-CTA counts of the candidates above the k-th key' T (high word) and equal to it (low word)
__global__ void __launch_bounds__(CUT_THREADS) cut_count_kernel(const float* __restrict__ keys, int cap, int n, int k,
                                                                const unsigned int* __restrict__ hist,
                                                                unsigned long long* __restrict__ counts, int nblk) {
  __shared__ uint32_t s_t;
  __shared__ unsigned long long s_warp[CUT_THREADS / 32];
  const int p = blockIdx.y;
  if (threadIdx.x < 32) {
    uint32_t t, above;
    cut_select(hist + (size_t)p * 4 * 256, 4, (uint32_t)k, t, above);
    if (threadIdx.x == 0) s_t = t;
  }
  __syncthreads();
  const uint32_t T = s_t;
  const float* K = keys + (size_t)p * cap;
  const int base = blockIdx.x * CUT_CHUNK;
  unsigned long long c = 0;
#pragma unroll 4
  for (int it = 0; it < CUT_ITEMS; ++it) {
    const int i = base + it * CUT_THREADS + threadIdx.x;
    if (i < n) {
      const uint32_t key = score_key(K[i]);
      c += key > T ? (1ull << 32) : (key == T ? 1ull : 0ull);
    }
  }
  unsigned long long total;
  cut_block_scan(c, s_warp, total);
  if (threadIdx.x == 0) counts[(size_t)p * nblk + blockIdx.x] = total;
}

// stable compaction of the k selected candidates into (~key', index) pairs at out[p][0, k)
__global__ void __launch_bounds__(CUT_THREADS) cut_scatter_kernel(const float* __restrict__ keys, int cap, int n, int k,
                                                                  const unsigned int* __restrict__ hist,
                                                                  const unsigned long long* __restrict__ counts,
                                                                  int nblk, unsigned long long* __restrict__ tmp) {
  __shared__ uint32_t s_t, s_above;
  __shared__ unsigned long long s_warp[CUT_THREADS / 32];
  const int p = blockIdx.y;
  if (threadIdx.x < 32) {
    uint32_t t, above;
    cut_select(hist + (size_t)p * 4 * 256, 4, (uint32_t)k, t, above);
    if (threadIdx.x == 0) { s_t = t; s_above = above; }
  }
  unsigned long long before = 0;                       // counts of the CTAs before this one
  for (int j = threadIdx.x; j < blockIdx.x; j += CUT_THREADS) before += counts[(size_t)p * nblk + j];
  unsigned long long prev;
  cut_block_scan(before, s_warp, prev);                // also orders s_t / s_above before their reads
  const uint32_t T = s_t, need_eq = (uint32_t)k - s_above;
  const float* K = keys + (size_t)p * cap;
  const int first = blockIdx.x * CUT_CHUNK + threadIdx.x * CUT_ITEMS;   // this thread's contiguous run
  uint32_t key[CUT_ITEMS];
  unsigned long long c = 0;
#pragma unroll
  for (int j = 0; j < CUT_ITEMS; ++j) {
    key[j] = first + j < n ? score_key(K[first + j]) : 0u;
    if (first + j < n) c += key[j] > T ? (1ull << 32) : (key[j] == T ? 1ull : 0ull);
  }
  unsigned long long total;
  const unsigned long long start = prev + cut_block_scan(c, s_warp, total);
  uint32_t gt = (uint32_t)(start >> 32), eq = (uint32_t)start;
  unsigned long long* out = tmp + (size_t)p * 2 * cap;
#pragma unroll
  for (int j = 0; j < CUT_ITEMS; ++j) {
    if (first + j >= n) break;
    const unsigned long long pair = ((unsigned long long)(~key[j]) << 32) | (uint32_t)(first + j);
    if (key[j] > T) {
      out[gt + min(eq, need_eq)] = pair;
      ++gt;
    } else if (key[j] == T) {
      if (eq < need_eq) out[gt + eq] = pair;
      ++eq;
    }
  }
}

// The sort of run_sort over n candidates per problem when only the first k (<= n) are kept; same outputs.
static void run_topk_cut(const float* keys, int problems, int cap, int n, int k, int* order, int* nvalid,
                         const NmsWorkspace& ws, cudaStream_t st) {
  const int nblk = cdiv(n, CUT_CHUNK);
  LUMI_REQUIRE(ws.cut_hist && nblk <= ws.cut_blocks && k <= n && n <= cap, "top-k cut: missing scratch");
  LUMI_CUDA_CHECK(cudaMemsetAsync(ws.cut_hist, 0, (size_t)problems * 4 * 256 * sizeof(unsigned int), st));
  const dim3 g(nblk, problems);
  for (int r = 0; r < 4; ++r) {
    cut_hist_kernel<<<g, CUT_THREADS, 0, st>>>(keys, cap, n, k, r, ws.cut_hist);
    count_launch();
    LUMI_CUDA_CHECK(cudaGetLastError());
  }
  cut_count_kernel<<<g, CUT_THREADS, 0, st>>>(keys, cap, n, k, ws.cut_hist, ws.cut_counts, nblk);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
  cut_scatter_kernel<<<g, CUT_THREADS, 0, st>>>(keys, cap, n, k, ws.cut_hist, ws.cut_counts, nblk, ws.sort_tmp);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
  if (k > 4096)
    sort_desc_radix_kernel<32, true><<<problems, 1024, 0, st>>>(keys, cap, k, nullptr, k, ws.sort_tmp, order, nvalid);
  else
    sort_desc_radix_kernel<8, true><<<problems, 256, 0, st>>>(keys, cap, k, nullptr, k, ws.sort_tmp, order, nvalid);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
}

// ------------------------------------------------------------------ gather sorted
__global__ void gather_sorted_kernel(const float* __restrict__ boxes, const float* __restrict__ keys,
                                     const int* __restrict__ order, const int* __restrict__ nvalid, int cap, int ncap,
                                     float* __restrict__ sboxes, float* __restrict__ sscores) {
  const int p = blockIdx.y;
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= nvalid[p]) return;
  const size_t src = (size_t)p * cap + order[(size_t)p * cap + r];
  const size_t dst = (size_t)p * ncap + r;
  reinterpret_cast<float4*>(sboxes)[dst] = reinterpret_cast<const float4*>(boxes)[src];
  sscores[dst] = keys[src];
}

// ------------------------------------------------------------------ NMS bitmask matrix
// Normalised box (min/max corners + area) exactly as TF's IOU() computes them.
struct NBox { float ymin, xmin, ymax, xmax, area; };
__device__ __forceinline__ NBox normalise_box(float4 b) {
  NBox n;
  n.ymin = fminf(b.y, b.w); n.xmin = fminf(b.x, b.z); n.ymax = fmaxf(b.y, b.w); n.xmax = fmaxf(b.x, b.z);
  n.area = __fmul_rn(__fsub_rn(n.ymax, n.ymin), __fsub_rn(n.xmax, n.xmin));
  return n;
}
// Same decision as iou_gt() on pre-normalised boxes, for thr >= 0, with the cheap rejections first:
// no x- or y-overlap => inter == 0 => iou == 0 => not > thr.
__device__ __forceinline__ bool iou_gt_norm(const NBox& a, const NBox& b, float thr) {
  const float ix0 = fmaxf(a.xmin, b.xmin), ix1 = fminf(a.xmax, b.xmax);
  const float dx = __fsub_rn(ix1, ix0);
  if (!(dx > 0.f)) return false;
  const float iy0 = fmaxf(a.ymin, b.ymin), iy1 = fminf(a.ymax, b.ymax);
  const float dy = __fsub_rn(iy1, iy0);
  if (!(dy > 0.f)) return false;
  if (a.area <= 0.f || b.area <= 0.f) return false;
  const float inter = __fmul_rn(dy, dx);              // == max(dy,0)*max(dx,0) here
  const float uni = __fsub_rn(__fadd_rn(a.area, b.area), inter);
  if (inter == 0.f && uni > 0.f) return false;        // product underflowed to 0: iou == 0
  if (thr > 0.f && uni > 1e-30f && uni < 1e30f && inter < 1e30f) {
    const float t = __fmul_rn(thr, uni);
    if (inter < __fmul_rn(t, 0.99999905f)) return false;
    if (inter > __fmul_rn(t, 1.00000095f)) return true;
  }
  return __fdiv_rn(inter, uni) > thr;
}

__device__ __noinline__ bool iou_exact_gt(float inter, float uni, float thr) {
  return __fdiv_rn(inter, uni) > thr;                          // inter > 0, uni finite here; NaN/inf compare false
}

// grid (pair slot, problem); 64 threads; a block walks the upper-triangle (row block, col block) pairs
// of its problem with a grid stride, so launch cost follows the live candidate count, not the capacity.
// thr > 0 (every configuration in practice): branch-free inner loop -- the 2^-20 margin test decides
// almost every pair, the IEEE divide only runs for ratios within the margin of the threshold.
__global__ void __launch_bounds__(64) nms_mask_kernel(const float* __restrict__ sboxes, const int* __restrict__ nvalid,
                                                      int cap, int words, float thr,
                                                      unsigned long long* __restrict__ mask, int limit) {
  const int p = blockIdx.y;
  const int n = min(nvalid[p], limit);                // limit: only the first `limit` candidates (two-phase NMS)
  const int nw = (n + 63) >> 6;
  const long npairs = (long)nw * (nw + 1) / 2;
  __shared__ float4 cbox[64];        // raw boxes (generic path)
  __shared__ float4 cmm[64];         // (xmin, ymin, xmax, ymax)
  __shared__ float carea[64];        // area, or -1 for columns past the end
  const float4* B = reinterpret_cast<const float4*>(sboxes) + (size_t)p * cap;
  const int t = threadIdx.x;
  // pair index -> (rb, cb >= rb): row rb starts at rb*(2nw-rb+1)/2; decoded once, then advanced incrementally
  long pr = blockIdx.x;
  int rb = 0;
  if (pr < npairs) {
    const double disc = (2.0 * nw + 1.0) * (2.0 * nw + 1.0) - 8.0 * (double)pr;
    rb = (int)(((2.0 * nw + 1.0) - sqrt(disc)) * 0.5);
    if (rb < 0) rb = 0;
    if (rb > nw - 1) rb = nw - 1;
    while ((long)rb * (2 * nw - rb + 1) / 2 > pr) --rb;
    while ((long)(rb + 1) * (2 * nw - rb) / 2 <= pr) ++rb;
  }
  for (; pr < npairs; pr += gridDim.x) {
    while ((long)(rb + 1) * (2 * nw - rb) / 2 <= pr) ++rb;
    const int cb = rb + (int)(pr - (long)rb * (2 * nw - rb + 1) / 2);
    __syncthreads();
    {
      const bool in = cb * 64 + t < n;
      const float4 c = in ? B[cb * 64 + t] : make_float4(0.f, 0.f, 0.f, 0.f);
      const NBox nb = normalise_box(c);
      cbox[t] = c;
      cmm[t] = make_float4(nb.xmin, nb.ymin, nb.xmax, nb.ymax);
      carea[t] = (in && nb.area > 0.f) ? nb.area : INFINITY;   // inf union -> never > thr (matches iou == 0)
    }
    __syncthreads();
    const int i = rb * 64 + t;
    if (i >= n) continue;
    const float4 bi = B[i];
    unsigned long long bits = 0ull;
    if (thr > 0.f) {
      const NBox ni = normalise_box(bi);
      uint32_t lo = 0u, hi = 0u, alo = 0u, ahi = 0u;
      if (ni.area > 0.f) {
        // branch-free: `lo/hi` collect the pairs that are certainly above the threshold (ratio > thr (1 + 2^-20)),
        // `alo/ahi` the ones inside the +-2^-20 margin; only those (practically never) take the exact IEEE divide
        // afterwards.  The sign of fma(-t, union, inter) is the sign of the exact difference.
        const float thr_hi = __fmul_rn(thr, 1.00000095f), thr_lo = __fmul_rn(thr, 0.99999905f);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          uint32_t s_bits = 0u, m_bits = 0u;
#pragma unroll
          for (int jj = 0; jj < 32; ++jj) {
            const int j = h * 32 + jj;
            const float4 c = cmm[j];
            const float ca = carea[j];                         // +inf for columns that can never suppress
            const float dx = __fsub_rn(fminf(ni.xmax, c.z), fmaxf(ni.xmin, c.x));
            const float dy = __fsub_rn(fminf(ni.ymax, c.w), fmaxf(ni.ymin, c.y));
            const float inter = __fmul_rn(fmaxf(dy, 0.f), fmaxf(dx, 0.f));
            const float uni = __fsub_rn(__fadd_rn(ni.area, ca), inter);
            if (fmaf(-thr_hi, uni, inter) > 0.f) s_bits |= 1u << jj;
            if (fmaf(-thr_lo, uni, inter) >= 0.f) m_bits |= 1u << jj;   // includes the sure ones; NaN -> false
          }
          if (h == 0) { lo = s_bits; alo = m_bits; } else { hi = s_bits; ahi = m_bits; }
        }
      }
      bits = ((unsigned long long)hi << 32) | lo;
      unsigned long long amb = (((unsigned long long)ahi << 32) | alo) & ~bits;
      while (amb) {                                             // ratios within 2^-20 of the threshold
        const int j = __ffsll((long long)amb) - 1;
        amb &= amb - 1ull;
        const float4 c = cmm[j];
        const float dx = __fsub_rn(fminf(ni.xmax, c.z), fmaxf(ni.xmin, c.x));
        const float dy = __fsub_rn(fminf(ni.ymax, c.w), fmaxf(ni.ymin, c.y));
        const float inter = __fmul_rn(fmaxf(dy, 0.f), fmaxf(dx, 0.f));
        const float uni = __fsub_rn(__fadd_rn(ni.area, carea[j]), inter);
        if (iou_exact_gt(inter, uni, thr)) bits |= 1ull << j;
      }
      if (cb == rb) bits &= ~((2ull << t) - 1ull);            // only columns > i
    } else {                                                  // thr <= 0: generic exact path
      const int jmax = min(64, n - cb * 64);
      for (int j = 0; j < jmax; ++j) {
        const int col = cb * 64 + j;
        if (col > i && iou_gt(bi, cbox[j], thr)) bits |= 1ull << j;
      }
    }
    mask[((size_t)p * cap + i) * words + cb] = bits;
  }
}

// serial-scan reduce: one CTA per problem walks 64-box chunks in score order.  Per chunk: thread 0
// resolves the 64x64 diagonal word greedily (find-first-set over the still-alive bits, so the loop runs
// once per KEPT box), then all threads OR the kept rows into the running "removed" words.  The next
// chunk's diagonal words do not depend on the removal state, so they are prefetched during the OR phase.
__global__ void __launch_bounds__(256) nms_scan_kernel(const unsigned long long* __restrict__ mask,
                                                       const int* __restrict__ nvalid, int cap, int words,
                                                       int max_out, int* __restrict__ keep, int* __restrict__ nkeep) {
  extern __shared__ unsigned long long removed[];     // [words]
  __shared__ unsigned long long diag[2][64];
  __shared__ int s_kept[64];
  __shared__ int s_nk, s_total, s_done;
  const int p = blockIdx.x;
  const int n = nvalid[p];
  const int nw = (n + 63) >> 6;
  const unsigned long long* M = mask + (size_t)p * cap * words;
  for (int w = threadIdx.x; w < words; w += blockDim.x) removed[w] = 0ull;
  if (threadIdx.x == 0) { s_total = 0; s_done = (max_out <= 0 || n == 0) ? 1 : 0; }
  if (threadIdx.x < 64) diag[0][threadIdx.x] = (int)threadIdx.x < n ? M[(size_t)threadIdx.x * words] : 0ull;
  __syncthreads();
  const bool done0 = s_done != 0;                      // read by everyone before thread 0 can change it
  for (int c = 0; c < nw && !done0; ++c) {
    const unsigned long long* dg = diag[c & 1];
    if (threadIdx.x == 0) {
      unsigned long long cur = removed[c];
      const int lim = min(64, n - c * 64);
      const unsigned long long vmask = lim == 64 ? ~0ull : ((1ull << lim) - 1ull);
      unsigned long long avail = ~cur & vmask;
      int nk = 0, total = s_total;
      while (avail) {
        const int b = __ffsll((long long)avail) - 1;
        s_kept[nk++] = b;
        keep[(size_t)p * max_out + total] = c * 64 + b;
        if (++total >= max_out) { s_done = 1; break; }
        cur |= dg[b];
        avail = ~cur & vmask & ~((2ull << b) - 1ull);      // alive bits above b
      }
      s_nk = nk; s_total = total;
    }
    __syncthreads();
    if (s_done) break;
    unsigned long long next_diag = 0ull;               // prefetch (independent of the removal state)
    if (threadIdx.x < 64) {
      const int row = (c + 1) * 64 + threadIdx.x;
      if (row < n) next_diag = M[(size_t)row * words + (c + 1)];
    }
    const int nk = s_nk;
    for (int w = c + 1 + threadIdx.x; w < nw; w += blockDim.x) {
      unsigned long long acc = removed[w];
      int i = 0;
      for (; i + 4 <= nk; i += 4) {
        const unsigned long long a0 = M[(size_t)(c * 64 + s_kept[i]) * words + w];
        const unsigned long long a1 = M[(size_t)(c * 64 + s_kept[i + 1]) * words + w];
        const unsigned long long a2 = M[(size_t)(c * 64 + s_kept[i + 2]) * words + w];
        const unsigned long long a3 = M[(size_t)(c * 64 + s_kept[i + 3]) * words + w];
        acc |= (a0 | a1) | (a2 | a3);
      }
      for (; i < nk; ++i) acc |= M[(size_t)(c * 64 + s_kept[i]) * words + w];
      removed[w] = acc;
    }
    if (threadIdx.x < 64) diag[(c + 1) & 1][threadIdx.x] = next_diag;
    __syncthreads();
  }
  if (threadIdx.x == 0) nkeep[p] = s_total;
}

// Staged variant: the 64 mask rows of chunk c+1 (one contiguous block) are bulk-copied
// (cp.async.bulk -> mbarrier) into shared memory while chunk c is resolved, so the greedy walk never
// waits on an L2 round trip: diag resolve and the OR of the kept rows both read shared memory.
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"((uint64_t)src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// limit: scan only the first `limit` candidates.  base_count / index_map (second phase of the two-phase NMS): the
// keep list already holds base_count[p] entries, and candidate r of THIS scan is index_map[p][r] of the original list.
__global__ void __launch_bounds__(256) nms_scan_staged_kernel(const unsigned long long* __restrict__ mask,
                                                              const int* __restrict__ nvalid, int cap, int words,
                                                              int max_out, int* __restrict__ keep,
                                                              int* __restrict__ nkeep, int limit,
                                                              const int* __restrict__ base_count,
                                                              const int* __restrict__ index_map) {
  extern __shared__ __align__(16) unsigned long long sm64[];
  unsigned long long* removed = sm64;                         // [words]
  unsigned long long* buf = sm64 + words;                     // [2][64][words]
  __shared__ __align__(8) uint64_t full_bar[2];
  __shared__ int s_kept[64];
  __shared__ int s_nk, s_total, s_done;
  const int p = blockIdx.x;
  const int n = min(nvalid[p], limit);
  const int nw = (n + 63) >> 6;
  const unsigned long long* M = mask + (size_t)p * cap * words;
  const int* imap = index_map ? index_map + (size_t)p * cap : nullptr;
  for (int w = threadIdx.x; w < words; w += blockDim.x) removed[w] = 0ull;
  if (threadIdx.x == 0) {
    s_total = base_count ? base_count[p] : 0;
    s_done = (max_out <= 0 || n == 0 || s_total >= max_out) ? 1 : 0;
    mbar_init(&full_bar[0], 1); mbar_init(&full_bar[1], 1);
    fence_mbar_init();
  }
  __syncthreads();
  auto issue = [&](int c) {             // rows of chunk c are contiguous in the mask: one bulk copy -> buf[c & 1]
    const int rows = min(64, n - c * 64);
    const uint32_t bytes = (uint32_t)rows * (uint32_t)words * 8u;
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(&full_bar[c & 1], bytes);
      bulk_g2s(buf + (size_t)(c & 1) * 64 * words, M + (size_t)c * 64 * words, bytes, &full_bar[c & 1]);
    }
  };
  const bool done0 = s_done != 0;
  int last_issued = -1, last_waited = -1;                     // uniform across the CTA
  if (!done0 && nw > 0) {
    if (threadIdx.x < 64) issue(0);
    last_issued = 0;
  }
  for (int c = 0; c < nw && !done0; ++c) {
    mbar_wait(&full_bar[c & 1], ((uint32_t)c >> 1) & 1u);
    last_waited = c;
    if (c + 1 < nw) {                                         // buf[(c+1)&1] was last read in iteration c-1
      if (threadIdx.x < 64) { fence_proxy_async(); issue(c + 1); }
      last_issued = c + 1;
    }
    const unsigned long long* rows = buf + (size_t)(c & 1) * 64 * words;
    if (threadIdx.x == 0) {
      unsigned long long cur = removed[c];
      const int lim = min(64, n - c * 64);
      const unsigned long long vmask = lim == 64 ? ~0ull : ((1ull << lim) - 1ull);
      unsigned long long avail = ~cur & vmask;
      int nk = 0, total = s_total;
      while (avail) {
        const int b = __ffsll((long long)avail) - 1;
        s_kept[nk++] = b;
        keep[(size_t)p * max_out + total] = imap ? imap[c * 64 + b] : c * 64 + b;
        if (++total >= max_out) { s_done = 1; break; }
        cur |= rows[(size_t)b * words + c];
        avail = ~cur & vmask & ~((2ull << b) - 1ull);
      }
      s_nk = nk; s_total = total;
    }
    __syncthreads();
    if (s_done) break;
    const int nk = s_nk;
    for (int w = c + 1 + threadIdx.x; w < nw; w += blockDim.x) {
      unsigned long long acc = removed[w];
      for (int i = 0; i < nk; ++i) acc |= rows[(size_t)s_kept[i] * words + w];
      removed[w] = acc;
    }
    __syncthreads();
  }
  // never exit with a bulk copy still landing in this CTA's shared memory
  if (last_issued > last_waited) mbar_wait(&full_bar[last_issued & 1], ((uint32_t)last_issued >> 1) & 1u);
  if (threadIdx.x == 0) nkeep[p] = s_total;
}

// ---- two-phase ("lazy") NMS for long candidate lists.
// The bit-mask matrix costs N^2/2 pair tests although the greedy scan only ever reads the rows of KEPT boxes.  Phase 1
// resolves the first R1 candidates exactly as before (mask + scan on an R1 x R1 triangle).  A pre-filter then tests
// every later candidate against those kept boxes only (k1 x (N - R1) pairs) and the survivors -- the only later
// candidates that can still be kept -- are compacted in order; phase 2 runs mask + scan on the survivors and appends to
// the keep list through the index map.  Kept set and order are identical to the one-phase result (a candidate
// suppressed by a phase-1 keeper is suppressed in the greedy walk as well, and suppression among later candidates
// involves survivors only); the pair tests drop from N^2/2 to R1^2/2 + k1 (N - R1) + S^2/2.
constexpr int NMS_LAZY_R1 = 2048;
constexpr int NMS_LAZY_MIN = 4096;

// shared memory of nms_scan_staged_kernel: the removed words plus two chunks of 64 mask rows
static size_t staged_scan_smem(int words) { return ((size_t)words + 2 * 64 * (size_t)words) * sizeof(unsigned long long); }
constexpr size_t NMS_STAGED_SMEM_MAX = 200 * 1024;

int nms_path(int problems, int ncap, float thr) {
  if (staged_scan_smem(nms_words(ncap)) > NMS_STAGED_SMEM_MAX) return NMS_PATH_UNSTAGED;
  // two-phase when the mask kernel is a full-GPU kernel (several long lists at once): it shortens the step at
  // batch 8, but its longer kernel chain adds latency when one or two images are in flight.  LUMI_NMS_LAZY=0 / 1 forces it off / on.
  static const int lazy_env = [] { const char* e = getenv("LUMI_NMS_LAZY"); return e ? (atoi(e) != 0 ? 1 : 0) : -1; }();
  const bool lazy_ok = ncap >= NMS_LAZY_MIN && thr > 0.f && thr < INFINITY;
  return lazy_ok && (lazy_env == 1 || (lazy_env < 0 && problems >= 3)) ? NMS_PATH_TWO_PHASE : NMS_PATH_STAGED;
}

__global__ void __launch_bounds__(256) nms_prefilter_kernel(const float* __restrict__ sboxes,
                                                            const int* __restrict__ nvalid, int cap, float thr,
                                                            const int* __restrict__ keep, const int* __restrict__ nkeep,
                                                            int max_out, int r1, unsigned char* __restrict__ alive) {
  const int p = blockIdx.y;
  const int n = nvalid[p];
  const int k1 = nkeep[p];
  const int j = r1 + blockIdx.x * blockDim.x + threadIdx.x;
  if (r1 + (int)(blockIdx.x * blockDim.x) >= n || k1 >= max_out) return;        // whole block: nothing left to decide
  __shared__ NBox kb[256];
  const float4* B = reinterpret_cast<const float4*>(sboxes) + (size_t)p * cap;
  const bool mine = j < n;
  const NBox me = normalise_box(mine ? B[j] : make_float4(0.f, 0.f, 0.f, 0.f));
  bool dead = false;
  for (int base = 0; base < k1; base += 256) {
    __syncthreads();
    if (base + (int)threadIdx.x < k1) kb[threadIdx.x] = normalise_box(B[keep[(size_t)p * max_out + base + threadIdx.x]]);
    __syncthreads();
    const int m = min(256, k1 - base);
    if (mine && !dead)
      for (int i = 0; i < m; ++i)
        if (iou_gt_norm(kb[i], me, thr)) { dead = true; break; }
  }
  if (mine) alive[(size_t)p * cap + j] = dead ? 0 : 1;
}

// stable compaction of the survivors of candidates [r1, n): one CTA per problem
__global__ void __launch_bounds__(1024) nms_compact_kernel(const float* __restrict__ sboxes, const int* __restrict__ nvalid,
                                                           int cap, const unsigned char* __restrict__ alive,
                                                           const int* __restrict__ nkeep, int max_out, int r1,
                                                           float* __restrict__ sboxes2, int* __restrict__ index_map,
                                                           int* __restrict__ nvalid2) {
  const int p = blockIdx.x;
  const int n = nvalid[p];
  __shared__ int warp_tot[32];
  __shared__ int s_base;
  if (threadIdx.x == 0) s_base = 0;
  const bool finished = nkeep[p] >= max_out;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float4* B = reinterpret_cast<const float4*>(sboxes) + (size_t)p * cap;
  float4* B2 = reinterpret_cast<float4*>(sboxes2) + (size_t)p * cap;
  __syncthreads();
  if (!finished)
    for (int base = r1; base < n; base += 1024) {       // uniform trip count
      const int j = base + threadIdx.x;
      const int a = (j < n && alive[(size_t)p * cap + j]) ? 1 : 0;
      const unsigned bal = __ballot_sync(0xffffffffu, a);
      const int rank = __popc(bal & ((1u << lane) - 1u));
      if (lane == 0) warp_tot[warp] = __popc(bal);
      __syncthreads();
      int woff = 0, tot = 0;
      for (int w = 0; w < 32; ++w) { const int t = warp_tot[w]; if (w < warp) woff += t; tot += t; }
      const int start = s_base;
      if (a) {
        const int dst = start + woff + rank;
        B2[dst] = B[j];
        index_map[(size_t)p * cap + dst] = j;
      }
      __syncthreads();
      if (threadIdx.x == 0) s_base = start + tot;
      __syncthreads();
    }
  if (threadIdx.x == 0) nvalid2[p] = finished ? 0 : s_base;
}

static void launch_scan_staged(NmsWorkspace& ws, const unsigned long long* mask, const int* nvalid, int problems,
                               int max_out, int limit, const int* base_count, const int* index_map, cudaStream_t st) {
  const size_t staged_smem = staged_scan_smem(ws.words);
  static bool attr[64] = {false};        // cudaFuncSetAttribute is per device
  int dev = 0;
  LUMI_CUDA_CHECK(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64 || !__atomic_load_n(&attr[dev], __ATOMIC_ACQUIRE)) {
    LUMI_CUDA_CHECK(cudaFuncSetAttribute(nms_scan_staged_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)NMS_STAGED_SMEM_MAX));
    if (dev >= 0 && dev < 64) __atomic_store_n(&attr[dev], true, __ATOMIC_RELEASE);
  }
  nms_scan_staged_kernel<<<problems, 256, staged_smem, st>>>(mask, nvalid, ws.ncap, ws.words, max_out, ws.keep, ws.nkeep,
                                                            limit, base_count, index_map);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
}

static dim3 mask_grid(const NmsWorkspace& ws, int problems, int n_max) {
  // blocks walk their problem's (row block, column block) pairs with a grid stride; the x extent is sized so that
  // the whole launch is ~64 resident blocks per SM -- with hundreds of (image, class) problems whose candidate
  // lists are short (SSD: 640 problems, most rows filtered by min_prob) a fixed 2048-wide grid was 1.3 M blocks
  // that exit at once, and their block-launch overhead dominated the step
  const long nw = (n_max + 63) / 64;
  long maxpairs = nw * (nw + 1) / 2;
  long gx = ((long)sm_budget(0, ws.sm_limit) * 64 + problems - 1) / problems;
  if (gx > 2048) gx = 2048;
  if (gx > maxpairs) gx = maxpairs;
  if (gx < 1) gx = 1;
  return dim3((unsigned)gx, problems);
}

static void run_nms(NmsWorkspace& ws, int problems, float thr, int max_out, cudaStream_t st) {
  if (!problems) return;
  const int path = nms_path(problems, ws.ncap, thr);
  if (path == NMS_PATH_TWO_PHASE) {
    LUMI_REQUIRE(ws.sboxes2 != nullptr, "nms: missing two-phase scratch");
    const int R1 = NMS_LAZY_R1;
    nms_mask_kernel<<<mask_grid(ws, problems, R1), 64, 0, st>>>(ws.sboxes, ws.nvalid, ws.ncap, ws.words, thr, ws.mask, R1);
    count_launch();
    LUMI_CUDA_CHECK(cudaGetLastError());
    launch_scan_staged(ws, ws.mask, ws.nvalid, problems, max_out, R1, nullptr, nullptr, st);
    dim3 gp((unsigned)cdiv(ws.ncap - R1, 256), problems);
    nms_prefilter_kernel<<<gp, 256, 0, st>>>(ws.sboxes, ws.nvalid, ws.ncap, thr, ws.keep, ws.nkeep, max_out, R1, ws.alive);
    count_launch();
    LUMI_CUDA_CHECK(cudaGetLastError());
    nms_compact_kernel<<<problems, 1024, 0, st>>>(ws.sboxes, ws.nvalid, ws.ncap, ws.alive, ws.nkeep, max_out, R1,
                                                  ws.sboxes2, ws.index_map, ws.nvalid2);
    count_launch();
    LUMI_CUDA_CHECK(cudaGetLastError());
    nms_mask_kernel<<<mask_grid(ws, problems, ws.ncap - R1), 64, 0, st>>>(ws.sboxes2, ws.nvalid2, ws.ncap, ws.words, thr,
                                                                         ws.mask, 0x7fffffff);
    count_launch();
    LUMI_CUDA_CHECK(cudaGetLastError());
    launch_scan_staged(ws, ws.mask, ws.nvalid2, problems, max_out, 0x7fffffff, ws.nkeep, ws.index_map, st);
    return;
  }
  nms_mask_kernel<<<mask_grid(ws, problems, ws.ncap), 64, 0, st>>>(ws.sboxes, ws.nvalid, ws.ncap, ws.words, thr, ws.mask,
                                                                  0x7fffffff);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
  if (path == NMS_PATH_STAGED) {
    launch_scan_staged(ws, ws.mask, ws.nvalid, problems, max_out, 0x7fffffff, nullptr, nullptr, st);
  } else {
    size_t smem = (size_t)ws.words * sizeof(unsigned long long);
    nms_scan_kernel<<<problems, 256, smem, st>>>(ws.mask, ws.nvalid, ws.ncap, ws.words, max_out, ws.keep, ws.nkeep);
    count_launch();
    LUMI_CUDA_CHECK(cudaGetLastError());
  }
}

// ------------------------------------------------------------------ RPN chain
// The top-k cut replaces the one-CTA sort of all anchors from this many anchors per kept candidate on.  On an H100
// (DESIGN section 4.2) the cut made the R50 step faster at 4 and 6 anchors per kept candidate; at 2.4 its RPN chain
// was faster but the pipelined step was not, because its full-GPU kernels contend with the other half-batch's convs.
constexpr long RPN_CUT_RATIO = 4;

__global__ void rpn_decode_kernel(const float* __restrict__ cls, const float* __restrict__ box, long img_stride_cls,
                                  long img_stride_box, int A, const float* __restrict__ anchors, RpnParams p, int cap,
                                  float* __restrict__ keys, float* __restrict__ boxes) {
  const int img = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.na) return;
  const int cell = i / A, a = i % A;
  const float* cp = cls + (size_t)img * img_stride_cls + (size_t)cell * p.cls_stride + p.cls_off + 2 * a;
  const float* bp = box + (size_t)img * img_stride_box + (size_t)cell * p.box_stride + p.box_off + 4 * a;
  float score;
  if (p.logits) {          // rpn.py:160-163: reshape(-1,2) softmax, foreground = column 1
    const float s0 = cp[0], s1 = cp[1];
    const float m = fmaxf(s0, s1);
    const float e0 = expf(__fsub_rn(s0, m)), e1 = expf(__fsub_rn(s1, m));
    score = __fdiv_rn(e1, __fadd_rn(e0, e1));
  } else {
    score = cp[1];
  }
  const float4 an = reinterpret_cast<const float4*>(anchors)[i];
  float4 b = decode_box(an, bp[0], bp[1], bp[2], bp[3], 1.f, 1.f);
  bool ok = (score >= p.min_prob) && area_positive(b);
  float im_h = p.im_h, im_w = p.im_w;
  if (p.tab) {             // packed batch: the image's own size, and only the cells of its own grid
    const int th = p.tab[img].th, tw = p.tab[img].tw;
    im_h = (float)th; im_w = (float)tw;
    const int fh = (th + p.feat_stride - 1) / p.feat_stride, fw = (tw + p.feat_stride - 1) / p.feat_stride;
    ok = ok && cell / p.grid_w < fh && cell % p.grid_w < fw;
  }
  if (p.filter_outside) ok = ok && (an.x >= 0.f && an.y >= 0.f && an.z < im_w && an.w < im_h);
  if (!p.clip_after_nms) b = clip_box(b, im_h, im_w);
  const size_t o = (size_t)img * cap + i;
  keys[o] = ok ? score : -1.f;
  reinterpret_cast<float4*>(boxes)[o] = b;
}

__global__ void rpn_output_kernel(const float* __restrict__ sboxes, const float* __restrict__ sscores,
                                  const int* __restrict__ keep, const int* __restrict__ nkeep, int cap, int max_out,
                                  int clip, float im_h, float im_w, const ResizeSrc* __restrict__ tab,
                                  float* __restrict__ proposals, float* __restrict__ scores, int* __restrict__ counts) {
  const int img = blockIdx.y;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int nk = nkeep[img];
  if (j == 0) counts[img] = nk;
  if (j >= max_out) return;
  float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
  float s = 0.f;
  if (j < nk) {
    const size_t src = (size_t)img * cap + keep[(size_t)img * max_out + j];
    b = reinterpret_cast<const float4*>(sboxes)[src];
    s = sscores[src];
    if (clip) b = tab ? clip_box(b, (float)tab[img].th, (float)tab[img].tw) : clip_box(b, im_h, im_w);
  }
  reinterpret_cast<float4*>(proposals)[(size_t)img * max_out + j] = b;
  scores[(size_t)img * max_out + j] = s;
}

void launch_rpn_proposals(const float* cls, const float* box, long img_stride_cls, long img_stride_box, int A,
                          const float* anchors, int nimg, const RpnParams& p, NmsWorkspace& ws, float* proposals,
                          float* scores, int* counts, cudaStream_t st) {
  LUMI_REQUIRE(p.na <= ws.cap && nimg <= ws.problems, "rpn_proposals: workspace too small");
  if (!nimg || !p.na) return;
  dim3 g1(cdiv(p.na, 256), nimg);
  rpn_decode_kernel<<<g1, 256, 0, st>>>(cls, box, img_stride_cls, img_stride_box, A, anchors, p, ws.cap, ws.keys,
                                        ws.boxes);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
  // problem stride is ws.cap; candidates per problem p.na: fill the tail with invalid once if na < cap
  if (p.na < ws.cap) {
    LUMI_CUDA_CHECK(cudaMemset2DAsync(ws.keys + p.na, (size_t)ws.cap * sizeof(float), 0xFF,
                                      (size_t)(ws.cap - p.na) * sizeof(float), nimg, st));   // 0xFFFFFFFF = NaN -> invalid
  }
  if (ws.cut_hist && (long)p.na >= RPN_CUT_RATIO * (long)p.pre_nms_top_n)
    run_topk_cut(ws.keys, nimg, ws.cap, p.na, p.pre_nms_top_n, ws.order, ws.nvalid, ws, st);
  else
    run_sort(ws.keys, nimg, ws.cap, p.na, nullptr, p.pre_nms_top_n, ws.order, ws.nvalid, ws.sort_tmp, st);
  LUMI_REQUIRE(p.pre_nms_top_n <= ws.ncap || p.na <= ws.ncap, "rpn_proposals: NMS workspace smaller than pre_nms_top_n");
  dim3 g2(cdiv(ws.ncap, 256), nimg);
  gather_sorted_kernel<<<g2, 256, 0, st>>>(ws.boxes, ws.keys, ws.order, ws.nvalid, ws.cap, ws.ncap, ws.sboxes,
                                           ws.sscores);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
  const float thr = p.apply_nms ? p.nms_threshold : INFINITY;
  LUMI_REQUIRE(p.post_nms_top_n <= ws.max_out, "rpn_proposals: post_nms_top_n exceeds workspace");
  run_nms(ws, nimg, thr, p.post_nms_top_n, st);
  dim3 g3(cdiv(p.post_nms_top_n, 256), nimg);
  rpn_output_kernel<<<g3, 256, 0, st>>>(ws.sboxes, ws.sscores, ws.keep, ws.nkeep, ws.ncap, p.post_nms_top_n,
                                        p.clip_after_nms, p.im_h, p.im_w, p.tab, proposals, scores, counts);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
}

size_t det_final_scratch_bytes(int nimg, int nc, int class_max) {
  const size_t fcap = (size_t)nc * class_max;
  return (size_t)nimg * fcap * 8 + (size_t)nimg * 4 + 16 + (size_t)nimg * 2 * fcap * sizeof(unsigned long long);
}

// ------------------------------------------------------------------ per-class detection chain
__global__ void det_decode_kernel(const float* __restrict__ boxes_in, long boxes_img_stride,
                                  const int* __restrict__ row_counts, const float* __restrict__ deltas,
                                  const float* __restrict__ cls_prob, DetParams p, int cap, float* __restrict__ keys,
                                  float* __restrict__ boxes) {
  const int prob_id = blockIdx.y;               // img*nc + c
  const int img = prob_id / p.nc, c = prob_id % p.nc;
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= p.r) return;
  const size_t o = (size_t)prob_id * cap + r;
  const bool live = row_counts == nullptr || r < row_counts[img];
  if (!live) { keys[o] = -1.f; return; }
  const size_t row = (size_t)img * p.r + r;
  const float prob = cls_prob[row * p.prob_stride + c + 1];
  const float* dp = deltas + row * p.delta_stride + (p.shared_deltas ? 0 : 4 * c);
  const float4 bin = reinterpret_cast<const float4*>(boxes_in)[(size_t)img * (boxes_img_stride / 4) + r];
  float4 b = decode_box(bin, dp[0], dp[1], dp[2], dp[3], p.var0, p.var1);
  b = p.tab ? clip_box(b, (float)p.tab[img].th, (float)p.tab[img].tw) : clip_box(b, p.im_h, p.im_w);
  const bool ok = (prob >= p.min_prob) && area_positive(b);
  keys[o] = ok ? prob : -1.f;
  reinterpret_cast<float4*>(boxes)[o] = b;
}

// concat per-class selections (class-major, NMS selection order) as sparse keys [img][nc*class_max]
__global__ void det_concat_kernel(const float* __restrict__ sscores, const int* __restrict__ keep,
                                  const int* __restrict__ nkeep, int nc, int cap, int class_max,
                                  float* __restrict__ fkeys) {
  const int prob_id = blockIdx.y;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= class_max) return;
  const int img = prob_id / nc, c = prob_id % nc;
  float v = -1.f;
  if (j < nkeep[prob_id]) v = sscores[(size_t)prob_id * cap + keep[(size_t)prob_id * class_max + j]];
  fkeys[((size_t)img * nc + c) * class_max + j] = v;
}

__global__ void det_output_kernel(const float* __restrict__ sboxes, const float* __restrict__ sscores,
                                  const int* __restrict__ keep, const int* __restrict__ forder,
                                  const int* __restrict__ fnvalid, int nc, int cap, int class_max, int total_max,
                                  float* __restrict__ objects, int* __restrict__ labels, float* __restrict__ probs,
                                  int* __restrict__ counts, float* __restrict__ records) {
  const int img = blockIdx.y;
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  const int nv = fnvalid[img];
  // optional packed all-gather record of this image: {count, boxes[K][4], scores[K], labels[K]} as float32
  float* rec = records ? records + (size_t)img * (1 + 6 * (size_t)total_max) : nullptr;
  if (k == 0) { counts[img] = nv; if (rec) rec[0] = (float)nv; }
  if (k >= total_max) return;
  float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
  float s = 0.f;
  int lab = -1;
  if (k < nv) {
    const int idx = forder[(size_t)img * nc * class_max + k];
    const int c = idx / class_max, j = idx % class_max;
    const int prob_id = img * nc + c;
    const size_t src = (size_t)prob_id * cap + keep[(size_t)prob_id * class_max + j];
    b = reinterpret_cast<const float4*>(sboxes)[src];
    s = sscores[src];
    lab = c;
  }
  reinterpret_cast<float4*>(objects)[(size_t)img * total_max + k] = b;
  probs[(size_t)img * total_max + k] = s;
  labels[(size_t)img * total_max + k] = lab;
  if (rec) {
    float* rb = rec + 1 + 4 * (size_t)k;
    rb[0] = b.x; rb[1] = b.y; rb[2] = b.z; rb[3] = b.w;
    rec[1 + 4 * (size_t)total_max + k] = s;
    rec[1 + 5 * (size_t)total_max + k] = (float)lab;
  }
}

// records of the RPN-only mode (predicting.py:85-92: objects = proposals, labels = 0) and of any caller that has
// plain (boxes, scores, labels, counts) arrays: same layout as det_output_kernel writes.
__global__ void pack_records_kernel(const float* __restrict__ boxes, const float* __restrict__ scores,
                                    const int* __restrict__ labels, const int* __restrict__ counts, int kmax,
                                    float* __restrict__ records) {
  const int img = blockIdx.y;
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  float* rec = records + (size_t)img * (1 + 6 * (size_t)kmax);
  if (k == 0) rec[0] = (float)counts[img];
  if (k >= kmax) return;
  const float4 b = reinterpret_cast<const float4*>(boxes)[(size_t)img * kmax + k];
  float* rb = rec + 1 + 4 * (size_t)k;
  rb[0] = b.x; rb[1] = b.y; rb[2] = b.z; rb[3] = b.w;
  rec[1 + 4 * (size_t)kmax + k] = scores[(size_t)img * kmax + k];
  rec[1 + 5 * (size_t)kmax + k] = (float)labels[(size_t)img * kmax + k];
}
void launch_pack_records(const float* boxes, const float* scores, const int* labels, const int* counts, int nimg,
                         int kmax, float* records, cudaStream_t st) {
  if (!nimg || !kmax) return;
  dim3 g(cdiv(kmax, 128), nimg);
  pack_records_kernel<<<g, 128, 0, st>>>(boxes, scores, labels, counts, kmax, records);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
}

// final_keys: scratch of det_final_scratch_bytes(): [nimg][nc*class_max] float keys, int order [same],
// int nvalid[nimg], then the radix ping-pong buffers
void launch_class_detections(const float* boxes_in, long boxes_img_stride, const int* row_counts, const float* deltas,
                             const float* cls_prob, int nimg, const DetParams& p, NmsWorkspace& ws, float* final_keys,
                             float* objects, int* labels, float* probs, int* counts, cudaStream_t st, float* records) {
  const int P = nimg * p.nc;
  LUMI_REQUIRE(P <= ws.problems && p.r <= ws.cap && p.class_max == ws.max_out, "class_detections: workspace mismatch");
  if (!P || !p.r) return;
  dim3 g1(cdiv(p.r, 256), P);
  det_decode_kernel<<<g1, 256, 0, st>>>(boxes_in, boxes_img_stride, row_counts, deltas, cls_prob, p, ws.cap, ws.keys,
                                        ws.boxes);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
  if (p.r < ws.cap)
    LUMI_CUDA_CHECK(cudaMemset2DAsync(ws.keys + p.r, (size_t)ws.cap * sizeof(float), 0xFF,
                                      (size_t)(ws.cap - p.r) * sizeof(float), P, st));
  run_sort(ws.keys, P, ws.cap, p.r, nullptr, ws.cap, ws.order, ws.nvalid, ws.sort_tmp, st);
  dim3 g2(cdiv(ws.ncap, 256), P);
  gather_sorted_kernel<<<g2, 256, 0, st>>>(ws.boxes, ws.keys, ws.order, ws.nvalid, ws.cap, ws.ncap, ws.sboxes,
                                           ws.sscores);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
  run_nms(ws, P, p.nms_threshold, p.class_max, st);
  const int fcap = p.nc * p.class_max;
  float* fkeys = final_keys;
  int* forder = reinterpret_cast<int*>(final_keys + (size_t)nimg * fcap);
  int* fnvalid = forder + (size_t)nimg * fcap;
  unsigned long long* fscratch = reinterpret_cast<unsigned long long*>(
      (reinterpret_cast<uintptr_t>(fnvalid + nimg) + 15) & ~(uintptr_t)15);
  dim3 g3(cdiv(p.class_max, 128), P);
  det_concat_kernel<<<g3, 128, 0, st>>>(ws.sscores, ws.keep, ws.nkeep, p.nc, ws.ncap, p.class_max, fkeys);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
  run_sort(fkeys, nimg, fcap, fcap, nullptr, p.total_max, forder, fnvalid, fscratch, st);
  dim3 g4(cdiv(p.total_max, 128), nimg);
  det_output_kernel<<<g4, 128, 0, st>>>(ws.sboxes, ws.sscores, ws.keep, forder, fnvalid, p.nc, ws.ncap, p.class_max,
                                        p.total_max, objects, labels, probs, counts, records);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
}

// ------------------------------------------------------------------ cross-window merge (lumi_predict_windows)
void plan_window_merge(const int* win_src, const int* labels, const int* counts, int nwin, int kmax, int nsrc, int nc,
                       int class_max, int total_max, WindowMergePlan& plan) {
  plan = WindowMergePlan();
  plan.nsrc = nsrc; plan.nc = nc; plan.class_max = class_max; plan.total_max = total_max; plan.kmax = kmax;
  LUMI_REQUIRE(nwin >= 0 && kmax >= 1 && nsrc >= 1 && nc >= 1 && class_max >= 1 && total_max >= 1 &&
                   (long long)nwin * kmax <= INT32_MAX,
               "window merge: need nwin >= 0, kmax, nsrc, nc, class_max, total_max >= 1 and nwin * kmax < 2^31");
  const size_t P = (size_t)nsrc * nc;
  std::vector<long long> len(P, 0);
  for (int k = 0; k < nwin; ++k) {
    LUMI_REQUIRE(win_src[k] >= 0 && win_src[k] < nsrc, "window merge: window source out of range");
    LUMI_REQUIRE(counts[k] >= 0 && counts[k] <= kmax, "window merge: detection count out of range");
    for (int r = 0; r < counts[k]; ++r) {
      const int lab = labels[(size_t)k * kmax + r];
      LUMI_REQUIRE(lab >= 0 && lab < nc, "window merge: detection label out of range");
      len[(size_t)win_src[k] * nc + lab]++;
    }
  }
  std::vector<long long> start(P + 1, 0);
  for (size_t p = 0; p < P; ++p) start[p + 1] = start[p] + len[p];
  plan.candidates = start[P];
  // every list in window order, then rank within the window
  std::vector<int> flat((size_t)plan.candidates);
  std::vector<long long> fill(start.begin(), start.end() - 1);
  for (int k = 0; k < nwin; ++k)
    for (int r = 0; r < counts[k]; ++r)
      flat[(size_t)fill[(size_t)win_src[k] * nc + labels[(size_t)k * kmax + r]]++] = k * kmax + r;
  std::vector<int> order;
  for (size_t p = 0; p < P; ++p) if (len[p]) order.push_back((int)p);
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return len[a] > len[b]; });
  plan.longest = order.empty() ? 0 : (int)len[order[0]];
  for (size_t i = 0; i < order.size();) {
    const long long cap = len[order[i]];
    const long long take = std::min<long long>((long long)order.size() - (long long)i,
                                               std::max<long long>(1, plan.candidates / cap));
    plan.groups.push_back({(int)take, (int)cap, (long long)plan.slots.size(), (int)plan.lists.size()});
    for (long long j = 0; j < take; ++j) {
      const int p = order[i + j];
      plan.lists.push_back(p);
      plan.slots.insert(plan.slots.end(), flat.begin() + start[p], flat.begin() + start[p] + len[p]);
      plan.slots.insert(plan.slots.end(), (size_t)(cap - len[p]), -1);
    }
    plan.elems = std::max(plan.elems, take * cap);
    plan.pmax = std::max(plan.pmax, (int)take);
    plan.mask_words = std::max(plan.mask_words, (size_t)(take * cap) * (size_t)nms_words((int)cap));
    i += (size_t)take;
  }
}

namespace {
struct MergeScratch {
  NmsWorkspace ws;              // the groups' sort / NMS buffers, viewed per group as [problems][cap]
  float* kboxes; float* kscores; int* kkeep; int* knkeep;   // kept detections per list [nsrc * nc][class_max]
  float* final_keys;            // det_final_scratch_bytes(nsrc, nc, class_max)
  size_t bytes;
};
// Carves the scratch of a plan out of `base` (nullptr: sizes only).
MergeScratch carve_merge(const WindowMergePlan& pl, uint8_t* base) {
  size_t off = 0;
  auto take = [&](size_t bytes) {
    uint8_t* p = base ? base + off : nullptr;
    off += (bytes + 255) / 256 * 256;
    return p;
  };
  MergeScratch m{};
  const size_t E = (size_t)std::max<long long>(pl.elems, 1), pm = (size_t)std::max(pl.pmax, 1);
  const size_t lists = (size_t)pl.nsrc * pl.nc, kept = lists * pl.class_max;
  // the kept rows first: their place depends on (nsrc, nc, class_max) alone, so in a reused buffer whatever a list's
  // row still holds is a kept row of an earlier call (never read: knkeep is cleared each call), not another buffer
  m.kboxes = (float*)take(kept * 16);
  m.kscores = (float*)take(kept * 4);
  m.kkeep = (int*)take(kept * 4);
  m.knkeep = (int*)take(lists * 4);
  m.ws.keys = (float*)take(E * 4);
  m.ws.boxes = (float*)take(E * 16);
  m.ws.order = (int*)take(E * 4);
  m.ws.nvalid = (int*)take(pm * 4);
  m.ws.sboxes = (float*)take(E * 16);
  m.ws.sscores = (float*)take(E * 4);
  m.ws.mask = (unsigned long long*)take(std::max<size_t>(pl.mask_words, 1) * 8);
  m.ws.keep = (int*)take(pm * pl.class_max * 4);
  m.ws.nkeep = (int*)take(pm * 4);
  m.ws.sort_tmp = (unsigned long long*)take(E * 2 * 8);
  if (pl.longest >= NMS_LAZY_MIN) {             // two-phase NMS scratch, as nms_workspace_alloc
    m.ws.sboxes2 = (float*)take(E * 16);
    m.ws.index_map = (int*)take(E * 4);
    m.ws.alive = (unsigned char*)take(E);
    m.ws.nvalid2 = (int*)take(pm * 4);
  }
  m.final_keys = (float*)take(det_final_scratch_bytes(pl.nsrc, pl.nc, pl.class_max));
  m.bytes = off;
  return m;
}
}  // namespace

size_t window_merge_bytes(const WindowMergePlan& plan) { return carve_merge(plan, nullptr).bytes; }

// slot i of a group: its candidate's box in source pixels and its score, or key -1 for padding
__global__ void window_gather_kernel(const float* __restrict__ wboxes, const float* __restrict__ wscores,
                                     const float4* __restrict__ wmap, const int* __restrict__ slots, int kmax,
                                     long long n, float* __restrict__ keys, float* __restrict__ boxes) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = slots[i];
  if (c < 0) { keys[i] = -1.f; return; }
  const float4 m = wmap[c / kmax];              // {y0, x0, s_y, s_x}
  float4 b = reinterpret_cast<const float4*>(wboxes)[c];
  b.x = __fadd_rn(__fdiv_rn(b.x, m.w), m.y);
  b.y = __fadd_rn(__fdiv_rn(b.y, m.z), m.x);
  b.z = __fadd_rn(__fdiv_rn(b.z, m.w), m.y);
  b.w = __fadd_rn(__fdiv_rn(b.w, m.z), m.x);
  reinterpret_cast<float4*>(boxes)[i] = b;
  keys[i] = wscores[c];
}

// a group's NMS selections into their list's row of the kept buffers, in selection order (keep = identity there)
__global__ void window_keep_kernel(const float* __restrict__ sboxes, const float* __restrict__ sscores,
                                   const int* __restrict__ keep, const int* __restrict__ nkeep,
                                   const int* __restrict__ lists, int cap, int class_max, float* __restrict__ kboxes,
                                   float* __restrict__ kscores, int* __restrict__ kkeep, int* __restrict__ knkeep) {
  const int p = blockIdx.y;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int list = lists[p], nk = nkeep[p];
  if (j == 0) knkeep[list] = nk;
  if (j >= nk || j >= class_max) return;
  const size_t src = (size_t)p * cap + keep[(size_t)p * class_max + j];
  const size_t dst = (size_t)list * class_max + j;
  reinterpret_cast<float4*>(kboxes)[dst] = reinterpret_cast<const float4*>(sboxes)[src];
  kscores[dst] = sscores[src];
  kkeep[dst] = j;
}

void launch_window_merge(const WindowMergePlan& plan, const int* d_slots, const int* d_lists, const float* wboxes,
                         const float* wscores, const float4* wmap, float thr, int sm_limit, void* scratch,
                         float* boxes, float* scores, int* labels, int* counts, cudaStream_t st) {
  MergeScratch m = carve_merge(plan, static_cast<uint8_t*>(scratch));
  const int lists = plan.nsrc * plan.nc, cm = plan.class_max;
  if (!lists) return;
  LUMI_CUDA_CHECK(cudaMemsetAsync(m.knkeep, 0, (size_t)lists * sizeof(int), st));
  for (const WindowMergePlan::Group& g : plan.groups) {
    NmsWorkspace ws = m.ws;
    ws.problems = g.problems; ws.cap = ws.ncap = g.cap; ws.words = nms_words(g.cap);
    ws.max_out = cm; ws.sm_limit = sm_limit;
    const long long n = (long long)g.problems * g.cap;
    window_gather_kernel<<<(unsigned)cdiv64(n, 256), 256, 0, st>>>(wboxes, wscores, wmap, d_slots + g.slot0,
                                                                   plan.kmax, n, ws.keys, ws.boxes);
    count_launch();
    LUMI_CUDA_CHECK(cudaGetLastError());
    run_sort(ws.keys, g.problems, g.cap, g.cap, nullptr, g.cap, ws.order, ws.nvalid, ws.sort_tmp, st);
    gather_sorted_kernel<<<dim3(cdiv(g.cap, 256), g.problems), 256, 0, st>>>(ws.boxes, ws.keys, ws.order, ws.nvalid,
                                                                              g.cap, g.cap, ws.sboxes, ws.sscores);
    count_launch();
    LUMI_CUDA_CHECK(cudaGetLastError());
    run_nms(ws, g.problems, thr, cm, st);
    window_keep_kernel<<<dim3(cdiv(cm, 128), g.problems), 128, 0, st>>>(ws.sboxes, ws.sscores, ws.keep, ws.nkeep,
                                                                        d_lists + g.prob0, g.cap, cm, m.kboxes,
                                                                        m.kscores, m.kkeep, m.knkeep);
    count_launch();
    LUMI_CUDA_CHECK(cudaGetLastError());
  }
  // the labels of each source, label-major, top total_max: the tail of the per-class detection chain
  const int fcap = plan.nc * cm;
  float* fkeys = m.final_keys;
  int* forder = reinterpret_cast<int*>(fkeys + (size_t)plan.nsrc * fcap);
  int* fnvalid = forder + (size_t)plan.nsrc * fcap;
  unsigned long long* fscratch = reinterpret_cast<unsigned long long*>(
      (reinterpret_cast<uintptr_t>(fnvalid + plan.nsrc) + 15) & ~(uintptr_t)15);
  det_concat_kernel<<<dim3(cdiv(cm, 128), lists), 128, 0, st>>>(m.kscores, m.kkeep, m.knkeep, plan.nc, cm, cm, fkeys);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
  run_sort(fkeys, plan.nsrc, fcap, fcap, nullptr, plan.total_max, forder, fnvalid, fscratch, st);
  det_output_kernel<<<dim3(cdiv(plan.total_max, 128), plan.nsrc), 128, 0, st>>>(
      m.kboxes, m.kscores, m.kkeep, forder, fnvalid, plan.nc, cm, cm, plan.total_max, boxes, labels, scores, counts,
      nullptr);
  count_launch();
  LUMI_CUDA_CHECK(cudaGetLastError());
}

void run_window_merge(const float* wboxes, const float* wscores, const int* wlabels, const int* wcounts,
                      const int* win_src, const float4* wmap, int nwin, int kmax, int nsrc, int nc, int class_max,
                      int total_max, float thr, int sm_limit, const std::function<uint8_t*(size_t)>& scratch,
                      float* boxes, float* scores, int* labels, int* counts, int64_t stats[4], cudaStream_t st) {
  LUMI_REQUIRE(thr >= 0.f, "window merge: iou_threshold must be >= 0");     // NaN fails too
  LUMI_REQUIRE(nwin >= 1 && kmax >= 1 && (long long)nwin * kmax <= INT32_MAX,
               "window merge: need nwin, kmax >= 1 and nwin * kmax < 2^31");
  // one read of the windows' labels and counts lays out the per-(source, label) lists
  std::vector<int> hl((size_t)nwin * kmax), hc(nwin);
  LUMI_CUDA_CHECK(cudaMemcpyAsync(hl.data(), wlabels, hl.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
  LUMI_CUDA_CHECK(cudaMemcpyAsync(hc.data(), wcounts, hc.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
  LUMI_CUDA_CHECK(cudaStreamSynchronize(st));
  WindowMergePlan plan;
  plan_window_merge(win_src, hl.data(), hc.data(), nwin, kmax, nsrc, nc, class_max, total_max, plan);
  auto round16 = [](size_t b) { return (b + 15) / 16 * 16; };
  const size_t o_slots = round16(window_merge_bytes(plan));
  const size_t o_lists = o_slots + round16(plan.slots.size() * sizeof(int));
  uint8_t* base = scratch(o_lists + round16(plan.lists.size() * sizeof(int)));
  int* d_slots = reinterpret_cast<int*>(base + o_slots);
  int* d_lists = reinterpret_cast<int*>(base + o_lists);
  if (!plan.slots.empty())
    LUMI_CUDA_CHECK(cudaMemcpyAsync(d_slots, plan.slots.data(), plan.slots.size() * sizeof(int),
                                    cudaMemcpyHostToDevice, st));
  if (!plan.lists.empty())
    LUMI_CUDA_CHECK(cudaMemcpyAsync(d_lists, plan.lists.data(), plan.lists.size() * sizeof(int),
                                    cudaMemcpyHostToDevice, st));
  launch_window_merge(plan, d_slots, d_lists, wboxes, wscores, wmap, thr, sm_limit, base, boxes, scores, labels, counts,
                      st);
  stats[0] = (int64_t)(o_lists + plan.lists.size() * sizeof(int)); stats[1] = plan.candidates;
  stats[2] = plan.longest; stats[3] = (int64_t)plan.groups.size();
}

// ------------------------------------------------------------------ stand-alone sort / NMS
void launch_sort_desc(const float* scores, int n, int* idx_out, NmsWorkspace& ws, cudaStream_t st) {
  LUMI_REQUIRE(n <= ws.cap && ws.problems >= 1, "sort_desc: workspace too small");
  LUMI_CUDA_CHECK(cudaMemsetAsync(ws.keys, 0xFF, (size_t)ws.cap * sizeof(float), st));
  LUMI_CUDA_CHECK(cudaMemcpyAsync(ws.keys, scores, (size_t)n * sizeof(float), cudaMemcpyDeviceToDevice, st));
  run_sort(ws.keys, 1, ws.cap, n, nullptr, ws.cap, ws.order, ws.nvalid, ws.sort_tmp, st);
  LUMI_CUDA_CHECK(cudaMemcpyAsync(idx_out, ws.order, (size_t)n * sizeof(int), cudaMemcpyDeviceToDevice, st));
}

void launch_nms_batched(const float* boxes_sorted, const int* nvalid, int problems, float thr, int max_out,
                        NmsWorkspace& ws, int* keep, int* nkeep, cudaStream_t st) {
  LUMI_REQUIRE(problems <= ws.problems && ws.ncap == ws.cap && max_out <= ws.max_out, "nms_batched: workspace too small");
  if (!problems) return;
  LUMI_CUDA_CHECK(cudaMemcpyAsync(ws.sboxes, boxes_sorted, (size_t)problems * ws.cap * 4 * sizeof(float),
                                  cudaMemcpyDeviceToDevice, st));
  LUMI_CUDA_CHECK(cudaMemcpyAsync(ws.nvalid, nvalid, (size_t)problems * sizeof(int), cudaMemcpyDeviceToDevice, st));
  run_nms(ws, problems, thr, max_out, st);
  LUMI_CUDA_CHECK(cudaMemcpyAsync(keep, ws.keep, (size_t)problems * max_out * sizeof(int), cudaMemcpyDeviceToDevice,
                                  st));                  // run_nms writes keep rows of max_out entries
  LUMI_CUDA_CHECK(cudaMemcpyAsync(nkeep, ws.nkeep, (size_t)problems * sizeof(int), cudaMemcpyDeviceToDevice, st));
}

__global__ void set_int_kernel(int* p, int v) { *p = v; }

void launch_nms_sorted(const float* boxes_sorted, int n, float thr, int max_out, NmsWorkspace& ws, int* keep,
                       int* nkeep, cudaStream_t st) {
  LUMI_REQUIRE(n <= ws.ncap && max_out <= ws.max_out, "nms_sorted: workspace too small");
  LUMI_CUDA_CHECK(cudaMemcpyAsync(ws.sboxes, boxes_sorted, (size_t)n * 4 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  set_int_kernel<<<1, 1, 0, st>>>(ws.nvalid, n);
  count_launch();
  run_nms(ws, 1, thr, max_out, st);
  LUMI_CUDA_CHECK(cudaMemcpyAsync(keep, ws.keep, (size_t)max_out * sizeof(int), cudaMemcpyDeviceToDevice, st));
  LUMI_CUDA_CHECK(cudaMemcpyAsync(nkeep, ws.nkeep, sizeof(int), cudaMemcpyDeviceToDevice, st));
}

}  // namespace lumi
