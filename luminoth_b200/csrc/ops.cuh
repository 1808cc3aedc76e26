// Launchers for the HBM-bound stages of the path (everything that is not a conv).
#pragma once
#include "common.cuh"

namespace lumi {

// ---- format conversion / preprocessing (elementwise.cu)
void launch_u8_to_act(const void* img, bool img_f32, Act out, const float* means /*3 or nullptr*/, cudaStream_t st);
void launch_f32_to_act(const float* x, Act out, cudaStream_t st);
// x2: (n, Ho+3, Wo+3, 16) space-to-depth staging of the 7x7/2 stem input (see elementwise.cu)
void launch_stem_s2d(const void* img, bool img_f32, int n, int h, int w, Act x2, const float* means, cudaStream_t st);
void launch_resize_bilinear(const void* src, bool src_f32, int h0, int w0, float* dst, int h, int w, cudaStream_t st);
void launch_pack_c3(const void* img, bool img_f32, int n, int h, int w, Act x2 /*(n,h+2,w+3,16)*/, cudaStream_t st);
void launch_act_to_f32(Act in, float* y, cudaStream_t st);
// pre_scale / pre_bias [c] (both or neither): out = relu(BN(max)) instead of the max (see elementwise.cu)
void launch_max_pool(Act in, Act out, int k, int stride, int pad_t, int pad_l, cudaStream_t st,
                     const float* pre_scale = nullptr, const float* pre_bias = nullptr);
void launch_l2norm_scale(Act in, Act out, const float* gamma, float eps, cudaStream_t st);
void launch_spatial_mean(Act in, Act out, cudaStream_t st);               // (R,h,w,C) -> (R,1,1,C)
void launch_softmax_rows(const float* x, float* y, int rows, int cols, int in_stride, cudaStream_t st);
void launch_frcnn_anchors(const int* ref /*A x 4*/, int A, int fh, int fw, int stride, float* out, cudaStream_t st);

// ---- ROI crop + 2x2 max pool (roi.cu) : roi_pool.py:68-95
// rois [nimg][rmax][4] (x1,y1,x2,y2 px), counts [nimg] (nullptr -> all rmax valid); out (nimg*rmax, pw, ph, C)
// and/or mean (nimg*rmax, 1, 1, C) = tf.reduce_mean over the pooled cells (either may be an empty Act).
// fmap_f32: fp32 NHWC copy of the feature map (n, fh, fw, c).  kernel: one of the ROI_* instance codes below, or -1
// for roi_kernel(c, ph, pw); a code whose shape preconditions fail throws LUMI_EINVAL.
void launch_roi_pool(const float* fmap_f32, int n, int fh, int fw, int c, const float* rois, const int* counts, int rmax,
                     float im_h, float im_w, int ph, int pw, Act out, Act mean, cudaStream_t st, int kernel = -1);
// Every kernel instance launch_roi_pool can start: the row-walk kernel at 6 / 5 / 4 resident CTAs per SM, the
// column-walk kernel at 4 / 8 channels per lane, and the round-1 cell kernel roi_pool_kernel<CPL, RB, NW>.
enum {
  ROI_ROWS_MINB6 = 0, ROI_ROWS_MINB5 = 1, ROI_ROWS_MINB4 = 2, ROI_COLS_CPL4 = 3, ROI_COLS_CPL8 = 4,
  ROI_CELLS_8_4_4 = 5, ROI_CELLS_8_4_8 = 6, ROI_CELLS_8_1_8 = 7, ROI_CELLS_4_1_8 = 8, ROI_KERNEL_COUNT = 9
};
// The instance launch_roi_pool picks for C channels and a ph x pw pooled size (host only; honours LUMI_ROI_KERNEL,
// LUMI_ROI_MINB, LUMI_ROI_COLS_CPL, LUMI_ROI_CPL, LUMI_ROI_RB and LUMI_ROI_NW, each read once per process), or -1
// when no instance takes the shape (C not a multiple of 8, a pooled side below 1, or 2 * (ph + pw) > 64).
int roi_kernel(int c, int ph, int pw);

// ---- proposal / detection chains (postproc.cu)
struct NmsWorkspace {
  // capacity: problems x cap candidates
  int problems = 0, cap = 0;    // cap: candidates per problem before the top-n cut (decode / sort capacity)
  int ncap = 0;                 // candidates per problem after the cut (sorted boxes / mask capacity), <= cap
  float* keys = nullptr;        // [P][cap]   score or -1 (invalid)
  float* boxes = nullptr;       // [P][cap][4] decoded (+clipped) boxes, input order
  int* order = nullptr;         // [P][cap]   sorted order (indices into input order)
  int* nvalid = nullptr;        // [P]        valid candidates (after top-n cut)
  float* sboxes = nullptr;      // [P][ncap][4] boxes in sorted order
  float* sscores = nullptr;     // [P][ncap]
  unsigned long long* mask = nullptr;  // [P][ncap][words]
  int words = 0;
  int* keep = nullptr;          // [P][max_out]
  int* nkeep = nullptr;         // [P]
  int max_out = 0;
  unsigned long long* sort_tmp = nullptr;  // global-memory sort scratch for cap > 32768
  // two-phase NMS (ncap >= 4096): survivors of the pre-filter, compacted in order
  float* sboxes2 = nullptr;     // [P][ncap][4]
  int* index_map = nullptr;     // [P][ncap]  compacted row -> row of sboxes
  unsigned char* alive = nullptr;  // [P][ncap]
  int* nvalid2 = nullptr;       // [P]
  // top-k cut ahead of the sort (ncap < cap, see run_topk_cut): radix-select histograms and per-CTA counts
  unsigned int* cut_hist = nullptr;         // [P][4 digits][256]
  unsigned long long* cut_counts = nullptr; // [P][cut_blocks] (candidates above the k-th key << 32 | equal to it)
  int cut_blocks = 0;
};
void nms_workspace_alloc(NmsWorkspace& ws, int problems, int cap, int max_out, int ncap = 0);
void nms_workspace_free(NmsWorkspace& ws);
// The NMS path of `problems` lists of up to ncap candidates at IoU threshold thr (host only, honours LUMI_NMS_LAZY):
// staged one-phase scan, two-phase (see postproc.cu), or the unstaged scan when the staged one's shared memory would
// exceed 200 KiB.
enum { NMS_PATH_STAGED = 0, NMS_PATH_TWO_PHASE = 1, NMS_PATH_UNSTAGED = 2 };
int nms_path(int problems, int ncap, float thr);

struct RpnParams {
  int na;                 // anchors per image
  float im_h, im_w;
  int pre_nms_top_n, post_nms_top_n;
  float nms_threshold, min_prob;
  int filter_outside, clip_after_nms, apply_nms;
  int logits;             // 1: cls input holds logits (softmax fused), 0: probabilities
  int cls_stride, cls_off, box_stride, box_off;  // per-anchor-cell channel layout of the fused head output
};
// cls/box: per image [na/A cells][channels]; anchors [na][4] float. Outputs per image [post_nms_top_n].
void launch_rpn_proposals(const float* cls, const float* box, long img_stride_cls, long img_stride_box, int A,
                          const float* anchors, int nimg, const RpnParams& p, NmsWorkspace& ws, float* proposals,
                          float* scores, int* counts, cudaStream_t st);

struct DetParams {
  int r;                  // rows (proposals / anchors) per image (capacity)
  int nc;                 // foreground classes
  float im_h, im_w, var0, var1, min_prob, nms_threshold;
  int class_max, total_max;
  int shared_deltas;      // 1: deltas [r][4] shared by all classes (SSD), 0: [r][4*nc]
  int prob_stride;        // floats between consecutive rows of cls_prob (>= nc+1)
  int delta_stride;       // floats between consecutive rows of deltas
};
size_t det_final_scratch_bytes(int nimg, int nc, int class_max);   // size of `final_keys` below
// boxes_in [nimg][r][4] (or shared anchors when boxes_img_stride == 0), row_counts [nimg] or nullptr
void launch_class_detections(const float* boxes_in, long boxes_img_stride, const int* row_counts, const float* deltas,
                             const float* cls_prob, int nimg, const DetParams& p, NmsWorkspace& ws, float* final_keys,
                             float* objects, int* labels, float* probs, int* counts, cudaStream_t st,
                             float* records = nullptr /* optional packed rows [nimg][1 + 6*total_max], see postproc.cu */);
void launch_pack_records(const float* boxes, const float* scores, const int* labels, const int* counts, int nimg,
                         int kmax, float* records, cudaStream_t st);

void launch_sort_desc(const float* scores, int n, int* idx_out, NmsWorkspace& ws, cudaStream_t st);
void launch_nms_sorted(const float* boxes_sorted, int n, float thr, int max_out, NmsWorkspace& ws, int* keep,
                       int* nkeep, cudaStream_t st);
// boxes_sorted [problems][ws.cap][4], nvalid [problems] (device); keep [problems][max_out], nkeep [problems]
void launch_nms_batched(const float* boxes_sorted, const int* nvalid, int problems, float thr, int max_out,
                        NmsWorkspace& ws, int* keep, int* nkeep, cudaStream_t st);

}  // namespace lumi
