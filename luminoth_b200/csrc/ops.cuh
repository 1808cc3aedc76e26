// Launchers for the HBM-bound stages of the path (everything that is not a conv).
#pragma once
#include "common.cuh"
#include <functional>
#include <vector>

namespace lumi {

// ---- format conversion / preprocessing (elementwise.cu)
// Pixel formats of the images a predict call reads (LUMI_PIXELS_* of the C ABI).  RGB and BGR: [h][w][3] uint8 or
// float32.  NV12: the Y plane [h][w], then [h/2][w/2] interleaved U, V pairs.  I420: Y [h][w], U [h/2][w/2], V
// [h/2][w/2].  YUV is uint8 with even h and w, converted with OpenCV's BT.601 limited-range integer formula.
enum { PIX_RGB = 0, PIX_BGR = 1, PIX_NV12 = 2, PIX_I420 = 3 };
__host__ __device__ constexpr bool pix_yuv(int format) { return format == PIX_NV12 || format == PIX_I420; }
// Bytes of one h x w image in `format` (esz: bytes per channel value of RGB / BGR).
inline size_t pixel_bytes(int format, int h, int w, int esz) {
  return pix_yuv(format) ? (size_t)h * w * 3 / 2 : (size_t)h * w * 3 * esz;
}
// Throws LUMI_EINVAL unless an h x w image (float32 when f32) can be read in `format`; `who` prefixes the message.
void check_pixel_format(int format, bool f32, int h, int w, const std::string& who);

// One source image of a fused resize: its first byte at `off` in the source buffer, h0 x w0 pixels, resized to its
// target th x tw with the scale factors hs = (float)h0 / th, ws = (float)w0 / tw (as launch_resize_bilinear computes
// them).  A uniform batch has th x tw = the batch's h x w; a packed batch (lumi_predict_sizes) places each image at the
// top left of its h x w canvas, and the per-image kernels below read th x tw from this one table.  pitch: pixels
// between the starts of two source rows -- w0 for a whole image.  A window of a larger source (lumi_predict_windows) is
// h0 x w0 with pitch the source's width; RGB / BGR windows have `off` at their top-left pixel and oy = ox = 0.  4:2:0
// chroma rows cannot be addressed from a window's odd origin, so YUV windows keep `off` at the source's first byte and
// give the window's origin (oy, ox) in the source; plane_h is the source's height, the rows of its Y plane, which its
// chroma planes follow.
struct ResizeSrc {
  long long off;
  int h0, w0;
  float hs, ws;
  int th, tw;
  int pitch;
  int oy, ox, plane_h;
};
// The pixels the input staging kernels read: with table == nullptr, img is the batch itself, n images of h x w in
// `format` one after the other; otherwise image i of the batch is table[i]'s source in img, bilinearly resized on the
// fly.  f32: float32 pixels, else uint8.  packed: pixels outside image i's th x tw are the zero padding (0 after the
// mean subtraction).
struct ImgSrc {
  const void* img;
  bool f32;
  const ResizeSrc* table;
  bool packed;
  int format = PIX_RGB;
};
// Stand-alone conversion (lumi_op_pixels_to_rgb): the h x w image src in `format` as [h][w][3] RGB of its dtype, read
// through the staging kernels' pixel reader.
void launch_pixels_to_rgb(const void* src, int format, bool f32, int h, int w, void* dst, cudaStream_t st);
void launch_u8_to_act(ImgSrc src, Act out /*(n,h,w,3)*/, const float* means /*3 or nullptr*/, cudaStream_t st);
void launch_f32_to_act(const float* x, Act out, cudaStream_t st);
// x2: (n, Ho+3, Wo+3, 16) space-to-depth staging of the 7x7/2 stem input (see elementwise.cu)
void launch_stem_s2d(ImgSrc src, int n, int h, int w, Act x2, const float* means, cudaStream_t st);
void launch_resize_bilinear(const void* src, bool src_f32, int h0, int w0, float* dst, int h, int w, cudaStream_t st);
void launch_pack_c3(ImgSrc src, int n, int h, int w, Act x2 /*(n,h+2,w+3,16)*/, cudaStream_t st);
void launch_act_to_f32(Act in, float* y, cudaStream_t st);
// pre_scale / pre_bias [c] (both or neither): out = relu(BN(max)) instead of the max (see elementwise.cu)
// tab (packed batch, SAME padding only): image i's input extent is ceil(tab[i].th / in_stride) x ceil(tw / in_stride)
// and its front padding the one SAME gives that extent; outputs past its own output extent are 0
void launch_max_pool(Act in, Act out, int k, int stride, int pad_t, int pad_l, cudaStream_t st,
                     const float* pre_scale = nullptr, const float* pre_bias = nullptr,
                     const ResizeSrc* tab = nullptr, int in_stride = 0);
// Packed batch: zeros the rows and columns of `a` past image i's extent ceil(tab[i].th / in_stride) (and tw) that a
// conv (kh x kw, stride, rate, front padding pad_t / pad_l) reads from image i's valid outputs -- the zero padding
// that image has when it runs alone.
void launch_band_clear(Act a, const ResizeSrc* tab, int in_stride, int kh, int kw, int stride, int rate, int pad_t,
                       int pad_l, cudaStream_t st);
void launch_l2norm_scale(Act in, Act out, const float* gamma, float eps, cudaStream_t st);
void launch_spatial_mean(Act in, Act out, cudaStream_t st);               // (R,h,w,C) -> (R,1,1,C)
void launch_softmax_rows(const float* x, float* y, int rows, int cols, int in_stride, cudaStream_t st);
void launch_frcnn_anchors(const int* ref /*A x 4*/, int A, int fh, int fw, int stride, float* out, cudaStream_t st);

// ---- ROI crop + 2x2 max pool (roi.cu) : roi_pool.py:68-95
// rois [nimg][rmax][4] (x1,y1,x2,y2 px), counts [nimg] (nullptr -> all rmax valid); out (nimg*rmax, pw, ph, C)
// and/or mean (nimg*rmax, 1, 1, C) = tf.reduce_mean over the pooled cells (either may be an empty Act).
// fmap_f32: fp32 NHWC copy of the feature map (n, fh, fw, c).  kernel: one of the ROI_* instance codes below, or -1
// for roi_kernel(c, ph, pw); a code whose shape preconditions fail throws LUMI_EINVAL.
// tab (packed batch): image i is tab[i].th x tw with a ceil(th / feat_stride) x ceil(tw / feat_stride) feature grid at
// the top left of the fh x fw map; its rois are normalised and sampled on that grid (im_h / im_w are then unused).
void launch_roi_pool(const float* fmap_f32, int n, int fh, int fw, int c, const float* rois, const int* counts, int rmax,
                     float im_h, float im_w, int ph, int pw, Act out, Act mean, cudaStream_t st, int kernel = -1,
                     const ResizeSrc* tab = nullptr, int feat_stride = 0);
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
  int sm_limit = 0;             // SMs the NMS mask grid is sized for (0: the device's; see sm_budget)
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
  // packed batch (or nullptr): image i is tab[i].th x tw, its anchors those of the cells inside its
  // ceil(th / feat_stride) x ceil(tw / feat_stride) grid at the top left of the grid_w cells wide canvas grid
  const ResizeSrc* tab;
  int feat_stride, grid_w;
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
  const ResizeSrc* tab;   // packed batch: image i is clipped to tab[i].th x tw instead of im_h x im_w (or nullptr)
};
size_t det_final_scratch_bytes(int nimg, int nc, int class_max);   // size of `final_keys` below
// boxes_in [nimg][r][4] (or shared anchors when boxes_img_stride == 0), row_counts [nimg] or nullptr
void launch_class_detections(const float* boxes_in, long boxes_img_stride, const int* row_counts, const float* deltas,
                             const float* cls_prob, int nimg, const DetParams& p, NmsWorkspace& ws, float* final_keys,
                             float* objects, int* labels, float* probs, int* counts, cudaStream_t st,
                             float* records = nullptr /* optional packed rows [nimg][1 + 6*total_max], see postproc.cu */);
void launch_pack_records(const float* boxes, const float* scores, const int* labels, const int* counts, int nimg,
                         int kmax, float* records, cudaStream_t st);

// ---- cross-window merge of lumi_predict_windows (postproc.cu)
// The per-(source, label) candidate lists of the window detections, laid out from their labels and counts on the host.
// Lists with candidates run in groups: sorted by length (longest first), a group takes lists while their count times
// the group's first (longest) length stays within the call's candidate total T, so every group's [problems][cap]
// buffers hold at most T candidates, whatever the number of classes and windows (DESIGN section 4.2).
struct WindowMergePlan {
  struct Group { int problems, cap; long long slot0; int prob0; };
  int nsrc = 0, nc = 0, class_max = 0, total_max = 0, kmax = 0;
  long long candidates = 0;     // T: window detections in the call
  int longest = 0;              // L: the longest list
  long long elems = 0;          // largest group's problems x cap (<= T)
  int pmax = 0;                 // most lists in one group
  size_t mask_words = 0;        // largest group's NMS bit mask, in u64 words
  std::vector<Group> groups;
  std::vector<int> slots;       // per group [problems][cap]: candidate (window * kmax + rank) or -1 (padding)
  std::vector<int> lists;       // per group [problems]: source * nc + label
};
// win_src [nwin] source of each window; labels [nwin][kmax], counts [nwin] (host) the windows' detections.
void plan_window_merge(const int* win_src, const int* labels, const int* counts, int nwin, int kmax, int nsrc, int nc,
                       int class_max, int total_max, WindowMergePlan& plan);
size_t window_merge_bytes(const WindowMergePlan& plan);     // device scratch launch_window_merge needs
// Maps each window detection to source pixels (x / s_x + x0, y / s_y + y0; wmap [nwin] = {y0, x0, s_y, s_x}), sorts
// each list by score (stable), runs greedy NMS at thr keeping class_max per list, and writes per source the top
// total_max of the kept detections, label-major on ties: boxes [nsrc][total_max][4], scores, labels, counts [nsrc].
// d_slots / d_lists: plan.slots / plan.lists on the device.
void launch_window_merge(const WindowMergePlan& plan, const int* d_slots, const int* d_lists, const float* wboxes,
                         const float* wscores, const float4* wmap, float thr, int sm_limit, void* scratch,
                         float* boxes, float* scores, int* labels, int* counts, cudaStream_t st);
// The whole merge after the window forwards, as lumi_predict_windows and lumi_op_window_merge run it: reads the
// windows' labels and counts [nwin][kmax], [nwin] (device) back, synchronising st; checks them, thr and win_src [nwin]
// (host); plans the lists; takes a device buffer of at least the bytes it asks `scratch` for; uploads the plan and
// launches launch_window_merge.  wmap [nwin] on the device.  stats = {merge workspace bytes, candidates, longest list,
// groups}.
void run_window_merge(const float* wboxes, const float* wscores, const int* wlabels, const int* wcounts,
                      const int* win_src, const float4* wmap, int nwin, int kmax, int nsrc, int nc, int class_max,
                      int total_max, float thr, int sm_limit, const std::function<uint8_t*(size_t)>& scratch,
                      float* boxes, float* scores, int* labels, int* counts, int64_t stats[4], cudaStream_t st);

void launch_sort_desc(const float* scores, int n, int* idx_out, NmsWorkspace& ws, cudaStream_t st);
void launch_nms_sorted(const float* boxes_sorted, int n, float thr, int max_out, NmsWorkspace& ws, int* keep,
                       int* nkeep, cudaStream_t st);
// boxes_sorted [problems][ws.cap][4], nvalid [problems] (device); keep [problems][max_out], nkeep [problems]
void launch_nms_batched(const float* boxes_sorted, const int* nvalid, int problems, float thr, int max_out,
                        NmsWorkspace& ws, int* keep, int* nkeep, cudaStream_t st);

}  // namespace lumi
