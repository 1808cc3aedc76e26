/* luminoth_b200 -- C ABI of the H100-native (sm_90a) detection inference engine.
 *
 * Drop-in boundary for the Faster R-CNN / SSD predict path of tryolabs/luminoth
 * (the reference).  The reference is pure Python on top
 * of TensorFlow 1.x: its "FFI" for this path is the TF session boundary in
 *   utils/predicting.py:20-107   graph build + weight restore   -> lumi_create / lumi_set_weight / lumi_finalize
 *   utils/predicting.py:109-112  session.run(fetches, {image})  -> lumi_predict
 *   utils/predicting.py:98-107   fetches objects/labels/probs   -> boxes/scores/labels/counts outputs
 * A maintainer binds these with ctypes (see INTEGRATION.md).  Plain pointers and
 * sizes only; no torch / C++ types.  Every function returns 0 on success, a
 * negative LUMI_E* code otherwise; lumi_last_error() gives the message.
 *
 * Threading: one engine = one CUDA stream + workspace, NOT re-entrant (the
 * Python wrapper holds a lock, like the single tf.Session of the reference).
 */
#ifndef LUMINOTH_B200_H
#define LUMINOTH_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LUMI_OK 0
#define LUMI_EINVAL -1    /* bad argument / unsupported configuration  (ValueError in the wrapper) */
#define LUMI_ECUDA -2     /* CUDA runtime / driver failure             (RuntimeError) */
#define LUMI_ESTATE -3    /* call order violated (e.g. predict before finalize) */
#define LUMI_ENOWEIGHT -4 /* a variable the graph needs was never set  (ValueError) */
#define LUMI_EOVERFLOW -5 /* an activation left the fp16x2 split range (RuntimeError, never silent) */

typedef struct lumi_engine lumi_engine;

/* Library / device info.  lumi_version: static string.  lumi_device_count: visible CUDA devices (0 without a GPU). */
const char* lumi_version(void);
int lumi_device_count(void);

/* Build an engine for the model described by cfg_json = json.dumps(config)
 * (the merged YAML config, luminoth/utils/config.py:14-22; model.type selects
 * 'fasterrcnn' | 'ssd' like models/models.py:7-17).  max_batch images per
 * lumi_predict call, each at most max_h x max_w after preprocessing. */
int lumi_create(const char* cfg_json, int device, int max_batch, int max_h, int max_w, lumi_engine** out);

/* Feed one TF variable (fp32, HOST pointer) by its checkpoint name, TF layout:
 * conv [kh,kw,Cin,Cout], linear [in,out], vectors [C].  Replaces
 * tf.train.Saver.restore (predicting.py:51-63). */
int lumi_set_weight(lumi_engine* e, const char* tf_var_name, const float* host_data, const int64_t* shape, int ndim);

/* Number of variables the graph needs / names (for the wrapper's random-init path, predicting.py:64-72). */
int lumi_num_weights(lumi_engine* e);
int lumi_weight_info(lumi_engine* e, int index, const char** name, int64_t* shape4, int* ndim);

/* Fold BN, split weights into fp16 hi/lo planes, build TMA descriptors, allocate the workspace. */
int lumi_finalize(lumi_engine* e);

/* Run the forward pass on n images of identical size h x w (already resized
 * like datasets/object_detection_dataset.py:71-83), RGB, NHWC.
 *   images      uint8 [n,h,w,3]; host pointer (images_on_device = 0, copied H2D inside)
 *               or device pointer (images_on_device = 1)
 *   boxes       float [n, kmax, 4]  (x1,y1,x2,y2) in resized-image pixels
 *   scores      float [n, kmax]
 *   labels      int32 [n, kmax]     0-based foreground ids (quirk Q9)
 *   counts      int32 [n]           valid rows per image
 * kmax = lumi_max_detections(e).  Outputs are host pointers when
 * outputs_on_device = 0 (copied D2H + synchronised before returning) or device
 * pointers (asynchronous on lumi_stream(e)). */
int lumi_predict(lumi_engine* e, const void* images, int images_on_device, int n, int h, int w,
                 float* boxes, float* scores, int32_t* labels, int32_t* counts, int outputs_on_device);

/* Same call for float32 images [n,h,w,3]: what the reference's graph sees when the dataset preprocessing
 * resized the input (utils/image.py:38-147 produces non-integer pixel values; predicting.py:110-112 feeds them
 * as they are).  lumi_predict is the exact special case of integer-valued pixels. */
int lumi_predict_f32(lumi_engine* e, const float* images, int images_on_device, int n, int h, int w,
                     float* boxes, float* scores, int32_t* labels, int32_t* counts, int outputs_on_device);

int lumi_max_detections(lumi_engine* e);

/* Multi-GPU detection exchange (SURVEY 8e; the reference has no counterpart -- it predicts one image at a time,
 * tasks.py:146-154): when `device_records` is non-NULL every following lumi_predict ALSO writes, from the same
 * kernel that writes boxes/scores/labels, one packed float32 row per image
 *   {count, boxes[kmax][4], scores[kmax], labels[kmax]}      (1 + 6*kmax floats)
 * into the caller's DEVICE buffer [max_batch][1 + 6*kmax] -- the send buffer of the per-step ncclAllGather.
 * NULL switches it off. */
int lumi_set_record_output(lumi_engine* e, float* device_records);
void* lumi_stream(lumi_engine* e);            /* cudaStream_t the engine launches on */
int lumi_synchronize(lumi_engine* e);
/* Kernels launched by the last lumi_predict (our own kernels, for bench.py's gpu_launches). */
int lumi_last_launch_count(lumi_engine* e);

/* Per-category device timing (CUDA events on the engine stream around our kernels; bench.py's roofline).
 * lumi_profile_read drains the spans recorded since the last read: "name:spans:total_ms:work;..."
 * (work = algorithmic FLOPs for conv_*, algorithmic bytes for roi_pool). */
int lumi_profile_enable(lumi_engine* e, int enable);
const char* lumi_profile_read(lumi_engine* e);
/* Per-conv-layer detail of the spans drained by the last lumi_profile_read:
 * "layer:spans:total_ms:flops;..." in execution order. */
const char* lumi_profile_read_layers(lumi_engine* e);

/* Choose the convolution implementation: 0 = fp32 SIMT implicit GEMM everywhere,
 * 1 = wgmma fp16x2-split tensor-core kernel wherever the layer qualifies (default). */
int lumi_set_conv_impl(lumi_engine* e, int impl);

/* Work scheduling of the tensor-core convolution: 0 = whole output tiles only, 1 (default) = stream-K (the
 * K loops of all tiles cut into equal per-SM ranges, partial tiles summed in a fixed order) for layers whose
 * tile count would leave SMs idle in the last wave, 2 = stream-K wherever it is applicable. Results
 * are deterministic in every mode; modes differ in fp32 summation order only. */
int lumi_set_conv_streamk(lumi_engine* e, int mode);

/* 1 (default): lumi_predict splits the batch in two halves that run on two streams, so the latency-bound
 * proposal / NMS kernels of one half overlap the convolutions of the other. 0: single stream. Results are
 * identical either way (images are independent). Off automatically while profiling or tapping. */
int lumi_set_pipeline(lumi_engine* e, int enable);

/* 1 (default): the forward of every (half-)batch shape is captured into a CUDA graph the second time the shape is
 * seen and replayed afterwards (one launch instead of ~40-75 kernels: removes the launch gaps that bound small-batch
 * latency). 0: plain stream launches. Results are bit-identical either way. Env LUMI_GRAPHS=0 sets the default.
 * lumi_last_graph_replays: how many (half-)batch forwards of the last lumi_predict were graph replays. */
int lumi_set_graphs(lumi_engine* e, int enable);
int lumi_last_graph_replays(lumi_engine* e);

/* 1: also materialise intermediates the fused production path never writes (the "roi_pool" tap when
 * ROI crop + max-pool + mean run as one kernel) -- config.train.debug in the reference. Default 0. */
int lumi_set_debug_taps(lumi_engine* e, int enable);

/* Debug taps for parity tests (models' debug fetches, predicting.py:104-107):
 * copy a named intermediate of the LAST lumi_predict to host as fp32.
 * Names: "conv_feature_map", "rpn_cls_prob", "rpn_bbox_pred", "all_anchors",
 * "proposals", "proposal_scores", "proposal_counts", "roi_pool", "rcnn_cls_prob",
 * "rcnn_bbox_offsets", SSD: "cls_prob", "loc_pred", "all_anchors", "fmap_<i>".
 * Call with out = NULL to query the element count in *numel. */
int lumi_get_tensor(lumi_engine* e, const char* name, float* out, int64_t capacity, int64_t* numel, int64_t* shape4);

const char* lumi_last_error(lumi_engine* e);  /* e may be NULL: last error of lumi_create */
void lumi_destroy(lumi_engine* e);

/* ---- stand-alone operators on DEVICE buffers (per-kernel parity tests and
 * micro-benchmarks; each is one stage of the path, same kernels the engine uses).
 * All launch on `stream` (cudaStream_t, may be NULL) and synchronise it before returning
 * (temporaries are released). ---- */

const char* lumi_op_last_error(void);      /* message of the last failed lumi_op_* call on this thread */

/* conv2d NHWC fp32 in/out (converted to/from the fp16x2 split planes internally).
 * w: TF layout [kh,kw,cin,cout] fp32 on DEVICE.  scale/bias [cout] or NULL.
 * residual NHWC fp32 [n,ho,wo,cout] or NULL.  act: 0 none, 1 relu, 2 relu6.
 * padding: 0 VALID, 1 SAME, 2 explicit slim conv2d_same.  impl: 0 SIMT, 1 wgmma
 * (whole-tile schedule), 2 wgmma with the stream-K schedule forced; 3-11 write the fp16x2 split planes the engine
 * passes between layers: 3 two consumer warpgroups, 4 / 5 four warpgroups on short-K layers (5: + stream-K),
 * 6 / 7 2-CTA clusters multicasting the weight tile (7: + stream-K), 8 / 9 halo-patch kernels on 3x3 stride-1 layers
 * (9: + stream-K), 10 / 11 halo patches on 2-CTA clusters (11: + stream-K), 12 as 3 with the register epilogue, 13 the
 * SIMT kernel writing split planes (what the engine stores under conv_impl = simt), 14 / 15 as 3 on 128 x 256 tiles
 * (15: + stream-K; C_out padded to a multiple of 256 only).  Returns LUMI_EOVERFLOW when a split output (codes 3-15)
 * exceeds the split range, |x| > 65504. */
int lumi_op_conv2d(const float* x, int n, int h, int w, int cin, const float* wgt, int kh, int kw, int cout,
                   int stride, int rate, int padding, const float* scale, const float* bias,
                   const float* residual, int act, int impl, float* y, int* ho, int* wo, void* stream);

/* lumi_op_conv2d with the pre-activation output of a pre-activation ResNet unit, as the engine fuses it into the conv
 * epilogue: p = relu(fmaf(x^, pre_scale[c], pre_bias[c])) where x^ is the output x as stored in its fp16x2 split
 * planes.  pre_scale / pre_bias [cout] on DEVICE.  y (x) and p are NHWC fp32 read back from the split planes; y may be
 * NULL to write p only; y and p both NULL is a shape query.  impl: 0 or 13 SIMT, or one of the split-output codes 3-7,
 * 12 (12: as 3 with the register epilogue).  Returns LUMI_EOVERFLOW when x or p exceeds the split range. */
int lumi_op_conv2d_preact(const float* x, int n, int h, int w, int cin, const float* wgt, int kh, int kw, int cout,
                          int stride, int rate, int padding, const float* scale, const float* bias,
                          const float* residual, int act, int impl, const float* pre_scale, const float* pre_bias,
                          float* y, float* p, int* ho, int* wo, void* stream);

/* The conv launch with every output and residual option the engine uses.  The arguments of lumi_op_conv2d, plus:
 *   residual  NHWC fp32 [n,res_h,res_w,cout] on DEVICE or NULL, read at (oy*res_stride, ox*res_stride): res_stride 2
 *             with the input's resolution is slim's `subsample` shortcut of a bottleneck unit; res_stride 1 with
 *             res_h = ho, res_w = wo is lumi_op_conv2d's residual.
 *   pre_scale, pre_bias  NULL (no pre-activation output; y is required) or the pre-activation of
 *             lumi_op_conv2d_preact (p required, y may be NULL to write p only).
 * impl: the codes of lumi_op_conv2d; with a pre-activation output those of lumi_op_conv2d_preact.  y and p both NULL
 * is a shape query.  Returns LUMI_EOVERFLOW when a split output exceeds the split range. */
int lumi_op_conv2d_io(const float* x, int n, int h, int w, int cin, const float* wgt, int kh, int kw, int cout,
                      int stride, int rate, int padding, const float* scale, const float* bias, const float* residual,
                      int res_h, int res_w, int res_stride, int act, int impl, const float* pre_scale,
                      const float* pre_bias, float* y, float* p, int* ho, int* wo, void* stream);

/* The tensor-core weight packing of a conv layer, on HOST pointers and without any CUDA call.  w: TF layout
 * [kdim = kh*kw*cin][cout] fp32; scale [cout] or NULL (1).  Writes hi, lo: [cout][kdim] fp16 bit patterns of the split
 * of w[:, c] * 2^e[c], and scale_tc [cout] = scale[c] * 2^-e[c] rounded once to fp32.  e[c] puts max|w[:, c]| in
 * [2^13, 2^14), clamped to [-126, 126]; an all-zero column gets e = 0 (DESIGN section 2). */
int lumi_pack_conv_weights(const float* w, int kdim, int cout, const float* scale, uint16_t* hi, uint16_t* lo,
                           float* scale_tc);

/* tf.image.resize_images(BILINEAR) of TF 1.x (legacy kernel, align_corners=False) on one HWC image with 3 channels,
 * utils/image.py:94-97,139-142.  src: DEVICE uint8 (src_is_f32 = 0) or float32 (1) [h0,w0,3]; dst DEVICE float32 [h,w,3]. */
int lumi_op_resize_bilinear(const void* src, int src_is_f32, int h0, int w0, float* dst, int h, int w, void* stream);

/* max_pool NHWC fp32. padding 0 VALID / 1 SAME. */
int lumi_op_max_pool(const float* x, int n, int h, int w, int c, int k, int stride, int padding, float* y, void* stream);

/* max_pool followed by the pre-activation of a pre-activation ResNet unit: y = relu(fmaf(m^, pre_scale[c],
 * pre_bias[c])), m^ the max as stored in its split planes.  pre_scale / pre_bias [c] on DEVICE. */
int lumi_op_max_pool_preact(const float* x, int n, int h, int w, int c, int k, int stride, int padding,
                            const float* pre_scale, const float* pre_bias, float* y, void* stream);

/* ROI crop + 2x2 max pool: roi_pool.py:68-95.  Like the reference, the crop is 2pw rows x 2ph columns (quirk Q4), so
 * y is [r,pw,ph,c].  rois [r,4] (x1,y1,x2,y2) px, all pooled from image 0 of fmap; roi_batch is not read (it must be
 * NULL when n > 1).  C a multiple of 8, ph, pw >= 1, 2 * (ph + pw) <= 64. */
int lumi_op_roi_pool(const float* fmap, int n, int fh, int fw, int c, const float* rois, const int32_t* roi_batch,
                     int r, float im_h, float im_w, int ph, int pw, float* y, void* stream);

/* The ROI kernel instance lumi_op_roi_pool / the engine launch for c channels at a ph x pw pooled size: 0-2 the
 * row-walk kernel at 6 / 5 / 4 resident CTAs per SM, 3-4 the column-walk kernel at 4 / 8 channels per lane, 5-8 the
 * cell kernel <channels per lane, rois per CTA, warps> = <8,4,4>, <8,4,8>, <8,1,8>, <4,1,8>; -1 when no instance
 * takes the shape.  Honours LUMI_ROI_KERNEL, _MINB, _COLS_CPL, _CPL, _RB and _NW (each read once per process).  Host
 * only. */
int lumi_roi_kernel(int c, int ph, int pw);

/* The ROI stage as the engine runs it on n images: fmap [n,fh,fw,c] fp32, rois [n,rmax,4] (x1,y1,x2,y2) px, counts [n]
 * valid rois per image or NULL (all rmax), all on DEVICE.  kernel: -1 for lumi_roi_kernel(c, ph, pw), else a code of
 * lumi_roi_kernel (LUMI_EINVAL when its shape preconditions fail).  Outputs, each NULL or DEVICE: pooled
 * [n*rmax,pw,ph,c] and mean [n*rmax,c], the fused tf.reduce_mean over the pooled cells; at least one is required.
 * Rows r >= counts[img] come out 0.  Both are written through the engine's fp16x2 split planes, which start out as
 * NaN, so an element the kernel skips reads back as NaN. */
int lumi_op_roi_pool_batched(const float* fmap, int n, int fh, int fw, int c, const float* rois, const int32_t* counts,
                             int rmax, float im_h, float im_w, int ph, int pw, int kernel, float* pooled, float* mean,
                             void* stream);

/* tf.reduce_mean(x, [1, 2]) through split planes, as the engine's RCNN head runs it after the resnet_v1_101 tail and
 * for pooled features that did not fuse the mean: x [r,h,w,c] fp32 on DEVICE (split into planes first), y [r,c]. */
int lumi_op_spatial_mean(const float* x, int r, int h, int w, int c, float* y, void* stream);

/* Softmax over the first cols entries of each of rows rows of x (in_stride floats apart, >= cols); y [rows,cols]
 * dense.  The engine reads the C + 1 class logits out of fc rows 5C + 1 wide.  DEVICE pointers. */
int lumi_op_softmax_rows(const float* x, int rows, int cols, int in_stride, float* y, void* stream);

/* Sort scores descending (ties: lower index first); idx_out [n] int32. */
int lumi_op_sort_desc(const float* scores, int n, int32_t* idx_out, void* stream);

/* Greedy NMS == tf.image.non_max_suppression on boxes [n,4] (x1,y1,x2,y2),
 * ALREADY sorted by score desc.  keep [max_out] int32 indices, *num_keep on device. */
int lumi_op_nms_sorted(const float* boxes_sorted, int n, float iou_threshold, int max_out,
                       int32_t* keep, int32_t* num_keep, void* stream);

/* Which NMS path `problems` lists of up to ncap sorted candidates take at this IoU threshold: 0 the one-phase staged
 * scan, 1 the two-phase NMS (>= 3 lists of >= 4096 candidates, 0 < thr < inf, or env LUMI_NMS_LAZY=1; =0 turns it
 * off), 2 the one-phase unstaged scan (lists too long for the staged scan's shared memory).  Host only. */
int lumi_nms_path(int problems, int ncap, float iou_threshold);

/* lumi_op_nms_sorted on `problems` lists at once, through the engine's batched NMS: boxes_sorted [problems,cap,4],
 * nvalid [problems] int32 (each in [0, cap]), all on DEVICE.  keep [problems,max_out] int32 (entries past
 * num_keep[p] undefined), num_keep [problems].  The path is lumi_nms_path(problems, cap, iou_threshold). */
int lumi_op_nms_batched(const float* boxes_sorted, const int32_t* nvalid, int problems, int cap, float iou_threshold,
                        int max_out, int32_t* keep, int32_t* num_keep, void* stream);

/* The RPN proposal chain as the engine runs it on a (half-)batch: cls / box hold nimg images at the given per-image
 * strides (floats), each [na / A cells][channels]; anchor a of a cell reads its two class values at
 * cell * cls_stride + cls_off + 2a (logits = 1: softmax logits, 0: probabilities, foreground second) and its deltas at
 * cell * box_stride + box_off + 4a.  anchors [na,4] shared by the images.  The workspace holds cap >= na candidates
 * per image (the engine sizes it for its largest image) and min(cap, pre_nms_top_n) after the top-n cut.  Outputs
 * proposals [nimg,post_nms_top_n,4], scores [nimg,post_nms_top_n], counts [nimg] on DEVICE. */
int lumi_op_rpn_proposals_batched(const float* cls, const float* box, int64_t img_stride_cls, int64_t img_stride_box,
                                  int A, const float* anchors, int nimg, int na, int cap, float im_h, float im_w,
                                  int pre_nms_top_n, int post_nms_top_n, float nms_threshold, float min_prob,
                                  int filter_outside, int clip_after_nms, int apply_nms, int logits, int cls_stride,
                                  int cls_off, int box_stride, int box_off, float* proposals, float* scores,
                                  int32_t* counts, void* stream);

/* The per-class detection chain as the engine runs it on nimg images: boxes_in [nimg][r][4] at boxes_img_stride
 * floats per image (0: one set of anchors shared by all images), row_counts [nimg] valid rows per image or NULL (all
 * r), cls_prob rows of prob_stride floats and deltas rows of delta_stride floats ([nimg * r] rows each; deltas hold 4
 * values per class, or 4 shared ones when shared_deltas = 1).  Outputs objects [nimg,total_max,4], labels, probs
 * [nimg,total_max], count [nimg] and, when records is not NULL, the packed rows of lumi_set_record_output
 * [nimg][1 + 6 * total_max], all on DEVICE. */
int lumi_op_class_detections_batched(const float* boxes_in, int64_t boxes_img_stride, const int32_t* row_counts,
                                     const float* deltas, const float* cls_prob, int nimg, int r, int nc, float im_h,
                                     float im_w, float var0, float var1, float min_prob, float nms_threshold,
                                     int class_max, int total_max, int shared_deltas, int prob_stride,
                                     int delta_stride, float* objects, int32_t* labels, float* probs, int32_t* count,
                                     float* records, void* stream);

/* RPN proposal chain (rpn_proposal.py:41-197) for one image: cls_prob [na,2], bbox_pred [na,4],
 * anchors [na,4] float; outputs proposals [post_nms_top_n,4], scores, count (device). */
int lumi_op_rpn_proposals(const float* cls_prob, const float* bbox_pred, const float* anchors, int na,
                          float im_h, float im_w, int pre_nms_top_n, int post_nms_top_n, float nms_threshold,
                          float min_prob, int filter_outside, int clip_after_nms,
                          float* proposals, float* scores, int32_t* count, void* stream);

/* Per-class detection chain (rcnn_proposal.py:46-164 when ssd_order = 0; ssd/proposal.py:41-171 when 1)
 * for one image: boxes_in [r,4] (proposals or anchors), deltas [r,4*nc] (rcnn) or [r,4] (ssd),
 * cls_prob [r,nc+1]; outputs objects [total_max,4], labels, probs, count (device). */
int lumi_op_class_detections(const float* boxes_in, const float* deltas, const float* cls_prob, int r, int nc,
                             float im_h, float im_w, float var0, float var1, float min_prob, float nms_threshold,
                             int class_max, int total_max, int ssd_order,
                             float* objects, int32_t* labels, float* probs, int32_t* count, void* stream);

/* ---- input path (SURVEY 8f-2): JPEG decode on the GPU with nvJPEG (bound at run time; LUMI_ECUDA when the
 * library is not installed).  Replaces PIL's Image.open(...).convert('RGB') of predict.py:69-79 for JPEG files.
 * data/nbytes: the encoded file.  out: RGB interleaved uint8 [h,w,3] -- host pointer (out_on_device = 0) or device
 * pointer (1) of `capacity` bytes; out = NULL only queries *height / *width.  Note: nvJPEG and libjpeg differ by
 * +-1..2 grey levels on chroma edges, so detections on nvJPEG pixels are not bit-comparable with the reference's. */
int lumi_decode_jpeg(const unsigned char* data, size_t nbytes, int device, unsigned char* out, size_t capacity,
                     int out_on_device, int* height, int* width);
const char* lumi_jpeg_last_error(void);

/* ---- measurement hook (no reference counterpart, not on the predict path): do the 32 lanes of one `mbarrier.try_wait` warp instruction ever get different answers?  One CTA
 * per SM, `rounds` barrier phases; *diverged_rounds = rounds (summed over CTAs) in which the lanes' attempt counts differed. */
int lumi_op_trywait_probe(int rounds, unsigned* diverged_rounds, unsigned* max_spread, unsigned* mean_attempts);

#ifdef __cplusplus
}
#endif
#endif /* LUMINOTH_B200_H */
