/* siammask_b200 — C ABI of the H100-native SiamMask per-frame inference hot path.
 *
 * The reference (foolwood/SiamMask) has no FFI for this path: the boundary is the duck-typed Python
 * object `state['net']` used by tools/test.py (siamese_init :155, siamese_track :201,203,257).  The entry
 * points below are what a binding for that object needs; each cites the reference method it replaces.
 * `siammask_b200/custom.py` is the ctypes binding that restores the Python API on top of them
 * (see INTEGRATION.md).
 *
 * Conventions: plain pointers and sizes only.  All *device* pointers are fp32 NCHW exactly as the
 * reference exchanges them (tools/test.py:61-64,205-206); the caller owns every I/O buffer, the engine
 * owns weights, workspace and per-slot caches.  Work is enqueued on `stream` (a cudaStream_t passed as
 * void*) and returns without synchronising.  Return value 0 = ok, negative = error with the message in
 * sm_last_error() (thread local).  Nothing here ever falls back to a CPU implementation: without a
 * CUDA device every compute entry point fails with an error.
 */
#ifndef SIAMMASK_B200_H
#define SIAMMASK_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct sm_engine sm_engine;

enum { SM_PRECISION_EXACT = 0, /* fp16 hi+lo operands, 3 tensor-core MMAs per k-step: fp32-class results */
       SM_PRECISION_FAST = 1   /* single fp16 MMA per k-step */ };
enum { SM_BACKEND_TENSOR = 0,  /* wgmma implicit-GEMM convolutions */
       SM_BACKEND_SIMT = 1     /* CUDA-core reference convolutions (debug / bisecting only) */ };
enum { SM_TRACK_MASK_FEATURES = 1, /* keep p0/p1/p2 + mask corr feature for sm_refine (track_mask) */
       SM_TRACK_MASK_HEAD = 2      /* also evaluate the 256->3969 mask head (dead under --refine) */ };

typedef struct sm_config {
  int32_t search_size;   /* hp.instance_size: 255 (config_davis.json) or e.g. 383 */
  int32_t max_batch;     /* largest B passed to sm_track / sm_template */
  int32_t num_slots;     /* tracker streams whose template kernels stay cached on the device */
  int32_t precision;     /* SM_PRECISION_* */
  int32_t backend;       /* SM_BACKEND_* */
  int32_t anchor_num;    /* len(ratios)*len(scales), models/siammask_sharp.py:17 (5) */
  int32_t with_mask;     /* build mask_model + refine_model (siammask_sharp) or RPN only (siamrpn_resnet) */
} sm_config;

/* One checkpoint tensor: reference state-dict name (SURVEY App. B), host fp32 data, shape. */
typedef struct sm_tensor_desc {
  const char* name;
  const float* data;
  int32_t ndim;
  int64_t shape[4];
} sm_tensor_desc;

/* Custom.__init__ — experiments/siammask_sharp/custom.py:162-168 */
int sm_engine_create(const sm_config* cfg, sm_engine** out);
void sm_engine_destroy(sm_engine* e);

/* load_pretrain + model.load_state_dict — utils/load_helper.py:30-54.  Folds eval-mode BatchNorm
 * (eps 1e-5) into the convolutions, repacks to the kernels' layouts and uploads.  Copies; the caller
 * keeps ownership of `tensors`. */
int sm_engine_load_weights(sm_engine* e, const sm_tensor_desc* tensors, int32_t n);

/* The packed device weight arena (layout is a pure function of sm_config).  Multi-GPU init: rank 0
 * calls sm_engine_load_weights, every rank broadcasts [ptr, ptr+bytes) with NCCL, the other ranks
 * call sm_engine_adopt_weights. */
int sm_engine_weight_blob(sm_engine* e, void** dev_ptr, size_t* bytes);
int sm_engine_adopt_weights(sm_engine* e);

/* Static activation scales.  Activations live in HBM as two fp16 planes of value * 2^s (22 significant bits), so
 * |value * 2^s| must stay below 65504 and well above fp16's subnormals.  Without calibration s = 0 everywhere, which fits
 * BN-normalised checkpoints (activations O(1)..O(10^3)).  sm_engine_calibrate runs template + track_mask (+ mask head)
 * + refine on a representative sample batch (z f32 [B,3,127,127], x f32 [B,3,S,S], device; slots 0..B-1 are
 * overwritten), measures max |value| per tensor and re-packs every layer with per-tensor power-of-two scales chosen
 * for ~64x headroom: conv + BN is linear and ReLU / max-pool / crops commute with a positive scale, so the scales are
 * free at run time and results are unchanged.  Needs the weights to have come through sm_engine_load_weights on this
 * engine; the scales travel inside the weight arena (broadcast / packed file).
 * sm_engine_status: synchronises and returns flags; bit 0 = some activation left fp16's range since the last calibrate /
 * engine creation (results invalid: calibrate with representative data); bit 1 = a slot table passed to
 * sm_template_slots / sm_step_slots held an entry outside [0, num_slots): that stream was skipped and its outputs are
 * undefined. */
int sm_engine_calibrate(sm_engine* e, int32_t B, const float* z_nchw, const float* x_nchw, void* stream);
int sm_engine_status(sm_engine* e, int32_t* flags);

/* Custom.template — custom.py:173-174.  z: device f32 [B,3,127,127].  Caches, for slots
 * slot0..slot0+B-1, the template feature and the three conv_kernel outputs (models/rpn.py:64),
 * which the reference recomputes every frame. */
int sm_template(sm_engine* e, int32_t slot0, int32_t B, const float* z_nchw, void* stream);

/* sm_template with a slot table: stream b's kernels are cached in slot slots[b].  slots: device int32 [B], owned by the
 * caller; precondition: entries distinct and in [0, num_slots) (an entry out of range skips that stream and sets bit 1
 * of sm_engine_status).  Lets tracker streams join a running batch in any free slots. */
int sm_template_slots(sm_engine* e, int32_t B, const int32_t* slots, const float* z_nchw, void* stream);

/* Custom.track / Custom.track_mask — custom.py:176-186.  x: device f32 [B,3,S,S] paired with slots
 * slot0..slot0+B-1.  cls: f32 [B,2A,R,R], loc: f32 [B,4A,R,R], mask: f32 [B,3969,R,R] or NULL.
 * flags: SM_TRACK_*. */
int sm_track(sm_engine* e, int32_t slot0, int32_t B, const float* x_nchw, float* cls, float* loc, float* mask,
             int32_t flags, void* stream);

/* Custom.track_refine — custom.py:188-190 -> Refine.forward(test=True) :131-154.  pos: device int32 [B,2]
 * (dy,dx) per stream; out: device f32 [B,127*127].  Uses the features cached by the preceding
 * sm_track(..., SM_TRACK_MASK_FEATURES) with the same B. */
int sm_refine(sm_engine* e, int32_t B, const int32_t* pos, float* out, void* stream);

/* get_subwindow_tracking — tools/test.py:67-110 — on the device: frames uint8 HWC (BGR as cv2.imread returns them),
 * frame b at frames + b*frame_stride (stride 0 = all streams share one frame); boxes int32 [B][8] (device) =
 * {context_xmin, context_ymin, original_sz, uint8(avg_chans[0..2]), 0, 0} in frame coordinates BEFORE padding (the
 * window may leave the frame; those pixels take the average colour, :89-100).  Resizes original_sz -> model_size
 * bit-exactly like cv2.resize(INTER_LINEAR) on 8-bit data and writes out f32 [B][3][model][model] (:61-64). */
int sm_crop_resize(const uint8_t* frames, size_t frame_stride, int32_t H, int32_t W, const int32_t* boxes, int32_t B,
                   int32_t model_size, float* out, void* stream);

/* sm_crop_resize where stream b crops frame frame_idx[b] (device int32 [B]; each entry indexes a frame that exists):
 * K objects of G videos read the G frames in place instead of a per-stream copy. */
int sm_crop_resize_indexed(const uint8_t* frames, size_t frame_stride, int32_t H, int32_t W, const int32_t* frame_idx,
                           const int32_t* boxes, int32_t B, int32_t model_size, float* out, void* stream);

/* Images of different sizes in one packed buffer (the *_ragged / *_sized entry points below): the images are
 * concatenated into one contiguous device buffer, and a device table of sm_image_desc locates each.  offset counts
 * elements of the buffer's type from the buffer's start: a uint8 HWC/BGR frame is h*w*3 bytes, an annotation or label
 * map h*w bytes, a pasted mask h*w floats.  An entry with h == 0 or w == 0 is an empty image (nothing reads it). */
typedef struct sm_image_desc {
  int64_t offset;
  int32_t h, w;
} sm_image_desc;

/* sm_crop_resize_indexed over frames of different sizes: stream b crops the frame frame_desc[frame_idx[b]] (base
 * frames + offset, h rows, w columns) of the packed uint8 buffer `frames`.  Arithmetic and output as sm_crop_resize.
 * frame_desc, frame_idx (device int32 [B]) and boxes are device tables; B == 0 is a no-op. */
int sm_crop_resize_ragged(const uint8_t* frames, const sm_image_desc* frame_desc, const int32_t* frame_idx,
                          const int32_t* boxes, int32_t B, int32_t model_size, float* out, void* stream);

/* Mask paste-back — crop_back() in siamese_track, tools/test.py:263-282: cv2.warpAffine(src f32 [B][src_h][src_w],
 * maps f64 [B][6] (forward 2x3 maps, device), (dst_w, dst_h), INTER_LINEAR, BORDER_CONSTANT, border_value), bit-exact
 * with OpenCV's fixed-point coordinate generation.  dst f32 [B][dst_h][dst_w].  All device pointers. */
int sm_warp_affine(const float* src, int32_t src_h, int32_t src_w, const double* maps, float* dst, int32_t dst_h,
                   int32_t dst_w, float border_value, int32_t B, void* stream);

/* sm_warp_affine for B square side x side sources into destinations of different sizes: image b is written at
 * dst + dst_desc[b].offset, dst_desc[b].h x dst_desc[b].w floats (device table).  max_h / max_w bound every h / w
 * (they size the grid).  Each image equals sm_warp_affine's output for its own size, bit for bit. */
int sm_warp_affine_ragged(const float* src, int32_t side, const double* maps, float* dst, const sm_image_desc* dst_desc,
                          int32_t B, int32_t max_h, int32_t max_w, float border_value, void* stream);

/* Multi-object label map of track_vos — tools/test.py:480-523 — fused with the paste-back, for G videos of one frame
 * size H x W.  The objects of video g are entries obj_offsets[g] .. obj_offsets[g+1]-1 (device int32 [G+1]) of objects
 * (device int32 [n][2] = {kind, arg}):
 *   SM_OBJ_TRACKED: arg = row of masks f32 [rows][side][side] (sigmoid masks) and maps f64 [rows][6] (forward maps of
 *                   sm_tracker_update); value = cv2.warpAffine(mask, map, (W, H), INTER_LINEAR, BORDER_CONSTANT, -1),
 *                   bit for bit with sm_warp_affine;
 *   SM_OBJ_INIT:    arg = label id; value = anno[g] == id ? 1 : 0 (anno uint8 [G][H][W]; may be NULL without such objects);
 *   SM_OBJ_IDLE:    value = -1.
 * labels uint8 [G][H][W] = (first argmax over the video's objects + 1) * (max > seg_thr), compared in double like the
 * reference's float64 pred_masks; label k+1 is the video's k-th object, not its annotation id.  Precondition: at most
 * 255 objects per video (a video with more is labelled 0 everywhere instead of with wrapped labels).  Per-object
 * frames are never materialised.  Objects whose four taps all miss the mask are skipped at that pixel, which is exact
 * for seg_thr >= -1 (required). */
enum { SM_OBJ_IDLE = 0, SM_OBJ_TRACKED = 1, SM_OBJ_INIT = 2 };
int sm_paste_labels(const float* masks, int32_t side, const double* maps, const uint8_t* anno, const int32_t* obj_offsets,
                    const int32_t* objects, int32_t G, int32_t H, int32_t W, double seg_thr, uint8_t* labels,
                    void* stream);

/* sm_paste_labels fused with the per-object IoU counts of MultiBatchIouMeter (tools/test.py:421-456), the score
 * track_vos computes for a video, for one frame of G videos.  masks, side, maps, anno, obj_offsets, objects, seg_thr and
 * labels are those of sm_paste_labels, and labels equals its output bit for bit; anno is required.  target_ids (device
 * int32 [n], n = obj_offsets[G]) is the annotation value entry i is scored against (1..255), or -1 for an entry that is
 * not scored (it matches no pixel).  For each of the T thresholds thrs (device f64 [T]), label_t = (first argmax + 1) *
 * (max > thrs[t]) in double, and counts (device int32 [n][T][2]) = (intersection, union) of label_t == k+1 and
 * anno[g] == target_ids[i], where k is entry i's position within its video.  The call sets counts itself.
 * Preconditions:
 *   - T <= 32 and thrs[t] >= -1: objects whose four taps all miss the mask are skipped, which is exact only for
 *     thresholds >= -1; a threshold below -1 yields counts (-1, -1);
 *   - the scored target ids of a video are unique;
 *   - at most 255 objects per video (a video with more gets no labels and no counts).
 * One pass over each frame; per-object frames are never materialised.  All pointers are device pointers. */
int sm_paste_labels_iou(const float* masks, int32_t side, const double* maps, const uint8_t* anno,
                        const int32_t* obj_offsets, const int32_t* objects, const int32_t* target_ids, int32_t G,
                        int32_t H, int32_t W, double seg_thr, uint8_t* labels, const double* thrs, int32_t T,
                        int32_t* counts, void* stream);

/* Fused paste-back + IoU counts of IouMeter.add (utils/average_meter_helper.py:71-113), the per-frame score of
 * tools/tune_vos.py, for B streams of one frame size H x W.  Stream b's value v at a pixel is
 * cv2.warpAffine(masks[b], maps[b], (W, H), INTER_LINEAR, BORDER_CONSTANT, -1), bit for bit with sm_warp_affine
 * (masks f32 [B][side][side] sigmoid masks, maps f64 [B][6] forward maps of sm_tracker_update*), and the annotation is
 * anno[video[b]] (anno uint8 [G][H][W], video int32 [B] in [0, G), not checked here).  For each of the T <= 32
 * thresholds thrs (f64 [T]), counts int32 [B][T][2] = (intersection, union) of pred = v > thrs[t] and target = anno > 0.
 * The comparison is made in double, (double)v > thr, as NumPy 2 evaluates float32_array > np.float64; NumPy 1.x
 * compared in float32, which differs only where v == (float)thr and (float)thr rounded up.
 * Precondition: thrs[t] >= -1.  It makes pixels whose four taps all miss the mask exact without visiting them (their
 * value is -1); a threshold below -1 yields counts (-1, -1) instead.  Frame-sized per-stream masks are never
 * materialised; all pointers are device pointers. */
int sm_mask_iou(const float* masks, int32_t side, const double* maps, const uint8_t* anno, const int32_t* video,
                int32_t B, int32_t H, int32_t W, const double* thrs, int32_t T, int32_t* counts, void* stream);

/* Init boxes of track_vos (tools/test.py:483-496): for each query q = (video g, label id) of queries (device int32
 * [Q][2]), boxes[q] (device int32 [Q][4]) = x, y, w, h = cv2.boundingRect(anno[g] == id); (0, 0, 0, 0) when no pixel
 * carries the id. */
int sm_label_boxes(const uint8_t* anno, int32_t G, int32_t H, int32_t W, const int32_t* queries, int32_t Q, int32_t* boxes,
                   void* stream);

/* sm_paste_labels / sm_paste_labels_iou / sm_label_boxes for G videos of different sizes: video g's annotation is read
 * from, and its labels are written to, anno / labels + video_desc[g].offset (h x w bytes; video_desc is a device
 * table of G entries).  max_h / max_w bound every h / w (they size the grid).  Each video's labels, counts and boxes
 * equal those of the uniform entry point run on that video alone, bit for bit.  G == 0 / Q == 0 is a no-op. */
int sm_paste_labels_ragged(const float* masks, int32_t side, const double* maps, const uint8_t* anno,
                           const int32_t* obj_offsets, const int32_t* objects, const sm_image_desc* video_desc, int32_t G,
                           int32_t max_h, int32_t max_w, double seg_thr, uint8_t* labels, void* stream);
int sm_paste_labels_iou_ragged(const float* masks, int32_t side, const double* maps, const uint8_t* anno,
                               const int32_t* obj_offsets, const int32_t* objects, const int32_t* target_ids,
                               const sm_image_desc* video_desc, int32_t G, int32_t max_h, int32_t max_w, double seg_thr,
                               uint8_t* labels, const double* thrs, int32_t T, int32_t* counts, void* stream);
int sm_label_boxes_ragged(const uint8_t* anno, const sm_image_desc* video_desc, int32_t G, const int32_t* queries,
                          int32_t Q, int32_t* boxes, void* stream);

/* Region overlap of the VOT supervised protocol (tools/test.py:341-354): for each of B pairs, overlap[b] (device f32
 * [B]) = the VOT toolkit's compute_polygon_overlap(poly_a[b], poly_b[b], bounds left 0, top 0, right W, bottom H) as
 * pyvotkit's vot_overlap calls it (flags 0: the non-legacy rasteriser), bit for bit.  poly_a / poly_b are device f32
 * [B][8] 4-point polygons x0, y0, .. x3, y3.  The restatement keeps C's types: float for the bounds, the offset into the
 * union box, pixelY - y[i] and the edge deltas; double for the node x and the a1 / a2 ratio test; no FMA contraction;
 * round() half away from zero; (int) truncating.  Each mask row is the union of its spans (a pixel covered twice counts
 * once), and columns up to W inside the union box count.  Both early exits return 0; an empty union returns x86's 0/0
 * NaN (0xFFC00000), which the protocol treats as "not lost".
 * Precondition: every coordinate is finite and within +-2^20 px.  Beyond that C's (int) of an out-of-range double is
 * undefined and x86 and the GPU disagree; the Python wrapper checks it.  (W+1)*(H+1) must fit in int32. */
int sm_vot_overlap(const float* poly_a, const float* poly_b, int32_t B, int32_t W, int32_t H, float* overlap, void* stream);

/* sm_vot_overlap with per-pair bounds: pair b uses (W, H) = wh[b] (device int32 [B][2]), same types and rounding.
 * Each (W+1)*(H+1) must fit in int32 and W, H >= 1 (not checked on the device; the Python wrapper checks them). */
int sm_vot_overlap_sized(const float* poly_a, const float* poly_b, int32_t B, const int32_t* wh, float* overlap,
                         void* stream);

/* Per-frame overlaps of VOT results as pysot's calculate_accuracy computes them (utils/pysot/utils/statistics.py) for
 * a result file written by track_vot and read back by load_tracker.  rec: device f64 [>= T][S][5], frame f of stream s
 * at rec[(f * S + s) * 5] = (entry code, x, y, w, h) with code 1 init, 2 lost, 0 skipped, 3 a location.  gt: device
 * f32 [G][gt_frames][8] gt polygons; seq: device int32 [S] the sequence g of each stream; wh: device int32 [S][2] the
 * stream's (W, H); lengths: device int32 [S] the stream's T.
 * Outputs device f32 [T][S]: acc with bounds (W, H) and burn-in 10 (NaN on the init entry and the 9 frames after it),
 * eao with bounds (W - 1, H - 1) and no burn-in.  An entry other than a location is NaN (0x7FC00000) in both, as is
 * every frame f >= lengths[s].  A location passes through the result file first: each value v becomes
 * rint((double)(float)v * 1e4) / 1e4 (the "%.4f" print and strtod read-back), and the rectangle's vertices x + w, y + h
 * are summed in double and stored as floats, as pyvotkit's vot_overlap does.  The overlap itself is sm_vot_overlap's
 * rasteriser, bit for bit, with the location's rectangle as poly_a.
 * Preconditions (not checked on the device): lengths[s] <= T; 0 <= seq[s] < G; 2 <= W, H and (W+1)*(H+1) fits in
 * int32; the gt rows and the rounded rectangles inside sm_vot_overlap's coordinate precondition.  2 * T * S <= INT32_MAX. */
int sm_vot_trajectory_overlap(const double* rec, int32_t T, int32_t S, const float* gt, int32_t gt_frames,
                              const int32_t* seq, const int32_t* wh, const int32_t* lengths, float* acc, float* eao,
                              void* stream);

/* Bytes of device workspace sm_vot_eao_accumulate needs for T frames and S streams (0 for bad sizes). */
size_t sm_vot_eao_workspace_size(int32_t T, int32_t S);

/* Adds S streams' VOT scores (the 'all' tag of pysot's AccuracyRobustnessBenchmark and EAOBenchmark) into R score rows.
 * eao / acc: the planes of sm_vot_trajectory_overlap, f32 [T][S]; rec: the same record (its entry codes are read);
 * lengths: device int32 [S]; combo: device int32 [S], the score row of each stream (a row outside [0, R) takes no
 * stream).  Score state, device f64: num / den [R][cap], tail_in / tail_out [R][2], stats [R][4].
 *   num[r][i] += sum of fweight * mean(fragment[1..i]) and den[r][i] += sum of fweight over the fragments of row r's
 *   streams alive at column i (1 <= i < cap), with EAOBenchmark's fragments: for a stream with no lost entry the
 *   overlaps with their NaNs; otherwise one fragment per start point (0 and f + 5 <= T for every lost entry f), NaN
 *   read as 0, zero-padded unless it is the last one.  The expected-overlap curve is num / den (0 where den is 0).
 *   Columns i >= tail_from also receive the non-last fragments of earlier calls: tail_in[r] = (sum of fweight *
 *   fragment sum, sum of fweight); tail_out = tail_in plus this call's.  Grow cap between calls by copying num / den
 *   into a wider zeroed buffer and passing the old cap as tail_from; pass tail_from = cap otherwise.
 *   stats[r] += (sum and count of the non-NaN acc overlaps, number of lost entries, frames) of row r's streams.
 * Streams are visited in ascending order and every output has one writer, so equal inputs give equal bits.
 * Preconditions: lengths[s] <= T <= cap; R <= 65535; tail_in and tail_out do not alias; workspace is device memory of
 * at least sm_vot_eao_workspace_size(T, S) bytes, 8-byte aligned. */
int sm_vot_eao_accumulate(const float* eao, const float* acc, const double* rec, int32_t T, int32_t S,
                          const int32_t* lengths, const int32_t* combo, int32_t R, int32_t cap, int32_t tail_from,
                          const double* tail_in, double* tail_out, double* num, double* den, double* stats,
                          void* workspace, size_t workspace_bytes, void* stream);

/* Score / box post-processing + argmax of siamese_track — tools/test.py:205-254 — on the device, so that
 * sm_track -> sm_select -> sm_refine needs no host round trip.  All pointers are device pointers:
 * cls/loc as returned by sm_track; anchors f32 [A*R*R][4] = (cx,cy,w,h) in generate_anchor order (tools/test.py:113-129);
 * window f32 [A*R*R] (tiled hanning, :157-161); target_sz_in_crop f64 [B][2] = target_sz * scale_x (:226; float64 as
 * in the reference, whose penalty terms are evaluated in float64).
 * Outputs: best_idx int32 [B] (np.argmax of pscore, :237 — incl. its NaN rule: the first NaN wins), pos int32 [B][2] =
 * (delta_y, delta_x) (:253-254), records f32 [B][8] = decoded box cx,cy,w,h of the winner in crop units (:209-212),
 * score, penalty, pscore, best index (exact: < 2^24). */
int sm_select(sm_engine* e, int32_t B, const float* cls, const float* loc, const float* anchors, const float* window,
              const double* target_sz_in_crop, double penalty_k, double window_influence, int32_t* best_idx, int32_t* pos,
              float* records, void* stream);

/* Device-resident tracker state for B concurrent streams — the host arithmetic of siamese_track around the network
 * (tools/test.py:172-200, 239-249, 263-282, 305-315), float64 as numpy evaluates it, so that frame k+1's crop follows
 * from frame k's result without a host round trip.  state f64 [B][4] = target_pos (x, y), target_sz (w, h), device.
 *  sm_tracker_prepare: search window of the next frame -> boxes int32 [B][8] for sm_crop_resize (:180-198, :71-76),
 *    target_sz_in_crop f64 [B][2] for sm_select / sm_step (:226), aux f64 [B][4] = scale_x, round(s_x), crop_box x0, y0.
 *  sm_tracker_update: records f32 [B][8] of sm_select / sm_step + aux -> lr-smoothed, frame-clamped state (:239-249,
 *    :305-315; the penalty of the winner is re-evaluated in float64); maps f64 [B][6] (may be NULL) = forward affine map
 *    of crop_back (:263-275) for sm_warp_affine; out f64 [B][8] (may be NULL) = x, y, w, h, score, penalty, lr, best index.
 *    im_wh int32 [B][2] = frame width, height. */
typedef struct sm_tracker_hp {
  double context_amount, penalty_k, window_influence, lr;   /* utils/tracker_config.py:10-21 / config_davis.json */
  int32_t exemplar_size, instance_size, total_stride, base_size, out_size, reserved;
} sm_tracker_hp;
int sm_tracker_prepare(int32_t B, const double* state, const int32_t* avg_chans, const sm_tracker_hp* hp, int32_t* boxes,
                       double* target_sz_in_crop, double* aux, void* stream);
int sm_tracker_update(int32_t B, double* state, const float* records, const double* aux, const int32_t* im_wh,
                      const sm_tracker_hp* hp, int32_t anchor_num, int32_t score_size, double* maps, double* out,
                      void* stream);
/* sm_tracker_update with per-stream hyper-parameters: hp_table (device f64 [B][3] = penalty_k, window_influence, lr)
 * supplies stream b's penalty_k and lr; context_amount, sizes and strides stay those of *hp.  With every row equal to
 * the struct's values it computes what sm_tracker_update computes, bit for bit. */
int sm_tracker_update_hp(int32_t B, double* state, const float* records, const double* aux, const int32_t* im_wh,
                         const sm_tracker_hp* hp, const double* hp_table, int32_t anchor_num, int32_t score_size,
                         double* maps, double* out, void* stream);

/* One whole frame of siamese_track (tools/test.py:201-261) on the device, all pointers device pointers:
 * sm_track(flags) -> sm_select -> sm_refine at the position sm_select chose (refine_out != NULL needs
 * SM_TRACK_MASK_FEATURES) -> optionally mask_col f32 [B][3969] = mask[b, :, dy, dx] (:259-260; needs
 * SM_TRACK_MASK_HEAD and `mask`).  Unlike the three separate calls, the engine's two lanes run their halves of the
 * batch start to end without meeting in between.  refine_out / mask / mask_col may be NULL. */
int sm_step(sm_engine* e, int32_t slot0, int32_t B, const float* x_nchw, const double* target_sz_in_crop,
            const float* anchors, const float* window, double penalty_k, double window_influence, int32_t flags,
            float* cls, float* loc, float* mask, int32_t* best_idx, int32_t* pos, float* records, float* refine_out,
            float* mask_col, void* stream);

/* sm_step with a slot table: stream b correlates with the template cached in slot slots[b] (device int32 [B], caller
 * owned, entries in [0, num_slots); out-of-range entries as in sm_template_slots).  Under graph replay the table's
 * contents are read at run time, so a caller may rewrite it between calls that reuse the same pointer. */
int sm_step_slots(sm_engine* e, int32_t B, const int32_t* slots, const float* x_nchw, const double* target_sz_in_crop,
                  const float* anchors, const float* window, double penalty_k, double window_influence, int32_t flags,
                  float* cls, float* loc, float* mask, int32_t* best_idx, int32_t* pos, float* records, float* refine_out,
                  float* mask_col, void* stream);

/* sm_step_slots with per-stream hyper-parameters instead of the two scalars: hp is a device f64 [B][3] table of
 * (penalty_k, window_influence, lr) rows (lr is read by sm_tracker_update_hp, not here), so that one batch can run
 * different tracker settings, e.g. a grid search over them.  Stream b's selection, including records[b][5] (its
 * penalty), uses row b.  Like the slot table, the hp table's contents are read at run time under graph replay. */
int sm_step_slots_hp(sm_engine* e, int32_t B, const int32_t* slots, const double* hp, const float* x_nchw,
                     const double* target_sz_in_crop, const float* anchors, const float* window, int32_t flags,
                     float* cls, float* loc, float* mask, int32_t* best_idx, int32_t* pos, float* records,
                     float* refine_out, float* mask_col, void* stream);

/* The same frame through HOST buffers: H2D of x and target_sz_in_crop, sm_step on staging buffers, D2H of the
 * records (always) and of whichever of refine / mask_col / cls / loc are non-NULL.  anchors / window stay device
 * pointers (per-tracker constants, tools/test.py:142-161).  Asynchronous with the ticket protocol of
 * sm_track_host_async (wait with sm_track_host_wait); with SM_TRACK_MASK_HEAD the raw 3969-channel head output stays on
 * the device (the reference reads one column of it, :259-260). */
typedef struct sm_step_io {
  const float* x_host;        /* f32 [B,3,S,S] */
  const double* tsz_host;     /* f64 [B,2] target_sz * scale_x */
  const float* anchors_dev;   /* f32 [A*R*R,4] device */
  const float* window_dev;    /* f32 [A*R*R] device */
  double penalty_k, window_influence;
  int32_t flags;              /* SM_TRACK_* */
  float* records_host;        /* f32 [B,8], required */
  float* refine_host;         /* f32 [B,127*127] or NULL */
  float* mask_col_host;       /* f32 [B,3969] or NULL */
  float* cls_host;            /* f32 [B,2A,R,R] or NULL */
  float* loc_host;            /* f32 [B,4A,R,R] or NULL */
} sm_step_io;
int sm_step_host_async(sm_engine* e, int32_t slot0, int32_t B, const sm_step_io* io, void* stream, int32_t* ticket);

/* Whole step through HOST buffers (pinned recommended): H2D of x, track(+mask features), optional refine,
 * D2H of cls / loc / refine logits, then stream synchronise.  mask_out_host may be NULL (no refine). */
int sm_track_host(sm_engine* e, int32_t slot0, int32_t B, const float* x_host, float* cls_host, float* loc_host,
                  const int32_t* pos_host, float* mask_out_host, void* stream);

/* Asynchronous form of sm_track_host: returns at once with a ticket (0/1); sm_track_host_wait(ticket) blocks
 * until that step's results are in the host buffers.  Two staging sets alternate, so submitting step k+1 before
 * waiting for step k overlaps its H2D (and step k's D2H) with compute.  Host buffers must stay valid (and pinned,
 * for real overlap) until the wait returns.  For B >= 16 the two halves of the batch run on two internal lanes
 * (own streams) that are ordered only by the ticket: the results are defined after sm_track_host_wait, not by
 * `stream` order; the next stream-ordered entry point (sm_template / sm_track / sm_refine / sm_export) joins the lanes
 * into its stream first. */
int sm_track_host_async(sm_engine* e, int32_t slot0, int32_t B, const float* x_host, float* cls_host, float* loc_host,
                        const int32_t* pos_host, float* mask_out_host, void* stream, int32_t* ticket);
int sm_track_host_wait(sm_engine* e, int32_t ticket);

/* conv2d_dw_group — models/rpn.py:32-38, standalone: x f32 [B,C,H,W], k f32 [B,C,kh,kw] ->
 * out f32 [B,C,H-kh+1,W-kw+1], all device pointers. */
int sm_xcorr_depthwise(const float* x, const float* k, float* out, int32_t B, int32_t C, int32_t H, int32_t W,
                       int32_t kh, int32_t kw, void* stream);

/* F.conv2d + folded affine (+ReLU) as a standalone operator, used by the kernel-level parity tests:
 * x f32 NCHW [B,Cin,H,W], w f32 [Cout,Cin,KH,KW], scale/shift f32 [Cout] (may be NULL), out f32 NCHW.
 * backend/precision as in sm_config. */
int sm_conv2d(const float* x, const float* w, const float* scale, const float* shift, float* out, int32_t B,
              int32_t Cin, int32_t H, int32_t W, int32_t Cout, int32_t KH, int32_t KW, int32_t stride, int32_t pad,
              int32_t dil, int32_t relu, int32_t backend, int32_t precision, void* stream);

/* Copies a cached intermediate of the last sm_template / sm_track as f32 NCHW (parity checks):
 * "p0","p1","p2","p3","search","corr_cls","corr_loc","corr_mask","zf".  shape4 receives [B,C,H,W];
 * with out == NULL only the shape is returned. */
int sm_export(sm_engine* e, const char* what, float* out, int64_t* shape4, void* stream);

/* CUDA-graph replay of sm_track / sm_refine (off by default).  A call whose arguments (pointers, batch, flags,
 * stream) repeat is captured on its second occurrence and replayed afterwards: one graph launch instead of ~80
 * kernel launches — for the launch-bound small-batch / single-stream tracker loop. */
int sm_engine_set_graphs(sm_engine* e, int32_t on);

/* Per-launch CUDA-event timing on the caller's stream (bench.py's roofline leg).  While enabled every kernel
 * launch is bracketed by events; sm_profile_dump synchronises and returns tab-separated lines
 * "name\tcategory\tms\tflops\tbytes\n" (algorithmic FLOPs / bytes of that launch) and clears the log.
 * With buf == NULL or cap too small it returns the required size (call again). */
int sm_profile_enable(sm_engine* e, int32_t on);
int64_t sm_profile_dump(sm_engine* e, char* buf, size_t cap);

/* Number of kernel launches the engine has issued since creation (bench.py reports it). */
int64_t sm_launch_count(const sm_engine* e);
/* Device bytes held by the engine (weights + workspace + caches). */
size_t sm_engine_bytes(const sm_engine* e);

const char* sm_last_error(void);
const char* sm_version(void);

#ifdef __cplusplus
}
#endif
#endif /* SIAMMASK_B200_H */
