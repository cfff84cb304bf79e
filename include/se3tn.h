/* libse3tn -- C ABI of the H100-native (sm_90a) se(3)-TrackNet inference hot path.
 *
 * The upstream reference (wenbowen123/iros20-6d-pose-tracking @ 18dc5bac) is pure Python and has
 * no FFI of its own; its boundary is the Python class surface (SURVEY.md section 8b).  Each entry
 * point below is what a ctypes binding on the reference side would call INSTEAD of the cited
 * reference code.  All tensor arguments are plain device pointers owned by the caller (PyTorch in
 * the shipped host layer); every launch is enqueued on the caller's cudaStream_t (pass it as a
 * void*); nothing here synchronises the stream unless stated.  No exceptions or aborts cross the
 * boundary: every function returns SE3TN_OK or a negative code, text via se3tn_last_error().
 * A context is single-threaded; distinct contexts are independent.
 */
#ifndef SE3TN_H
#define SE3TN_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct se3tn_ctx se3tn_ctx;
typedef struct se3tn_track_opts se3tn_track_opts;   /* a tracking call's options (defined below) */

enum {
    SE3TN_OK = 0,
    SE3TN_ERR_INVALID = -1,      /* bad argument (null, size, alignment, unknown id) */
    SE3TN_ERR_CUDA = -2,         /* a CUDA runtime / driver call failed               */
    SE3TN_ERR_NOMEM = -3,
    SE3TN_ERR_STATE = -4,        /* e.g. forward before load_weights                  */
    SE3TN_ERR_UNSUPPORTED = -5   /* device is not sm_90                               */
};

/* Arithmetic of the 17 convolutions (accumulation is always fp32). */
enum {
    SE3TN_PREC_TF32 = 0,    /* wgmma tf32; operands rounded to tf32 (rna): 10-bit mantissas.  Fastest;
                               meets the 1e-3/1e-4 gate only for well-conditioned weights/inputs              */
    SE3TN_PREC_FP32 = 1,    /* plain FFMA direct convolution, no operand rounding (cross-check mode)         */
    SE3TN_PREC_BF16X3 = 2,  /* wgmma bf16 on bf16 hi/lo splits, 3 products per MAC: ~2^-16 relative
                               error (fp32-faithful for the gate) at 1.5x the tensor time of TF32            */
    SE3TN_PREC_BF16 = 3,    /* wgmma bf16, bf16 operands, 1 product per MAC (BASELINE configs[2])     */
    SE3TN_PREC_FP8 = 4,     /* the stems and 64-channel layers as SE3TN_PREC_BF16; the six trunk layers (convAB1 ...
                               {trans,rot}_conv2.conv2) on wgmma e4m3 with e4m3 activations and weights and
                               power-of-two scales.  Needs a weight set's activation scales (se3tn_calibrate_fp8 or
                               se3tn_set_fp8_scales).  Lossy: see DESIGN.md §2 for its measured error             */
    SE3TN_PREC_FP16 = 5     /* wgmma f16 on IEEE fp16 activations (2 bytes per channel, laid out as SE3TN_PREC_BF16)
                               and fp16 weights: the same 11-bit significand as tf32 at the 16-bit MMA rate.  The
                               stems read the bf16x3 input and run the bf16x3 arithmetic, then store fp16.  Encoding
                               rounds to nearest even and saturates |x| > 65504 to +-65504 (no inf).  No scales, no
                               calibration.  A step refuses a weight set with a weight of layers 2-13 above 65504 in
                               magnitude (SE3TN_ERR_STATE).  tf32's accuracy class: DESIGN.md §2                   */
};

/* SE3TN_PREC_FP8's activation scales, one per e4m3 tensor, in this order: CAT (convAB1's input), F1, T4, F2, then
 * H1 of the trans head, H1 of the rot head, H2 of the trans head, H2 of the rot head.  A stored e4m3 code q means
 * q * s.  Every scale is a power of two. */
#define SE3TN_FP8_SCALES 8
/* Headroom H of se3tn_calibrate_fp8: s = 2^ceil(log2(max|x| * H / 448)), so the calibration's largest value lands at
 * or below 448 / H (scripts/fp8_study.py: H = 1 ... 8 move the 6-vector's worst error by under 4 %; 2 is the lowest). */
#define SE3TN_FP8_HEADROOM 2

#define SE3TN_IMAGE_SIZE 176           /* reference dataset_info.yml:15 `resolution`          */
#define SE3TN_WEIGHT_BLOB_FLOATS 13528326u  /* see se3tn_load_weights                          */

/* ---- lifetime ------------------------------------------------------------------------------ */

/* Bytes of device workspace a context for batches of up to `max_batch` pairs needs. */
size_t se3tn_workspace_bytes(int max_batch);

/* Create a context on CUDA device `device` for up to `max_batch` RGB-D pairs per call.
 * `workspace` is a caller-owned device buffer of se3tn_workspace_bytes(max_batch) bytes, 1024-byte
 * aligned, that must outlive the context; pass NULL to let the library cudaMalloc its own.
 * Replaces: the `.cuda()` model placement in Tracker.__init__ (reference predict.py:156-158). */
int se3tn_create(int device, int max_batch, void* workspace, se3tn_ctx** out);
void se3tn_destroy(se3tn_ctx* ctx);

/* Message of the last error on `ctx` (or of the last failed se3tn_create when ctx is NULL). */
const char* se3tn_last_error(se3tn_ctx* ctx);

/* ---- per-object parameters --------------------------------------------------------------------
 * One weight set per object class (reference README.md:132: one checkpoint + mean/std per object).
 * `blob` is HOST memory: SE3TN_WEIGHT_BLOB_FLOATS float32 values produced by the packer
 * (weights.py: eval-mode BatchNorm folded into each conv, OIHW -> [Cout][tap*Cin + c] K-major),
 * in launch order:
 *   W[64][224],b[64]            x2   convA1, convB1        (7x7 s2; K = 7 rows x (8 px x 4 ch))
 *   W[64][576],b[64]            x6   convA2.{conv1,conv2}, convB2.{..}, convB3.{..}
 *   W[256][1152],b[256]              convAB1
 *   W[256][2304],b[256]         x2   convAB2.{conv1,conv2}
 *   W[1024][2304],b[1024]            trans_conv1 ++ rot_conv1 (Cout concatenated)
 *   W[1024][4608],b[1024]       x2   {trans,rot}_conv2.conv1, {trans,rot}_conv2.conv2 (2 groups)
 *   W[6][512],b[6]                   trans_out.0 ++ rot_out.0
 * Replaces: Se3TrackNet.load_state_dict (reference predict.py:151-155). */
int se3tn_load_weights(se3tn_ctx* ctx, int weight_id, const float* blob, size_t n_floats);

/* Device bytes one loaded weight set holds: the blob in fp32 and the conv weights in every storage format (storage.cuh), the
 * fp8 tables and the resident layers' stacked and permuted rows.  Weight ids are any int >= 0; the context's per-id tables
 * take one small row per id up to the largest. */
size_t se3tn_weight_set_bytes(void);

/* Per-object channel statistics (reference predict.py:657-658 mean.npy/std.npy): 8 values each,
 * A's 4 channels then B's.  `is_f64` selects the arithmetic of the normalisation so that it
 * reproduces numpy's for float32 resp. float64 mean/std arrays (data_augmentation.py:159-163). */
int se3tn_set_stats(se3tn_ctx* ctx, int weight_id, const void* mean8, const void* std8, int is_f64);

/* SE3TN_PREC_FP8's activation scales of weight set `weight_id` (SE3TN_FP8_SCALES values, the order above).
 * se3tn_calibrate_fp8 runs the SE3TN_PREC_BF16X3 forward of the set on n normalised pairs A, B (as se3tn_forward
 * takes them; n <= max_batch), reduces max|x| over each e4m3 tensor as stored, and sets s = 2^ceil(log2(max|x| *
 * SE3TN_FP8_HEADROOM / 448)) (1 where max|x| is 0).  It synchronises the device.
 * se3tn_set_fp8_scales sets saved ones: non-finite, non-positive or non-power-of-two values return SE3TN_ERR_INVALID.
 * se3tn_get_fp8_scales copies them out; a set without scales returns SE3TN_ERR_STATE.
 * The scales live at fixed device addresses: a captured step replays with the values set last.  An SE3TN_PREC_FP8
 * step for a set without scales returns SE3TN_ERR_STATE and launches nothing; se3tn_load_weights drops a set's scales. */
int se3tn_calibrate_fp8(se3tn_ctx* ctx, int weight_id, const float* A, const float* B, int n, void* stream);
int se3tn_set_fp8_scales(se3tn_ctx* ctx, int weight_id, const float* scales, int n_scales);
int se3tn_get_fp8_scales(se3tn_ctx* ctx, int weight_id, float* scales, int n_scales);

/* ---- the hot path ---------------------------------------------------------------------------- */

/* K0.  For each of n tracks: bbox of the previous pose (reference Utils.py:302-316), zero-padded
 * window + nearest-neighbour resize of the observed frame to 176x176 (Utils.py:320-359), depth
 * offset/clip (data_augmentation.py:134-144), channel normalisation (:154-164) and packing
 * (:179-189).  Results land in the context's conv-input buffers; optional outputs (any may be
 * NULL): out_A/out_B float32 (n,4,176,176) exactly as TrackDataset.processData returns them
 * (datasets.py:136-137), crop_rgb uint8 (n,176,176,3) / crop_depth uint16 (n,176,176) exactly
 * as crop_bbox returns them.
 *   frame_rgb  uint8  (H,W,3) device      frame_depth uint16 (H,W) device, millimetres
 *   K          4 doubles HOST: fx, fy, cx, cy
 *   poses      double (n,16) device, row-major 4x4 object-in-camera, metres
 *   object_width double (n) device, millimetres (Tracker.object_width, predict.py:136-142)
 *   rgbA uint8 (n,176,176,3), depthA uint16 (n,176,176) device: render_window's output contract
 *   weight_ids int32 (n) device or NULL (all 0): which mean/std row each track uses */
int se3tn_preprocess(se3tn_ctx* ctx, const uint8_t* frame_rgb, const uint16_t* frame_depth, int H, int W,
                     const double* K, const double* poses, const double* object_width,
                     const uint8_t* rgbA, const uint16_t* depthA, const int32_t* weight_ids, int n,
                     int precision, float* out_A, float* out_B, uint8_t* crop_rgb, uint16_t* crop_depth,
                     void* stream);

/* The post-transform half of TrackDataset.processData (reference datasets.py:136-137 ->
 * data_augmentation.py:124-196) on crops that already exist: rgbA/rgbB uint8 (n,176,176,3),
 * depthA/depthB uint16 (n,176,176), poses double (n,16) (A's pose: both depths are offset by its z).
 * out_A/out_B float32 (n,4,176,176) or both NULL; the conv-input buffers are filled either way. */
int se3tn_normalize(se3tn_ctx* ctx, const uint8_t* rgbA, const uint16_t* depthA,
                    const uint8_t* rgbB, const uint16_t* depthB, const double* poses,
                    const int32_t* weight_ids, int n, int precision, float* out_A, float* out_B, void* stream);

/* compute_bbox (reference Utils.py:302-316): out_bbox int32 (n,4,2), rows (x-,y-),(x-,y+),(x+,y-),(x+,y+),
 * columns (v,u).  K: 4 doubles HOST fx,fy,cx,cy; scale: 3 doubles HOST (the reference passes
 * (1000,1000,1000), or (1000,-1000,1000) for its GL renderer, predict.py:202,232). */
int se3tn_compute_bbox(se3tn_ctx* ctx, const double* poses, const double* K, const double* widths,
                       const double* scale, int32_t* out_bbox, int n, void* stream);

/* crop_bbox (reference Utils.py:320-359): zero-padded window [min v, max v) x [min u, max u) of the
 * frame, cv2.INTER_NEAREST-resized to (out_h, out_w).  bbox int32 (n,4,2) device. */
int se3tn_crop_bbox(se3tn_ctx* ctx, const uint8_t* frame_rgb, const uint16_t* frame_depth, int H, int W,
                    const int32_t* bbox, int n, int out_h, int out_w,
                    uint8_t* crop_rgb, uint16_t* crop_depth, void* stream);

/* Se3TrackNet.forward (reference se3_tracknet.py:81-112).  A, B: float32 (n,4,176,176) contiguous
 * NCHW device tensors.  out_trans/out_rot: float32 (n,3).  out_feature: float32 (n,256,22,22) or
 * NULL.  All n pairs use weight set `weight_id`. */
int se3tn_forward(se3tn_ctx* ctx, int weight_id, const float* A, const float* B, int n,
                  float* out_trans, float* out_rot, float* out_feature, int precision, void* stream);

/* The conv stack on whatever se3tn_preprocess left in the conv-input buffers (tracks
 * [first, first+n) of the last preprocess call). */
int se3tn_forward_preprocessed(se3tn_ctx* ctx, int weight_id, int first, int n,
                               float* out_trans, float* out_rot, float* out_feature, int precision, void* stream);

/* K6.  TrackDataset.processPredict (reference datasets.py:159-175): t' = t + trans*tn,
 * R' = Rodrigues(rot*rn) . R with the reference's float32/float64 dtype chain.
 * poses_in/poses_out double (n,16) device (may alias); trans/rot float32 (n,3) device. */
int se3tn_pose_update(se3tn_ctx* ctx, const double* poses_in, const float* trans, const float* rot,
                      double trans_normalizer, double rot_normalizer, double* poses_out, int n, void* stream);

/* K5.  The label half of TrackDataset.processData (reference datasets.py:141-150, Utils.py:363-367):
 * trans_label = (tB - tA)/tn, rot_label = Rodrigues^-1(normalize_cols(R_B R_A^T))/rn; double (n,3). */
int se3tn_so3_log(se3tn_ctx* ctx, const double* poses_a, const double* poses_b,
                  double trans_normalizer, double rot_normalizer,
                  double* trans_label, double* rot_label, int n, void* stream);

/* Tracker.on_track for n independent tracks of one frame (reference predict.py:217-296 with the
 * renderer's output passed in and the GUI calls dropped): K0 -> conv stack -> K6 on one stream.
 * weight_ids_host: int32 (n) HOST array or NULL (all 0), weight_ids_dev: the same values on the device (or NULL).
 * In the tensor-core modes tracks of ALL object classes share the same 14 conv launches: every work unit
 * takes its weight tensor map / bias from per-set device tables.  Any id order is correct; keeping equal ids
 * contiguous (dist.shard_tracks does) avoids shared-memory weight reloads in the 64-channel layers.  In
 * SE3TN_PREC_FP32 each contiguous run of equal ids is one batched forward.
 * out_trans/out_rot float32 (n,3) device scratch the caller provides (also returned).
 * poses_out may be poses_in: every read of a track's previous pose comes before its update is written, so tracks whose poses
 * stay in one device array, updated in place frame after frame, keep the step's addresses and its CUDA graph.
 * opts: the call's se3tn_track_opts, or NULL for the defaults (see there). */
int se3tn_track_batch(se3tn_ctx* ctx, const uint8_t* frame_rgb, const uint16_t* frame_depth, int H, int W,
                      const double* K, const double* poses_in, const double* object_width,
                      const uint8_t* rgbA, const uint16_t* depthA,
                      const int32_t* weight_ids_host, const int32_t* weight_ids_dev, int n,
                      double trans_normalizer, double rot_normalizer, int precision,
                      float* out_trans, float* out_rot, double* poses_out, const se3tn_track_opts* opts, void* stream);

/* The one exchange step of the sharded path (SURVEY.md 8e): all-gather of the updated poses over an EXISTING NCCL
 * communicator, for hosts that drive libse3tn without torch.distributed (the Python layer uses
 * torch.distributed.all_gather_into_tensor, dist.py).  nccl_comm: the host's ncclComm_t; local_poses double
 * (n_local,16) device; all_poses double (world*n_local,16) device, rank-major; every rank passes the same n_local.
 * NCCL is resolved at run time (dlopen of libnccl.so.2, the copy already loaded in the process if there is one);
 * SE3TN_ERR_UNSUPPORTED if it cannot be found.  The reference has no multi-GPU code to replace (SURVEY.md 2a). */
int se3tn_allgather_poses(se3tn_ctx* ctx, void* nccl_comm, const double* local_poses, double* all_poses, int n_local,
                          void* stream);

/* ---- pose-error metrics (SURVEY.md 8(f) "next" row 1; not on the per-frame path) ----------------------- */

/* Utils.add / Utils.adi (reference Utils.py:72-98) for n (pred, gt) pose pairs against one model point cloud:
 *   ADD   = mean_i |(R_p x_i + t_p) - (R_g x_i + t_g)|,   ADD-S = mean_i min_j |(R_g x_i + t_g) - (R_p x_j + t_p)|
 * model_pts double (m,3), pred / gt double (n,16), out_add / out_adi double (n), all device; either output may be NULL.
 * float64, exhaustive nearest neighbour (the reference uses scipy's cKDTree: same minimum). */
int se3tn_add_adi(se3tn_ctx* ctx, const double* model_pts, int m, const double* pred, const double* gt, int n,
                  double* out_add, double* out_adi, void* stream);

/* VOCap (reference eval_ycb.py:45-64): errs double (n) device, any order -> *out_ap on the HOST (0..1; the
 * reference multiplies by 100 when printing).  Synchronises the stream.  n == 0 or no error below 0.1 m -> 0
 * (the reference raises IndexError there). */
int se3tn_vocap(se3tn_ctx* ctx, const double* errs, int n, double* out_ap, void* stream);

/* Utils.add / Utils.adi for the poses of several objects in ONE launch, as eval_ycbineoat.py's eval_all scores a whole data set
 * (reference eval_ycbineoat.py:75-93, one Utils.add + Utils.adi call per pose there).  pts double (M,3) device: the model points
 * of n_sets objects, concatenated; set_offsets int32 (n_sets+1) HOST: object s owns points [set_offsets[s], set_offsets[s+1]);
 * pose_set int32 (n) HOST: the object of each pose; pred / gt double (n,16), out_add / out_adi double (n), device, either output
 * may be NULL (not both unless n == 0).  Each pose's values are bit-identical to se3tn_add_adi on that pose and its object's points.  SE3TN_ERR_INVALID
 * unless set_offsets starts at 0, increases strictly (no empty set) and ends at M, and every id is in [0, n_sets); nothing is
 * queued then.  The offsets and ids are staged through context-owned device memory, which grows with n and n_sets and is
 * shared with se3tn_vocap_sets: the metric calls of one context go on one stream, or the caller orders them. */
int se3tn_add_adi_sets(se3tn_ctx* ctx, const double* pts, int M, const int32_t* set_offsets, int n_sets, const int32_t* pose_set,
                       const double* pred, const double* gt, int n, double* out_add, double* out_adi, void* stream);

/* VOCap of each object's errors and of all of them in one call (reference eval_ycbineoat.py:95-109, which calls eval_ycb.py:45-64
 * once per object and once on the pooled errors).  errs double (n) and err_set int32 (n) device, any order -> out_ap double
 * (n_sets+1) HOST: the AP of set 0, ..., set n_sets-1, then of all n errors.  Each value is bit-identical to se3tn_vocap on the
 * same errors; a set with no error below 0.1 m, or none at all, gets 0.  Synchronises the stream.  An id outside [0, n_sets) is
 * SE3TN_ERR_INVALID (found on the device, so the call has run).  Scratch as se3tn_add_adi_sets: context-owned, grown only when a
 * call needs more, so a run of calls allocates nothing once the largest has been seen. */
int se3tn_vocap_sets(se3tn_ctx* ctx, const double* errs, const int32_t* err_set, int n, int n_sets, double* out_ap, void* stream);

/* Pose errors of several objects' poses in ONE launch, arguments as se3tn_add_adi_sets (pts, set_offsets, pose_set, pred, gt) plus:
 *   keep uint8 (n) device or NULL (every row kept): a row whose byte is 0 is not scored.
 *   out_errors double (n,4) device: per row the translation error |t - t_gt| in mm, the rotation geodesic angle in degrees
 *     acos(clamp((tr(R^T R_gt) - 1) / 2, -1, 1)) (the trace summed in row-major order), ADD and ADD-S; NaN in all four for a row
 *     that is not kept.  ADD / ADD-S are bit-identical to se3tn_add_adi_sets on the same rows (the same per-pose body).
 *   out_set int32 (n) device or NULL: each kept row's set id, -1 for a row that is not kept, so the caller can leave those rows out
 *     of se3tn_vocap_sets (or of anything else) without reading the mask on the host first.
 * Refusals and scratch as se3tn_add_adi_sets (every id is checked, kept or not); one launch, plain stream order. */
int se3tn_pose_errors_sets(se3tn_ctx* ctx, const double* pts, int M, const int32_t* set_offsets, int n_sets, const int32_t* pose_set,
                           const double* pred, const double* gt, const uint8_t* keep, int n, double* out_errors, int32_t* out_set,
                           void* stream);

/* ---- result videos: each track's model points drawn over its frame (not on the per-frame tracking path) ------------------------- */

/* The frames of the reference's result videos (getResultsYcb, predict.py:424-433; predictSequenceYcb / predictSequenceYcbInEOAT,
 * predict.py:549-560, 612-624) for n tracks of one frame:  model = copy.deepcopy(tracker.object_cloud); model.transform(pose);
 * uvs = project_points(model.points, K); cur_bgr = cvtColor(rgb, RGB2BGR); putText(cur_bgr, "frame:..", (W//2, H-50), ...,
 * color=(255,0,0)); for each uv: circle(cur_bgr, uv, radius=1, color=(0,255,255), thickness=-1); resize(cur_bgr, (W//2, H//2)).
 *   frame_rgb uint8 (H,W,3) device, H and W even; K HOST fx fy cx cy; poses double (n,16) device.
 *   pts double (M,3) device, set_offsets int32 (n_sets+1) HOST and track_set int32 (n) HOST: track i draws points
 *   [set_offsets[s], set_offsets[s+1]) of pts, s = track_set[i], each moved as x' = ((R00 x + R01 y) + R02 z) + t0 (fp64, no
 *   FMA) and projected as u = (x' fx) / z' + cx, v = (y' fy) / z' + cy, rounded half to even.  A point whose u or v is not finite
 *   or beyond +-2^30 is not drawn; a point behind the camera is drawn where it lands.  Each point sets the 5 pixels (u, v),
 *   (u+-1, v), (u, v+-1) that cv2.circle(radius=1, thickness=-1) sets, clipped to the frame.
 *   label_mask uint8 (label_h, W) device, or NULL for no label: rows [label_y0, label_y0 + label_h) of the frame, non-zero where
 *   cv2.putText sets a pixel; those pixels take (255,0,0) under or over the points, as label_order says.
 *   out_bgr uint8 (n, H/2, W/2, 3) device: each track's BGR image, halved as cv2.resize(INTER_LINEAR) halves it, which at an exact
 *   factor of 2 is (a + b + c + d + 2) >> 2 over each 2 x 2 block.
 * Plain stream launches, not part of any track step.  SE3TN_ERR_INVALID, with nothing queued, for an odd H or W, label rows
 * outside the frame, or offsets and ids that se3tn_add_adi_sets would refuse.  The offsets, ids and n one-bit-per-pixel dot masks
 * (n x H x W / 8 bytes) live in the metrics scratch of se3tn_add_adi_sets, on the same terms. */
#define SE3TN_LABEL_UNDER_POINTS 0   /* getResultsYcb, predict.py:427-431 */
#define SE3TN_LABEL_OVER_POINTS  1   /* predictSequenceYcb / YcbInEOAT, predict.py:553-556, 615-618 */
int se3tn_draw_tracks(se3tn_ctx* ctx, const uint8_t* frame_rgb, int H, int W, const double* K,
                      const double* poses, int n,
                      const double* pts, int M, const int32_t* set_offsets, int n_sets,
                      const int32_t* track_set,
                      const uint8_t* label_mask, int label_y0, int label_h, int label_order,
                      uint8_t* out_bgr, void* stream);

/* ---- input A: the rendered previous view (SURVEY.md 8(f) "next" row 2) ------------------------------------- */

/* The CAD model the renderer draws: what VispyRenderer.__init__ uploads as vertex / index buffers (reference
 * vispy_renderer.py:108-129).  HOST arrays, copied: pos float32 (nv,3) metres in the object frame, nrm float32 (nv,3)
 * unit normals, col uint8 (nv,3), faces int32 (nf,3).  mesh_id >= 0; a later call with the same id replaces the model;
 * on failure the id keeps its previous model.  A new model drops the context's captured steps: each is captured again on
 * its next call. */
int se3tn_set_mesh(se3tn_ctx* ctx, int mesh_id, const float* pos, const float* nrm, const uint8_t* col,
                   const int32_t* faces, int nv, int nf);

/* Tracker.render_window for n tracks (reference predict.py:193-215 -> vispy_renderer.py:135-178): the model at `poses`
 * rasterised into each track's 176x176 window (y-flipped orthographic crop of the pinhole projection, depth test LESS,
 * no culling, Lambert + ambient shading) -> rgbA uint8 (n,176,176,3) and depthA uint16 (n,176,176) mm, 0 = background,
 * both device -- exactly the arrays se3tn_preprocess / se3tn_track_batch take.  K: 4 doubles HOST (fx, fy, cx, cy);
 * poses double (n,16) device; object_width double (n) device; mesh_ids int32 (n) device or NULL (all 0). */
int se3tn_render(se3tn_ctx* ctx, const double* K, const double* poses, const double* object_width,
                 const int32_t* mesh_ids, int n, uint8_t* rgbA, uint16_t* depthA, void* stream);

/* The same for either of the reference's two producers of input A (predict.py:161-182 picks one from dataset_info['renderer']):
 *   SE3TN_RENDER_VISPY     what se3tn_render does (H, W ignored).
 *   SE3TN_RENDER_PYRENDER  offscreen_renderer.py:47-83 + predict.py:210-214: the model is drawn into the WHOLE H x W camera image
 *                          (pinhole K, near 0.1 m, far 2 m, ambient light only: unlit vertex colours), the metric depth becomes
 *                          uint16 mm, and crop_bbox (Utils.py:320-359: window from compute_bbox, zero outside the image, nearest-
 *                          neighbour resize to 176 x 176) cuts the track's window out of both.  Only the camera pixels the resize
 *                          picks are ever shaded; the full image is never materialised.  Per-fragment texture lookups of a
 *                          textured .obj are replaced by per-vertex colours. */
#define SE3TN_RENDER_VISPY 0
#define SE3TN_RENDER_PYRENDER 1
int se3tn_render_ex(se3tn_ctx* ctx, const double* K, const double* poses, const double* object_width,
                    const int32_t* mesh_ids, int n, int mode, int H, int W, uint8_t* rgbA, uint16_t* depthA, void* stream);

/* ---- live-sensor depth (SURVEY.md 8(f) "next" row 4) ------------------------------------------------------ */

/* fill_depth as the reference's ROS node applies it to every depth image before tracking (reference Utils.py:455-514,
 * predict_ros.py:38-41: extrapolate=False, bilateral): invert, 5x5 diamond dilate, 5x5 close, fill empties from a 7x7
 * dilation, 5x5 median, bilateral(5, 1.5, 2.0), invert back.  depth_mm uint16 (H,W) device -> out_mm uint16 (H,W) device
 * (= (fill_depth(depth/1e3) * 1000).astype(uint16)) and/or out_m float32 (H,W) metres; either may be NULL.  Bit-identical
 * to OpenCV up to the median; the bilateral's float32 accumulation order differs (|diff| ~ 5e-7 m). */
int se3tn_fill_depth(se3tn_ctx* ctx, const uint16_t* depth_mm, int H, int W, double max_depth,
                     uint16_t* out_mm, float* out_m, void* stream);

/* The same with the reference's two optional arguments (Utils.py:455: extrapolate=False, blur_type='bilateral'):
 * extrapolate != 0: every column's first valid value is extended to the top row and what is still empty takes a 31x31
 * dilation (Utils.py:486-497); blur_type SE3TN_BLUR_GAUSSIAN: cv2.GaussianBlur(5x5, sigma 0) on the valid pixels instead of
 * the bilateral filter (Utils.py:506-510). */
enum { SE3TN_BLUR_BILATERAL = 0, SE3TN_BLUR_GAUSSIAN = 1 };
int se3tn_fill_depth_ex(se3tn_ctx* ctx, const uint16_t* depth_mm, int H, int W, double max_depth, int extrapolate, int blur_type,
                        uint16_t* out_mm, float* out_m, void* stream);

/* ---- depth refinement: point-to-plane ICP of every track against the observed depth, inside the tracking step ---------- */

/* The network's correction is bounded (tanh x normaliser) and as precise as its checkpoint; the step already holds the (filled)
 * observed depth, the crop windows and a rasteriser.  With ICP on (se3tn_track_opts.icp), a render step runs, after the network's
 * last round and before the fit check, M fixed iterations of projective point-to-plane ICP per track, each render (depth +
 * triangle ids at poses_out, 2 launches) -> accumulate (1) -> solve (1), all on `stream` and inside the step's one CUDA graph:
 *   association: every crop pixel u of the render in the crop window of the current pose (se3tn_compute_bbox's window,
 *     se3tn_crop_bbox's nearest mapping, as the fit check takes it) whose triangle id is >= 0 reads frame pixel p; d_obs = the
 *     frame's depth there (the filled frame when the step fills), skipped when 0 or p lies outside the frame.  The ray
 *     r = K^-1 (p_x, p_y, 1) meets the plane of that triangle (unit normal n, posed by the current pose) at q; d_model = 1000 q_z.
 *     Skipped when |n . r / |r|| < 0.1 (grazing) or d_model <= 0.  Inlier: |d_obs - d_model| <= tau_mm; o = r d_obs / 1000.
 *   linear system: e = n . (q - o), J = [(q x n)^T, n^T] for the left increment xi = (w, v); per track the upper 21 entries of
 *     J^T J, J^T e, sum e^2 and the inlier count, summed in a fixed order (bit-reproducible across runs and graph replays).
 *   solve: Cholesky of J^T J in fp64.  count < min_inliers or a pivot <= 1e-12 x the largest diagonal entry: the pose stays bit
 *     for bit.  Otherwise xi = -(J^T J)^-1 J^T e, R <- Exp(w) R, t <- Exp(w) t + v (Rodrigues), poses_out updated in place.
 * Stats row per track, SE3TN_ICP_COLS doubles: inliers, rms_mm (point-to-plane, before the update), step_mm (how far the object's
 * origin moved), step_deg (the rotation's angle); steps are 0 when the update was skipped.  There is no early exit: the launch
 * count is the step's + 4 M.  The ICP render takes context scratch of its own, allocated at max_batch tracks by the first ICP
 * step and never moved: 176 x 176 x (4 bytes of triangle ids + 2 bytes of depth) per track, plus 256 bytes of sums (about
 * 186 KB a track).  The defaults the Python layer uses (tau 20 mm, min_inliers 100) are starting guesses, not tuned on a real
 * sensor; whether ICP improves a trained checkpoint's accuracy has not been measured. */
#define SE3TN_MAX_ICP_ITERATIONS 16
#define SE3TN_ICP_COLS 4      /* inliers, rms_mm (point-to-plane, before the update), step_mm, step_deg (0 when skipped) */
typedef struct se3tn_icp_opts {
    int32_t iterations;       /* 1..SE3TN_MAX_ICP_ITERATIONS */
    int32_t tau_mm;           /* association gate, 1..1000 */
    int32_t min_inliers;      /* 6..176*176 */
    int32_t reserved;         /* 0 */
} se3tn_icp_opts;             /* 16 bytes, no padding */

/* ---- multi-hypothesis tracking: several starts per track, the one whose model fits the frame best kept ---------------- */

/* A track that has slipped further than the network was trained to correct stays lost: the network pulls a pose back from
 * perturbations up to dataset_info's max_translation / max_rotation (reference produce_train_pair_data.py:90-110).  A hypothesis
 * step (se3tn_track_opts.hyp) looks around the previous pose instead of only at it.  For each of n tracks it
 *   1. draws S - 1 start poses around the previous pose P: hypothesis h >= 1 is P . inv(D), D = random_gaussian_magnitude(
 *      max_translation, max_rotation_deg) (reference Utils.py:372-404), composed as produce_train_pair_data.py:110 composes a
 *      training pair (A_in_cam = B_in_cam . inv(B_in_A)); hypothesis 0 is P itself;
 *   2. refines all n x S starts as one n x S-track render step (the options' fill, k rounds and fit check);
 *   3. keeps, per track, the hypothesis whose fit row has the highest inlier fraction inlier / model (compared exactly as int64
 *      cross products; model = 0 ranks last), then the lowest mean inlier residual residual / inlier (inlier = 0 ranks last),
 *      then the lowest h.  A frame without depth leaves every inlier count at 0 and keeps hypothesis 0 as long as hypothesis 0's
 *      model covers a pixel of its window (model > 0); when it covers none, the first h >= 1 whose model does wins.
 * Rows are track-major: track i's hypothesis h is row i S + h of every n x S array.  Draws: Philox4x32-10 (the generator of
 * se3tn_augment), key = seed, counter = (draw_keys[i] low word, high word, h, slot).  Each of the translation and the rotation
 * takes a direction from random_direction (theta = 2 pi U, phi = acos(2 U - 1)) and a magnitude from N(0, max), redrawn until
 * |m| <= max as the reference does, at most 64 times; a magnitude that never lands inside (probability ~1e-32) is clamped to +-max.
 * The rotation is cv2.Rodrigues of axis / |axis| * m / 180 * pi in fp64.  The draws depend on (seed, draw key, h) alone: not on
 * n, the precision, the route or anything else in the step.  S = 1 draws nothing and is the plain render step bit for bit.
 * Whether more hypotheses track better on a trained checkpoint has not been measured (README). */
#define SE3TN_MAX_HYPOTHESES 32
#define SE3TN_HYP_DRAWS 8     /* se3tn_draw_hypotheses' out_draws columns (below) */
typedef struct se3tn_hypothesis_opts {
    int32_t hypotheses, reserved;                  /* S in [1, SE3TN_MAX_HYPOTHESES]; reserved 0                            */
    int64_t seed;                                  /* the Philox key                                                         */
    double max_translation, max_rotation_deg;      /* metres, finite, in (0, 1]; degrees, in (0, 180]                        */
} se3tn_hypothesis_opts;                           /* 32 bytes, no padding                                                   */

/* ---- a tracking call's options and optional per-step arrays --------------------------------------------------------- */

/* Options of one tracking call (se3tn_track_batch, _render, _host, _render_host), passed by pointer; NULL means the defaults: no
 * fill, one round, no fit check, no ICP, no hypotheses.  Every field, and every field of what icp and hyp point to, is part of
 * what makes two steps the same (se3tn_last_step_was_graph).  The call reads nothing of it after it returns, and the context
 * keeps no option from one call to the next.  Refused with SE3TN_ERR_INVALID, the field named and nothing queued: a value
 * outside the ranges below, reserved != 0, icp and hyp together (ICP inside a hypothesis step is not supported), and, in
 * se3tn_track_batch / se3tn_track_host, iterations != 1, fit_tau_mm != 0, icp or hyp (they take input A from the caller: a later
 * round, ICP or a hypothesis cannot redraw it, and a weight id need not have a mesh for the fit check or ICP to draw).
 *
 * fill_depth != 0: fill the observed depth inside the step: fill_depth(frame_depth) exactly as se3tn_fill_depth_ex computes it
 * with fill_max_depth, fill_extrapolate (0 or not) and fill_blur (SE3TN_BLUR_*), with the same kernels, into context-owned
 * scratch, then K0 reads the filled frame.  A live sensor's raw depth image goes straight into the step, as the reference's ROS
 * node does with fill_depth before on_track (predict_ros.py:38-41: max_depth 2.0, extrapolate 0, bilateral).  fill_depth = 0:
 * the plain behaviour; the other fill fields are then ignored.  The caller's frame_depth is never written.  The fill adds its
 * launches to the step (8 bilateral, 6 gaussian, 3 more with extrapolate; see se3tn_last_launch_count), and no profiling slot
 * times it.  The host calls upload the whole depth frame instead of the crop-window rectangle, since the fill reads every pixel.
 * The scratch holds 2 x H x W floats plus the filled H x W uint16 frame and grows with the frame; growing it, here or in
 * se3tn_fill_depth[_ex], drops the context's captured steps.  fill_max_depth must be finite and > 0 as a float.
 *
 * iterations = k in [1, SE3TN_MAX_REFINE_ITERATIONS]: refine every track k times on this frame (se3tn_track_render[_host]): the
 * step is then exactly k successive single-round steps on the same frame (Tracker.on_track called k times, each from the pose
 * the previous call returned), in one call and one CUDA graph.  One step is the optional depth fill (once per step, not per
 * round), then k rounds of render (2 launches) -> K0 -> the 14 conv launches -> head / K6, each round drawing input A and
 * cropping B at the pose the round before wrote.  Round 0 reads poses_in; every later round reads and writes poses_out in place,
 * so poses_out == poses_in keeps working and the step's graph is replayed frame after frame.  out_trans / out_rot hold the last
 * round's network outputs; se3tn_last_launch_count counts fill + k x the launches of one round; profiling slots time the last
 * round.  SE3TN_PREC_FP32 runs the rounds as plain launches.  k = 1 is the single-round step.  se3tn_track_render_host uploads
 * the whole frame when k > 1 instead of the crop-window rectangle of the previous poses, since later rounds crop where the step
 * moved the tracks.  Whether more rounds improve accuracy depends on the checkpoint; it has not been measured on trained
 * weights.  se3tn_track_render's round_poses returns every round's poses from one step, and `predict --mode ycbv_recover`
 * scores them against the annotations of the YCB-Video key frames (README).
 *
 * fit_tau_mm = tau in [1, 1000]: check how well every track fits its frame (se3tn_track_render[_host]); 0 turns the check off.
 * After the last round (and ICP) the step draws each track's model at poses_out (the same mesh, mode, camera size and object
 * width as the rounds, depth only, into scratch of its own: the step's input A keeps the last round's) and compares the rendered
 * depth R with the observed depth O in the crop window of poses_out, cropped exactly as K0 crops input B (se3tn_compute_bbox's
 * window, se3tn_crop_bbox's nearest mapping, 0 outside the image; the filled frame when the step fills the depth).  R and O are
 * uint16 mm before any clipping.  Track i's row, SE3TN_FIT_COLS int32 over its 176 x 176 pixels:
 *   0 model     #(R > 0)
 *   1 observed  #(R > 0, O > 0)
 *   2 inlier    #(R > 0, O > 0, |O - R| <= tau_mm)
 *   3 front     #(R > 0, O > 0, O < R - tau_mm)   something in front of the model: occlusion
 *   4 behind    #(R > 0, O > 0, O > R + tau_mm)   the object is not where the model is
 *   5 residual  sum of |O - R| over the inliers, mm
 * observed = inlier + front + behind.  The rows are exact integers, independent of the order of the reduction.  The fit adds
 * 3 launches (render 2, fit 1; se3tn_last_launch_count) and no profiling slot; it is captured in the step's CUDA graph
 * (SE3TN_PREC_FP32 queues it as plain launches).  The step's poses, out_trans, out_rot and round_poses are bit for bit those of
 * the step without it.  se3tn_track_render: the rows land in a context-owned device buffer (max_batch x SE3TN_FIT_COLS int32,
 * allocated by the first step with the check on, never moved), whose address se3tn_fit_rows gives; the next step overwrites
 * them.  se3tn_track_render_host uploads the whole depth frame while the check is on (the window of poses_out is not known
 * before the step; rgb stays windowed) and brings the n rows back in its one copy out, into its out_fit.  How well the rows
 * predict tracking failure has not been measured on a trained checkpoint or real data (`predict --fit --score` reports it per
 * run, README).
 *
 * icp: NULL (ICP off: the step, its graph and its bits are those of a step that never mentions ICP), or the ICP options above
 * (HOST, read during the call only).  The block is allocated by the call, before anything is queued; scratch that cannot be
 * allocated is SE3TN_ERR_INVALID.  The host route uploads the whole depth frame while ICP is on.
 *
 * hyp: NULL (no expansion and no choice), or the hypothesis options above (HOST, read during the call only); hyp->hypotheses = 1
 * is the S = 1 hypothesis step, which draws nothing.  A hypothesis step needs fit_tau_mm (the choice ranks the fit rows) and
 * n x S <= max_batch.  It is the expansion, then the n x S-track render step's launches (its first render waits for the
 * expansion to complete), then the choice: se3tn_last_launch_count is that step's + 2.  The n x S starts, ids, widths and network
 * outputs live in context scratch (max_batch rows, allocated by the first call, never moved).  poses_out[i], out_trans[i] and
 * out_rot[i] are hypothesis out_choice[i]'s; poses_in is read only by the expansion, the step's first launch, so poses_out may be
 * poses_in.  The n x S step picks its split-K regime by n x S (n <= 4 is the latency mode), so hypothesis 0 matches a plain
 * n-track step bit for bit only when both land in the same regime.  The host route uploads the whole frame when S > 1 (the
 * starts' crop windows are drawn on the device). */
#define SE3TN_MAX_REFINE_ITERATIONS 8
#define SE3TN_FIT_COLS 6
struct se3tn_track_opts {
    int32_t fill_depth, fill_extrapolate, fill_blur, iterations;   /* fill_blur: SE3TN_BLUR_*; iterations 1..SE3TN_MAX_REFINE_ITERATIONS */
    double fill_max_depth;                                          /* metres; finite and > 0 as a float when fill_depth */
    int32_t fit_tau_mm, reserved;                                   /* fit_tau_mm 0: off, else 1..1000; reserved 0 */
    const se3tn_icp_opts* icp;                                      /* NULL: no ICP */
    const se3tn_hypothesis_opts* hyp;                               /* NULL: no expansion or choice */
};                                                                  /* 48 bytes on LP64, no padding */

/* The optional per-step arrays of se3tn_track_render (device pointers) and se3tn_track_render_host (host pointers), passed by
 * pointer; NULL means every field is NULL.  Each field is taken only where the step's options use it; one given where they do
 * not, or missing where they require it, is SE3TN_ERR_INVALID with the field named and nothing queued.  n tracks, k =
 * opts->iterations, M = opts->icp->iterations, S = opts->hyp->hypotheses:
 *   draw_keys    int64 (n), with hyp only; required when S > 1.  Each track's draw key.  On the device route it is read on the
 *                device, so one captured step replays frame after frame with fresh draws when the caller writes new keys into the
 *                same array; the host route sends it up with the poses.
 *   round_poses  double (k, n, 16), device route only: slot r - 1 receives every track's pose after round r, r = 1 .. k, bit for
 *                bit what an r-round step leaves in poses_out (slot k - 1 equals poses_out).  After each round the step copies
 *                poses_out there (a device-to-device copy inside the step's CUDA graph; SE3TN_PREC_FP32 queues it between its
 *                plain launches); se3tn_last_launch_count counts kernels only, so it reads as without it.  With hyp it is
 *                (k, n, S, 16): every round of every hypothesis.  ICP's iterations are not recorded here.
 *   hyp_poses    double (n, S, 16), with hyp on the device route only: every hypothesis after the last round.
 *   icp_poses    double (M, n, 16), with icp on the device route only: slot m - 1 receives every pose after ICP iteration m.
 *   out_fit      int32 (n, SE3TN_FIT_COLS).  Device route: with hyp only, and then required: the kept hypotheses' rows
 *                (se3tn_fit_rows then holds all n x S rows of the step; without hyp the rows stay there alone).  Host route:
 *                required exactly when opts->fit_tau_mm is set, brought back in the call's one copy out.
 *   out_choice   int32 (n), with hyp only, and then required: the hypothesis each track kept.
 *   out_icp      double (n, SE3TN_ICP_COLS), with icp only: the stats of the last ICP iteration.
 * Every pointer is part of the step's key: a step with round_poses and one without are two graphs, and both compute the same
 * poses_out.  Device route: SE3TN_ERR_INVALID, with nothing queued, for round_poses overlapping poses_in or poses_out; icp_poses
 * and out_icp overlapping poses_in, poses_out, round_poses or each other; with hyp, any output overlapping poses_in (except
 * poses_out == poses_in), draw_keys or another output. */
typedef struct se3tn_track_arrays {
    const int64_t* draw_keys;
    double* round_poses;
    double* hyp_poses;
    double* icp_poses;
    int32_t* out_fit;
    int32_t* out_choice;
    double* out_icp;
} se3tn_track_arrays;

/* *rows = the device rows of the fit check (max_batch x SE3TN_FIT_COLS int32).  SE3TN_ERR_STATE before the first step with the
 * check on. */
int se3tn_fit_rows(se3tn_ctx* ctx, const int32_t** rows);

/* The reference's own calling pattern as ONE call (Tracker.on_track, predict.py:217-296: numpy arrays in, numpy pose out):
 * every pointer is HOST memory.  The frame's crop-window rectangle, the poses, widths, input A and the ids are staged
 * through context-owned pinned memory into context-owned device buffers (stable addresses, so the step's CUDA graph is
 * replayed), se3tn_track_batch runs on them, and the call returns once poses_out (n x 16 doubles; out_trans / out_rot n x 3
 * floats, nullable) hold the result -- it synchronises `stream`.  frame_rgb uint8 (H,W,3), frame_depth uint16 (H,W) mm,
 * K = fx fy cx cy, poses double (n,16), object_width double (n) mm, rgbA uint8 (n,176,176,3), depthA uint16 (n,176,176),
 * weight_ids int32 (n) or NULL (all tracks use set 0).  Errors as se3tn_track_batch. */
int se3tn_track_host(se3tn_ctx* ctx, const uint8_t* frame_rgb, const uint16_t* frame_depth, int H, int W, const double* K,
                     const double* poses, const double* object_width, const uint8_t* rgbA, const uint16_t* depthA,
                     const int32_t* weight_ids, int n, double trans_normalizer, double rot_normalizer, int precision,
                     double* poses_out, float* out_trans, float* out_rot, const se3tn_track_opts* opts, void* stream);

/* ---- tracking from the previous poses and the frame alone: input A rendered inside the step ------------------------- */

/* Tracker.on_track for n tracks of one frame as the reference runs it (predict.py:217-296 with render_window at :246): the
 * models are rendered at poses_in, then K0 -> conv stack -> K6, all on `stream`.  Arguments as se3tn_track_batch without
 * rgbA / depthA; render_mode, render_H, render_W as mode, H, W of se3tn_render_ex (ignored in SE3TN_RENDER_VISPY).  Track i
 * draws mesh weight_ids[i] (mesh 0 when the ids are NULL): one network and one CAD model per object, both under one id.
 * Input A lands in context-owned device scratch (max_batch x 176 x 176 x 5 bytes, allocated by the first call).  One step
 * is render (2 launches) + the launches of se3tn_track_batch, captured as one CUDA graph (se3tn_last_step_was_graph);
 * SE3TN_PREC_FP32 renders and then runs its FFMA forwards without a graph.  Every id is checked on the host before anything is launched: an id without weights, statistics or a
 * mesh is SE3TN_ERR_STATE (the id is named; no other model is drawn in its place), n > max_batch, an unknown mode or a
 * camera image size out of range is SE3TN_ERR_INVALID.  poses_out may be poses_in, as in se3tn_track_batch.  opts selects the
 * step's extras (k rounds, the fit check, ICP, hypotheses: se3tn_track_opts); arrays, in HOST memory, holds their optional
 * device outputs (se3tn_track_arrays), or NULL; an arrays pointer into device memory is SE3TN_ERR_INVALID. */
int se3tn_track_render(se3tn_ctx* ctx, const uint8_t* frame_rgb, const uint16_t* frame_depth, int H, int W,
                       const double* K, const double* poses_in, const double* object_width,
                       int render_mode, int render_H, int render_W,
                       const int32_t* weight_ids_host, const int32_t* weight_ids_dev, int n,
                       double trans_normalizer, double rot_normalizer, int precision,
                       float* out_trans, float* out_rot, double* poses_out, const se3tn_track_opts* opts,
                       const se3tn_track_arrays* arrays, void* stream);

/* se3tn_track_render with every pointer in HOST memory, the reference's own calling pattern with rendering included: the
 * frame's crop-window rectangle, the poses, widths and ids go through se3tn_track_host's pinned staging (one copy in, one
 * copy out, stable device addresses so the step's graph is replayed); input A is rendered on the device and never crosses
 * the bus.  Synchronises `stream`.  Arguments as se3tn_track_host without rgbA / depthA, plus the render arguments of
 * se3tn_track_render; weight_ids int32 (n) or NULL (all tracks use set 0 and mesh 0).  arrays: the optional HOST arrays of
 * se3tn_track_arrays this route takes (draw_keys, out_fit, out_choice, out_icp), or NULL.  Errors as se3tn_track_render. */
int se3tn_track_render_host(se3tn_ctx* ctx, const uint8_t* frame_rgb, const uint16_t* frame_depth, int H, int W, const double* K,
                            const double* poses, const double* object_width, int render_mode, int render_H, int render_W,
                            const int32_t* weight_ids, int n, double trans_normalizer, double rot_normalizer, int precision,
                            double* poses_out, float* out_trans, float* out_rot, const se3tn_track_opts* opts,
                            const se3tn_track_arrays* arrays, void* stream);

/* The expansion alone, as a hypothesis step's first launch forms it: poses_in double (n,16), draw_keys int64 (n) (NULL when
 * S = 1) -> out_poses double (n, S, 16), all device.  out_draws double (n, S, SE3TN_HYP_DRAWS) device or NULL: per row the
 * translation direction's U_theta, U_phi, the rotation axis' U_theta, U_phi, the accepted magnitudes m_T (m) and m_R (degrees),
 * and the N(0, max) draws each took (1..64); all 0 in hypothesis 0's rows.  One plain launch.  Refused (SE3TN_ERR_INVALID,
 * nothing queued): hyp out of range, n x S > max_batch, draw_keys NULL with S > 1, an output overlapping an input or the other. */
int se3tn_draw_hypotheses(se3tn_ctx* ctx, const double* poses_in, const int64_t* draw_keys, int n, const se3tn_hypothesis_opts* hyp,
                          double* out_poses, double* out_draws, void* stream);

/* ---- start poses from a mask and the depth frame: render-and-compare over a rotation grid ---------------------------- */

/* Every tracking call refines a pose it is given.  se3tn_init_poses finds a first one, for n objects of one frame, from each
 * object's segmentation label and the depth frame alone (no network weights).  The stages, on `stream`, in this order:
 *   1. Mask statistics, per object i with label l_i, over the whole H x W frame: mask = #(seg == l_i), depth_px = #(seg == l_i,
 *      depth > 0), sum_u / sum_v = the sums of the mask pixels' columns / rows, z_med = the lower median (sorted index
 *      (depth_px - 1) / 2) of the mask's depths > 0, in mm.  Integer atomics and a 65536-bin histogram: exact and independent
 *      of the order of the reduction.  t0 = z_med / 1000 * K^-1 (sum_u / mask, sum_v / mask, 1) in fp64, metres.  status 1: the
 *      mask is empty; 2: depth_px < min_pixels.  (A status != 0 object is drawn at the placeholder t0 = (0, 0, 1).)
 *   2. Rotation grid: candidate c = v R + r, V viewpoints x R in-plane angles.  d_v is the Fibonacci-sphere direction
 *      z = 1 - (2 v + 1) / V, phi = v pi (3 - sqrt 5) in the object frame; R_c maps d_v to the camera's -z axis with the
 *      object's +z as the up vector (+y when |d_v.z| > 0.99) and then turns about the camera's z axis by 2 pi r / R.  fp64;
 *      every candidate sits at t0 (oracle/init_ref.py restates the formulas).
 *   3. Render and score: the n V R candidates are drawn (depth only, render_mode as se3tn_render_ex, mesh weight_ids[i])
 *      in chunks of max_batch rows, each chunk followed by a score launch: one 4-CTA cluster per row crops the observed depth O
 *      and the mask M = (seg == l_i) at the row's own window (se3tn_compute_bbox's window, se3tn_crop_bbox's nearest mapping,
 *      0 outside the frame) and counts, over the rendered depth R: model #(R>0), maskc #M, overlap #(R>0, M), pairs
 *      #(R>0, M, O>0) with S = sum (O - R) over them; then delta = floor((2 S + pairs) / (2 pairs)) mm (0 without pairs) and
 *      inlier #(R>0, M, O>0, |O - (R + delta)| <= tau_mm).
 *      Rank: the higher inlier / union (union = model + maskc - overlap; union 0 scores 0) as int64 cross products, then the
 *      higher overlap, then the lower candidate index.
 *   4. Keep K: per object, the K best candidates in rank order (exact: the rows are integers).  A kept pose moves along its
 *      ray by its row's delta: t = t0 (1 + delta / (1000 t0_z)).
 *   5. Refine (icp != NULL): icp->iterations ICP iterations (se3tn_icp_opts, the tracking step's render with triangle ids and
 *      accumulate / solve launches) on the n K kept poses as n K tracks, then each refined pose is rendered and scored as in
 *      3 at its own window with delta fixed at 0, and the best of the K by the same rank is kept.  Without icp the result is
 *      the top grid candidate.
 *   6. poses_out double (n, 16) device: one pose per object, all NaN when its status is not 0.  out_rows int32 (n,
 *      SE3TN_INIT_COLS) device: the kept candidate's score row
 *        0 status  1 candidate (v R + r)  2 model  3 maskc  4 overlap  5 pairs  6 inlier  7 delta_mm (0 after ICP)
 * Arguments: frame_depth uint16 (H, W) mm and seg uint8 (H, W), device, H W < 2^31; K HOST fx fy cx cy; labels HOST int32 (n), 1..255
 * (objects may share a label); object_width double (n) mm, device; render_mode / render_H / render_W as se3tn_track_render;
 * weight_ids_host / weight_ids_dev int32 (n), both or neither (mesh 0).  No CUDA graph: plain launches, no synchronisation,
 * except that a call needing more scratch than the context's init block holds first synchronises `stream` and grows it (the
 * block holds the histogram, 256 KB per object, the n V R grid poses, widths, ids and rows, and one chunk's rendered depth,
 * max_batch x 176 x 176 x 2 bytes).  The ICP stage uses the tracking step's ICP block (allocated by the call when no step
 * has), whose contents no step reads before writing, so tracking steps and their graphs are unaffected.
 * se3tn_last_launch_count: 2 (mask) + 1 (grid) + 3 per chunk + 1 (keep) [+ 4 M + 3 with icp] + 1 (choose).
 * Refused with SE3TN_ERR_INVALID, the field named and nothing queued: a NULL input or output, a value outside the ranges
 * below, reserved != 0, keep > V R, n K > max_batch, a label outside 1..255, an ICP option out of range, and an output
 * overlapping an input or another output.  An id without a mesh is SE3TN_ERR_STATE.  n = 0 queues nothing.
 * The defaults of Engine.init_spec (V 300, R 24, K 8, tau 20 mm, min_pixels 100, 5 ICP iterations) are starting guesses: how
 * well they do on real sensor data has not been measured (README). */
#define SE3TN_INIT_COLS 8
#define SE3TN_INIT_STATS 6
#define SE3TN_MAX_INIT_KEEP 32
typedef struct se3tn_init_opts {
    int32_t viewpoints, inplane;                   /* V in [1, 4096], R in [1, 360], V R <= 65536                            */
    int32_t keep, tau_mm;                          /* K in [1, SE3TN_MAX_INIT_KEEP], K <= V R, n K <= max_batch; [1, 1000]    */
    int32_t min_pixels, reserved;                  /* [1, 176 * 176]; 0                                                      */
    const se3tn_icp_opts* icp;                     /* NULL: the best grid candidate; else refine the K kept, rescore, keep the best */
} se3tn_init_opts;                                 /* 32 bytes on LP64, no padding                                           */

/* The optional device outputs of se3tn_init_poses, passed by pointer (HOST memory); NULL means every field is NULL.
 *   stats       int64 (n, SE3TN_INIT_STATS): status, mask, depth_px, sum_u, sum_v, z_med
 *   t0          double (n, 3): the start translation, metres
 *   cand_rows   int32 (n, V R, SE3TN_INIT_COLS): every candidate's score row, candidate c of object i at row i V R + c
 *   kept_rows   int32 (n, K, SE3TN_INIT_COLS): the K kept candidates' rows in rank order
 *   kept_poses  double (n, K, 16): their grid poses, moved along the ray by delta
 *   icp_poses   double (n, K, 16), with icp only: the kept poses after the ICP iterations
 *   icp_rows    int32 (n, K, SE3TN_INIT_COLS), with icp only: their rows, scored at delta 0
 *   icp_stats   double (n, K, SE3TN_ICP_COLS), with icp only: the last ICP iteration's stats of each kept pose */
typedef struct se3tn_init_arrays {
    int64_t* stats;
    double* t0;
    int32_t* cand_rows;
    int32_t* kept_rows;
    double* kept_poses;
    double* icp_poses;
    int32_t* icp_rows;
    double* icp_stats;
} se3tn_init_arrays;

int se3tn_init_poses(se3tn_ctx* ctx, const uint16_t* frame_depth, const uint8_t* seg, int H, int W, const double* K,
                     const int32_t* labels, const double* object_width, int render_mode, int render_H, int render_W,
                     const int32_t* weight_ids_host, const int32_t* weight_ids_dev, int n, const se3tn_init_opts* opts,
                     double* poses_out, int32_t* out_rows, const se3tn_init_arrays* arrays, void* stream);

/* ---- start poses from a 2D box and the depth frame ------------------------------------------------------------------ */

/* se3tn_init_boxes starts n objects of one frame from 2D boxes, as a detector gives them, instead of labels.  A box is
 * int32 (x0, y0, x1, y1) in frame pixels, half-open: the pixels with x0 <= u < x1 and y0 <= v < y1.  Boxes may overlap;
 * each object owns its box's pixels whatever the other boxes hold.  The stages are those of se3tn_init_poses with:
 *   1. Box statistics: the object's pixels are its box's pixels instead of seg == l_i.  stats keep their columns over them
 *      (mask = the box's pixel count, sum_u / mask = (x0 + x1 - 1) / 2 exactly; z_med the lower median; status 1 / 2 as
 *      before, an empty box (x1 == x0 or y1 == y0) gives status 1).  From the same histogram, D = `depths` depth candidates:
 *      z_d = the sorted depth at index k_d = max(0, floor(((2 d + 1) depth_px - D) / (2 D))), d = 0 .. D-1, the quantiles
 *      (2 d + 1) / 2 D of the box's depths (D = 1: the lower median), and t0_d = z_d / 1000 * K^-1 (u, v, 1) in fp64 on the
 *      ray through the box centre.  A box holds background as well as the object, so one median may lie behind it: the D
 *      depths let the score pick the one at which the silhouette fits.
 *   2. Grid: candidate c = d V R + v R + r is the mask grid's rotation (v, r) at t0_d.  All D V R candidates of an object
 *      compete in one ranking.
 *   3. Score: the mask score, with M = "the crop pixel's source frame pixel lies in the object's box".  Counts, delta,
 *      inlier and rank unchanged.
 *   4-6. Keep, refine and choose unchanged (a kept pose moves along its own ray by delta).
 * So for D = 1 and boxes that do not overlap, the call equals se3tn_init_poses on a label image in which each object's box
 * pixels carry its own label, on every output, bit for bit.
 * Arguments as se3tn_init_poses, with boxes HOST int32 (n, 4) in place of seg and labels (staged into the context's init
 * block) and depths D in [1, 8].  Shapes that differ: arrays->t0 double (n, D, 3); arrays->cand_rows int32 (n, D V R,
 * SE3TN_INIT_COLS), column 1 of a row is c above; keep <= D V R.  Refused with SE3TN_ERR_INVALID, the field named and nothing
 * queued, as se3tn_init_poses, and: depths outside [1, 8]; a box with x0 < 0, y0 < 0, x1 > W, y1 > H, x1 < x0 or y1 < y0.  An
 * id without a mesh is SE3TN_ERR_STATE.  Plain launches, no CUDA graph; the init block grows as se3tn_init_poses' (a call
 * that needs more first synchronises `stream`), and tracking steps and their graphs are unaffected.
 * se3tn_last_launch_count: 2 (box pass, depths) + 1 (grid) + 3 per chunk of the n D V R rows + 1 (keep) [+ 4 M + 3 with
 * icp] + 1 (choose).  The Python default D = 4 (Engine.init_boxes) is a starting guess, like the other init defaults. */
int se3tn_init_boxes(se3tn_ctx* ctx, const uint16_t* frame_depth, int H, int W, const double* K,
                     const int32_t* boxes, int depths, const double* object_width, int render_mode, int render_H, int render_W,
                     const int32_t* weight_ids_host, const int32_t* weight_ids_dev, int n, const se3tn_init_opts* opts,
                     double* poses_out, int32_t* out_rows, const se3tn_init_arrays* arrays, void* stream);

/* ---- re-initialisation: a start from the mask replaces a track the fit check finds lost ------------------------------ */

/* Three calls connect the fit check (se3tn_track_opts.fit_tau_mm) to se3tn_init_poses.  Engine.reinit runs them after a
 * tracking step; oracle/reinit_ref.py restates the rules in numpy.
 *   Lost.     Track i is below in a step when 1000 inlier < below_permille model, compared as int64; a track with model = 0 is
 *             below.  Each track has an int32 streak that persists across calls (the caller keeps it, zeroed at the start):
 *             streak + 1 when below, 0 otherwise.  A track is lost when its streak reaches `after`.
 *   Restart.  The lost tracks of a frame, in ascending track order, go through one se3tn_init_poses call, each with its own
 *             label, mesh and width, on the depth the step saw (the filled frame when the step fills).
 *   Accept.   A start replaces the tracked pose only when its init status is 0 and its fit row (se3tn_fit_poses: the step's
 *             fit check at the start) ranks strictly above the tracked pose's row, in the hypothesis choice's order: the
 *             higher inlier / model, then the lower residual / inlier, as int64 cross products (model = 0 or inlier = 0
 *             ranks last; a tie is not above).  The pose and the fit row are then both the start's.
 *   After an attempt the streak is 0 whatever the outcome, so a track is retried at most once every `after` frames.
 * Event codes per track and step (int32): 0 not below; 1 below, no attempt (the streak is short of `after`, or the track is
 * lost but no mask was given); 2 restarted, the pose is the start; 3 no start (init status != 0); 4 start rejected (it fits no
 * better than the tracked pose).
 * The defaults of Engine.reinit_spec / Tracker(reinit=) (below 0.5, after 3) are guesses, not tuned: `predict --fit --score`
 * reports how well the inlier fraction separates lost from kept tracks on a data set, which is what to choose them by. */
#define SE3TN_REINIT_NONE 0
#define SE3TN_REINIT_BELOW 1
#define SE3TN_REINIT_RESTARTED 2
#define SE3TN_REINIT_NO_START 3
#define SE3TN_REINIT_REJECTED 4
typedef struct se3tn_reinit_opts {
    int32_t below_permille, after;                 /* [1, 1000], [1, 1000]                                                   */
    int32_t reserved[2];                           /* 0                                                                      */
} se3tn_reinit_opts;                               /* 16 bytes, no padding                                                   */

/* The loss rule over one step's fit rows, one launch of one CTA: fit_rows int32 (n, SE3TN_FIT_COLS), streak int32 (n) in /
 * out, out_event int32 (n) (0 or 1 for every track), out_lost int32 (n + 1): the count of lost tracks, then their indices in
 * ascending order (a block scan: the order never depends on scheduling); entries past the count are not written.  All device.
 * Refused with SE3TN_ERR_INVALID, the field named and nothing queued: NULL arguments, n outside [0, max_batch], an option out
 * of range, reserved != 0, and an output overlapping fit_rows or another output.  se3tn_last_launch_count: 1. */
int se3tn_lost_tracks(se3tn_ctx* ctx, const int32_t* fit_rows, int n, const se3tn_reinit_opts* opts, int32_t* streak,
                      int32_t* out_event, int32_t* out_lost, void* stream);

/* The fit check of a tracking step (se3tn_track_opts.fit_tau_mm) at n given poses: each model is drawn (depth only, mesh
 * weight_ids[i], render_mode / render_H / render_W as se3tn_track_render) and compared with frame_depth in the crop window of
 * its pose.  Its rows equal, as exact integers, those a tracking step's fit check gives at the same poses on the same frame
 * with the same tau, mode, meshes and widths.  A pose with a non-finite entry draws nothing: its row is all 0.
 *   frame_depth uint16 (H, W) mm, poses double (n, 16), object_width double (n) mm, out_rows int32 (n, SE3TN_FIT_COLS): device;
 *   K HOST fx fy cx cy; weight_ids_host / weight_ids_dev int32 (n), both or neither (mesh 0); fit_tau_mm in [1, 1000].
 * Plain launches, no CUDA graph.  The rendered depth goes to scratch of the call's own (n x 176 x 176 x 2 bytes), which no
 * tracking step reads or writes: a call needing more than it holds synchronises `stream` and grows it.  The fit check's
 * rows (se3tn_fit_rows) and the step's input A are untouched.  se3tn_last_launch_count: 3 (render 2, fit 1).  Refused with
 * SE3TN_ERR_INVALID, nothing queued: NULL arguments, n outside [0, max_batch], tau out of range, a bad render mode, out_rows
 * overlapping an input; an id without a mesh is SE3TN_ERR_STATE. */
int se3tn_fit_poses(se3tn_ctx* ctx, const uint16_t* frame_depth, int H, int W, const double* K, const double* poses,
                    const double* object_width, int render_mode, int render_H, int render_W, const int32_t* weight_ids_host,
                    const int32_t* weight_ids_dev, int n, int fit_tau_mm, int32_t* out_rows, void* stream);

/* The accept rule for the starts of m lost tracks, one launch: start k belongs to track lost_idx[k] and comes with its init
 * row (init_rows int32 (m, SE3TN_INIT_COLS), se3tn_init_poses' out_rows) and its fit row (start_fit int32 (m, SE3TN_FIT_COLS),
 * se3tn_fit_poses at starts double (m, 16)).  In place over the n tracks: poses double (n, 16) and fit_rows int32 (n,
 * SE3TN_FIT_COLS) take the start's pose and row on a restart; streak int32 (n) is 0 for each of the m tracks; out_event int32
 * (n) is 2, 3 or 4 for each of them.  Tracks not in the list are not touched.  All device except lost_idx_host, a host copy
 * of lost_idx_dev that the checks read (as se3tn_lost_tracks' out_lost gives it after a copy back).  Refused with
 * SE3TN_ERR_INVALID, nothing queued: NULL arguments, n outside [0, max_batch], m outside [0, n], a lost index outside [0, n)
 * or repeated, and an in-place output overlapping an input or another output.  se3tn_last_launch_count: 1 (0 when m = 0). */
int se3tn_accept_starts(se3tn_ctx* ctx, const int32_t* lost_idx_host, const int32_t* lost_idx_dev, int m, const double* starts,
                        const int32_t* init_rows, const int32_t* start_fit, int n, double* poses, int32_t* fit_rows, int32_t* streak,
                        int32_t* out_event, void* stream);

/* ---- checkpoint validation: the loss of ready-made training pairs ---------------------------------------------------- */

/* Problem.validate's per-batch work (reference problems.py:106-132) as ONE step: for n pairs as TrackDataset.__getitem__ reads
 * them (datasets.py:70-112, crops already at 176 x 176), processData's post-transforms (datasets.py:136-137, se3tn_normalize),
 * Se3TrackNet.forward in eval mode and Se3TrackNet.loss (se3_tracknet.py:114-121) on the labels of datasets.py:141-150.
 *   rgbA, rgbB uint8 (n,176,176,3), depthA, depthB uint16 (n,176,176) mm, A_in_cam, B_in_cam double (n,16) row-major, device
 *   weight_ids_host / weight_ids_dev as in se3tn_track_batch (both NULL: every pair uses set 0)
 *   out_trans, out_rot float (n,3) device: the network's outputs
 *   out_sq float (n,6) device or NULL: per pair (pred - float(label))^2 in fp32, translation then rotation, as nn.MSELoss forms them
 *   out_labels double (n,6) device or NULL: trans_label then rot_label, bit-identical to se3tn_so3_log
 *   out_sums float (2) device: the sums of the n x 3 translation terms and of the n x 3 rotation terms, added in a fixed order that
 *     depends on n alone (thread t of one CTA adds pairs t, t+256, ... in order, then a tree); MSE = sum / (3 n).
 * In the tensor-core modes the loss terms are formed in the head kernel (labels in fp64 by the same device function as
 * se3tn_so3_log) and one more launch adds them: normalize + 8 resident convs + trunk + head + reduction = 12 launches, captured as
 * one CUDA graph (se3tn_last_step_was_graph).
 * SE3TN_PREC_FP32 runs one FFMA forward per contiguous run of equal ids and then one stand-alone loss launch, without a graph:
 * 1 + 17 per run + 1 launches.  Every id is checked on the host before anything is queued: an id without weights or statistics
 * is SE3TN_ERR_STATE (the id is named); n == 0 or n > max_batch is SE3TN_ERR_INVALID.  Without out_sq the terms go to a
 * context-owned max_batch x 6 float buffer, allocated by the first such call. */
int se3tn_eval_pairs(se3tn_ctx* ctx, const uint8_t* rgbA, const uint16_t* depthA, const uint8_t* rgbB, const uint16_t* depthB,
                     const double* A_in_cam, const double* B_in_cam,
                     const int32_t* weight_ids_host, const int32_t* weight_ids_dev, int n,
                     double trans_normalizer, double rot_normalizer, int precision,
                     float* out_trans, float* out_rot, float* out_sq, double* out_labels, float* out_sums, void* stream);

/* Se3TrackNet.loss (reference se3_tracknet.py:114-121) on predictions that already exist: trans, rot float (n,3), trans_label,
 * rot_label double (n,3), all device -> out_sums float (2) device, with the same loss terms and the same order of additions as
 * se3tn_eval_pairs (one launch, any n > 0): the two callers agree bit for bit.  MSE = sum / (3 n). */
int se3tn_pair_loss(se3tn_ctx* ctx, const float* trans, const float* rot, const double* trans_label, const double* rot_label, int n,
                    float* out_sums, void* stream);

/* ---- validation under the reference's train-time augmentations (data_augmentation.py:48-121, 217-267) ----------------------- */

/* The augmentation chain of the reference's train.py:85-92, in that order, on input B of each pair: HSVJitter, ChangeBright,
 * GaussianNoise, GaussianBlur, BlackCover (any subset; each stage's flag is 0 or 1).  Every random value of pair i comes from
 * Philox4x32-10 keyed by (seed, pair_index[i], draw slot) with the reference's distribution, so a pair's augmentation depends on
 * (seed, pair index) alone; given the draws, the arithmetic is the reference classes' bit for bit (cv2 4.13 on x86-64 for the
 * colour conversions and the blur).  DepthMissing, commented out in train.py, is refused (SE3TN_ERR_UNSUPPORTED). */
typedef struct se3tn_augment {
    uint64_t seed;
    int32_t hsv_jitter, change_bright, gaussian_noise, gaussian_blur, black_cover, depth_missing;   /* stage flags */
    double hsv_prob, hsv_noise[3];          /* HSVJitter(h_noise, s_noise, v_noise, prob): each channel's test, then U(-noise, noise) */
    double bright_mag[2];                   /* ChangeBright(mag): always applied, U(mag[0], mag[1]) */
    double noise_prob, noise_rgb, noise_depth;   /* GaussianNoise(rgb_noise, depth_noise, prob): std ~ U(0, noise), N(0, std) */
    double blur_prob; int32_t blur_max_kernel, reserved;   /* GaussianBlur(max_kernel_size, prob): k = 2 randint(1, max//2 + 1) + 1 */
    double cover_prob;                      /* BlackCover(prob) */
} se3tn_augment;

/* The per-pair draws, as se3tn_augment_draws writes them: SE3TN_AUG_PARAMS doubles per pair.
 *   0 HSVJitter on, 1-3 its h / s / v branch outcomes (0 / 1), 4-6 their magnitudes, 7 ChangeBright on, 8 its factor,
 *   9 / 10 GaussianNoise rgb branch / std, 11 / 12 depth branch / std, 13 / 14 GaussianBlur rgb branch / k, 15 / 16 depth branch / k,
 *   17 BlackCover branch, 18 / 19 the accepted corner (u column, v row), 20 its quadrant (0 top left, 1 top right, 2 bottom left,
 *   3 bottom right; -1: no cover), 21 corners drawn, 22 num_valid = sum of maskB's values, 23 maskB == 1 pixels left.
 * A magnitude is drawn whether or not its branch is taken.  BlackCover draws at most SE3TN_AUG_MAX_CORNERS corners (the reference
 * loops without end when no quadrant can keep half of num_valid); a pair that reaches the cap is left uncovered, quadrant -1. */
#define SE3TN_AUG_PARAMS 24
#define SE3TN_AUG_MAX_CORNERS 64

/* se3tn_eval_pairs on augmented pairs: the first nine rows of arguments as se3tn_eval_pairs, then
 *   segB uint8 (n,176,176) device, or NULL: BlackCover's maskB, or depthB > 100 without it (datasets.py:103-104)
 *   pair_index int64 (n) device: each pair's index, the key of its draws (read on the device, so a graph replays across batches)
 *   aug HOST: the chain; its values and whether segB is NULL join the step's key
 *   out_rgbB uint8 (n,176,176,3), out_depthB uint16 (n,176,176) device, nullable: the augmented crops the step evaluated.
 * Two more launches than se3tn_eval_pairs (the draws, then every stage in one pass over bands of rows) write the augmented B into
 * out_rgbB / out_depthB or context-owned scratch (max_batch x 176 x 176 x 5 bytes, allocated by the first such call); the
 * normalize launch reads it instead of rgbB / depthB, which are only read.  One CUDA graph, as se3tn_eval_pairs.  Refused on the
 * host before anything is queued: everything se3tn_eval_pairs refuses, a NULL pair_index or aug, and a chain se3tn_augment_draws
 * refuses, and out_rgbB / out_depthB overlapping an input or each other (the blur reads neighbouring rows of input B, so the
 * augmentation cannot run in place). */
int se3tn_eval_pairs_augmented(se3tn_ctx* ctx, const uint8_t* rgbA, const uint16_t* depthA, const uint8_t* rgbB, const uint16_t* depthB,
                               const double* A_in_cam, const double* B_in_cam,
                               const int32_t* weight_ids_host, const int32_t* weight_ids_dev, int n,
                               double trans_normalizer, double rot_normalizer, int precision,
                               float* out_trans, float* out_rot, float* out_sq, double* out_labels, float* out_sums,
                               const uint8_t* segB, const int64_t* pair_index, const se3tn_augment* aug,
                               uint8_t* out_rgbB, uint16_t* out_depthB, void* stream);

/* Exactly the draws se3tn_eval_pairs_augmented uses for pairs pair_index[0..n) (int64, device): out_params double
 * (n, SE3TN_AUG_PARAMS) device; BlackCover's corner needs maskB: segB uint8 (n,176,176) or, NULL, depthB uint16 (n,176,176) > 100.
 * out_noise_rgb double (n,176,176,3) and out_noise_depth double (n,176,176) device, nullable: GaussianNoise's N(0, std) fields at
 * every element, whatever the branch and the mask.  Plain stream launches.  Refused on the host (SE3TN_ERR_INVALID unless noted):
 * a NULL aug, pair_index, depthB or out_params, n <= 0 or n > max_batch, a stage flag other than 0 / 1, no stage enabled,
 * depth_missing set (SE3TN_ERR_UNSUPPORTED), a probability outside [0, 1], blur_max_kernel / 2 outside {1, 2, 3} (k outside
 * {3, 5, 7}), a non-finite magnitude or a negative noise magnitude, and an output overlapping an input or another output. */
int se3tn_augment_draws(se3tn_ctx* ctx, const se3tn_augment* aug, const uint16_t* depthB, const uint8_t* segB, const int64_t* pair_index,
                        int n, double* out_params, double* out_noise_rgb, double* out_noise_depth, void* stream);

/* The augmented crops alone, as se3tn_eval_pairs_augmented forms them (its two augmentation launches): rgbB uint8 (n,176,176,3),
 * depthB uint16 (n,176,176), segB as there, pair_index int64 (n), all device -> out_rgbB, out_depthB device (TrackDataset's
 * augmented rgbB / depthB).  Plain stream launches; refusals as se3tn_augment_draws. */
int se3tn_augment_crops(se3tn_ctx* ctx, const se3tn_augment* aug, const uint8_t* rgbB, const uint16_t* depthB, const uint8_t* segB,
                        const int64_t* pair_index, int n, uint8_t* out_rgbB, uint16_t* out_depthB, void* stream);

/* ---- held-out pairs from annotated frames: ProducerPurturb.generate (reference produce_train_pair_data.py:86-141) ------------- */

/* crop_bbox with its segmentation plane (reference Utils.py:320-359 with seg): rgb and depth exactly as se3tn_crop_bbox cuts them, and
 * seg uint8 (H,W) device through the same window and nearest-neighbour mapping, zero outside the image, never masked (Utils.py:346-349).
 * class_ids NULL: crop_seg uint8 (n,out_h,out_w) receives the labels.  class_ids int32 (n) device: crop_seg receives (label == class id)
 * as 0 / 1 and seg_count int32 (n) device (nullable) the number of ones.  One launch. */
int se3tn_crop_bbox_seg(se3tn_ctx* ctx, const uint8_t* frame_rgb, const uint16_t* frame_depth, const uint8_t* seg, int H, int W,
                        const int32_t* bbox, const int32_t* class_ids, int n, int out_h, int out_w,
                        uint8_t* crop_rgb, uint16_t* crop_depth, uint8_t* crop_seg, int32_t* seg_count, void* stream);

/* The two counts of the generator's visibility check (produce_train_pair_data.py:97-104) for m rows (pose, mesh id, class id) of one
 * frame:  out_visible[i] = #(seg == class_ids[i]) over the whole H x W seg frame (uint8, device);  out_covered[i] = the pixels of mesh
 * i's render at poses[i] over the whole H x W camera image in the SE3TN_RENDER_PYRENDER mode whose float32 linearised depth is > 0.1f
 * (np.sum(depth > 0.1) of Renderer.render's depth).  K HOST fx fy cx cy; poses double (m,16), class_ids int32 (m), outputs int32 (m),
 * device; mesh_ids_host / mesh_ids_dev int32 (m) (both NULL: mesh 0).  Plain stream launches (memsets + 3 kernels), not captured.  The
 * nearest-z planes (m x H x W words) are context-owned scratch that only grows.  Ids are checked on the host before anything is
 * queued: a missing mesh is SE3TN_ERR_STATE, m > max_batch SE3TN_ERR_INVALID.  The host then applies the reference's thresholds. */
int se3tn_visibility(se3tn_ctx* ctx, const uint8_t* seg, int H, int W, const double* K, const double* poses,
                     const int32_t* mesh_ids_host, const int32_t* mesh_ids_dev, const int32_t* class_ids, int m,
                     int32_t* out_visible, int32_t* out_covered, void* stream);

/* One step of ProducerPurturb.generate for n perturbed samples of one frame (produce_train_pair_data.py:118-128): compute_bbox of each
 * A_in_cam (object_width[i] mm, scale 1000), render A of mesh i at A_in_cam in the SE3TN_RENDER_PYRENDER mode over the H x W camera
 * image and crop it (what se3tn_render_ex gives), then crop B, its depth and its seg out of the frame through the same window
 * (se3tn_crop_bbox_seg with the class ids).  frame_rgb uint8 (H,W,3), frame_depth uint16 (H,W), seg uint8 (H,W), A_in_cam double (n,16),
 * object_width double (n), class_ids int32 (n), device; K HOST.  Outputs, device: rgbA, rgbB uint8 (n,176,176,3), depthA, depthB
 * uint16 (n,176,176), segB uint8 (n,176,176) 0 / 1 as the generator writes it, seg_count int32 (n) = #(segB == 1).  bbox + render (2) +
 * crop = 4 launches, captured as one CUDA graph keyed like the track steps (se3tn_last_step_was_graph).  Errors as se3tn_track_render:
 * ids checked on the host before anything is queued, a missing mesh is SE3TN_ERR_STATE, n > max_batch SE3TN_ERR_INVALID. */
int se3tn_perturb_pairs(se3tn_ctx* ctx, const uint8_t* frame_rgb, const uint16_t* frame_depth, const uint8_t* seg, int H, int W,
                        const double* K, const double* A_in_cam, const double* object_width,
                        const int32_t* mesh_ids_host, const int32_t* mesh_ids_dev, const int32_t* class_ids, int n,
                        uint8_t* rgbA, uint16_t* depthA, uint8_t* rgbB, uint16_t* depthB, uint8_t* segB, int32_t* seg_count,
                        void* stream);

/* The generator's threshold on a sample's segB pixel count (produce_train_pair_data.py:128): a sample is kept when seg_count >= it. */
#define SE3TN_PAIR_MIN_SEG 100

/* The kept rows of a se3tn_perturb_pairs step appended to per-queue validation batches, with no host read in between.  Row i
 * (rgbA, rgbB uint8 (n,176,176,3), depthA, depthB uint16 (n,176,176), seg_count int32 (n), A_in_cam, B_in_cam double (n,16), all
 * device) is kept when seg_count[i] >= SE3TN_PAIR_MIN_SEG and goes to queue q = queue_ids[i], slot tails_dev[q] + (the kept rows of
 * queue q before it), so each queue receives its rows in row order.  The queues are num_queues x cap rows in the layout
 * se3tn_eval_pairs reads: q_rgbA, q_rgbB uint8 (num_queues,cap,176,176,3), q_depthA, q_depthB uint16 (num_queues,cap,176,176),
 * q_A_in_cam, q_B_in_cam double (num_queues,cap,16), device; queue q's slot s is row q * cap + s.  tails_dev int32 (num_queues)
 * device: each advanced by its queue's kept rows.  Rejected rows and every other slot are left as they were.
 * One launch (16-byte copies; the CTA that finishes last advances the tails through a context-owned counter).  Checked on the host
 * before anything is queued, all SE3TN_ERR_INVALID: a null pointer, a device pointer not 16-byte aligned, n > max_batch, a queue
 * id outside [0, num_queues) (queue_ids_host, with its device copy queue_ids_dev), and a queue whose capacity cannot hold all the
 * rows sent to it, kept or not: tails_host[q] + #(rows of q) > cap, where tails_host (HOST, num_queues) is what tails_dev holds when
 * the append runs, or a bound above it (the tails last read back plus every row sent since).  On the device a row whose slot would reach cap is not
 * written, but its tail still advances, so an overflow shows in the tails read back.  n == 0 queues nothing. */
int se3tn_append_pairs(se3tn_ctx* ctx, const uint8_t* rgbA, const uint16_t* depthA, const uint8_t* rgbB, const uint16_t* depthB,
                       const int32_t* seg_count, const double* A_in_cam, const double* B_in_cam,
                       const int32_t* queue_ids_host, const int32_t* queue_ids_dev, int n,
                       int num_queues, int cap, const int32_t* tails_host, int32_t* tails_dev,
                       uint8_t* q_rgbA, uint16_t* q_depthA, uint8_t* q_rgbB, uint16_t* q_depthB, double* q_A_in_cam, double* q_B_in_cam,
                       void* stream);

/* se3tn_append_pairs with a fifth plane: segB uint8 (n,176,176) device, as se3tn_perturb_pairs writes it, goes with its row to
 * q_segB uint8 (num_queues,cap,176,176) device, slot q * cap + s like the other planes (BlackCover's mask when the queued pairs
 * are augmented).  The same single launch, copies and checks; segB and q_segB must also be non-null and 16-byte aligned.
 * se3tn_append_pairs' four planes, poses and tails come out byte for byte as it writes them. */
int se3tn_append_pairs_seg(se3tn_ctx* ctx, const uint8_t* rgbA, const uint16_t* depthA, const uint8_t* rgbB, const uint16_t* depthB,
                           const int32_t* seg_count, const double* A_in_cam, const double* B_in_cam,
                           const int32_t* queue_ids_host, const int32_t* queue_ids_dev, int n,
                           int num_queues, int cap, const int32_t* tails_host, int32_t* tails_dev,
                           uint8_t* q_rgbA, uint16_t* q_depthA, uint8_t* q_rgbB, uint16_t* q_depthB, double* q_A_in_cam, double* q_B_in_cam,
                           const uint8_t* segB, uint8_t* q_segB, void* stream);

/* ---- introspection (tests / profiling) -------------------------------------------------------- */

/* Device pointer + per-image float count of an internal NHWC activation buffer.
 * ids: 0 stemA 1 stemB 2 Y1A 3 Y1B 4 P1A 5 P1B 6 T1 7 T2 8 U 9 CAT 10 F1 11 T4 12 F2 13 H1 14 H2 15 H3 */
int se3tn_debug_buffer(se3tn_ctx* ctx, int id, float** ptr, size_t* floats_per_image);

/* Per-kernel device timing for bench.py's roofline line: when enabled, every launch of the hot path
 * is bracketed by CUDA events on the caller's stream.  se3tn_get_profile synchronises those events
 * and writes SE3TN_PROFILE_SLOTS durations (ms) of the LAST call: [0..13] the 14 conv launches in
 * schedule order, [14],[15] the two max-pools, [16] head, [17] preprocess/normalize, [18] pose update,
 * [19] input repack (se3tn_forward only), [20] render, [21] loss (se3tn_eval_pairs: the reduction of the head's loss terms, or
 * the stand-alone loss launch in SE3TN_PREC_FP32; se3tn_pair_loss).  Slots that did not run read 0. */
#define SE3TN_PROFILE_SLOTS 22
int se3tn_set_profiling(se3tn_ctx* ctx, int enable);
int se3tn_get_profile(se3tn_ctx* ctx, float* ms);

/* Device-side timeline of the conv kernels (contexts created with SE3TN_TRACE=1 in the environment): synchronises the
 * device and copies 14 x 256 x 8 uint64 to the HOST: for conv launch l and CTA b, 8 %globaltimer (ns) stamps of the LAST
 * forward -- 0 entry, 1 setup done, 2 first weights in shared memory, 3 first activation unit, 4 last MMA committed,
 * 5 first accumulator ready, 6 last epilogue done, 7 exit (low 8 bits replaced by the SM id); launch 8 (the trunk) is followed by
 * its per-unit stamps in 9-13.  Then, for the 8 resident-weight launches, SE3TN_TRACE_TILES x 4 per-tile stamps each (enough
 * for the stems at 64 images) -- 0 first activation unit, 1 last MMA completed, 2 accumulator handed to the epilogue, 3 epilogue
 * done (low 8 bits replaced by the CTA index); tiles that did not run read 0.  Profiling tool only. */
#define SE3TN_TRACE_TILES 5184
#define SE3TN_TRACE_WORDS (14 * 256 * 8 + 8 * SE3TN_TRACE_TILES * 4)
int se3tn_get_trace(se3tn_ctx* ctx, unsigned long long* out);

/* Number of kernels the last forward / track_batch / track_render / eval_pairs / pair_loss call on this context launched (for a
 * replayed CUDA graph: the kernels inside it; a step that fills the depth counts the fill's launches, and a step with the fit
 * check its 3: se3tn_track_opts).
 * se3tn_track_batch, se3tn_track_render, their _host variants and se3tn_eval_pairs capture each distinct step into a CUDA
 * graph the first time they see it and replay it afterwards -- one graph launch per step.  Two calls are the same step when
 * every value their kernels are given is the same: tracking or validation, n, precision, the frame's H and W, K, the two
 * normalizers, the first weight id and whether the ids use more than one set, the render mode and camera image size, the
 * depth fill, the refinement count and fit check of a step that renders input A (se3tn_track_opts),
 * and the address of every device array, in or out.  A replay reads what those
 * arrays hold at the time, and a call's host ids only decide the first id and the mix.  SE3TN_GRAPH=0 in the environment,
 * an enabled profiler or SE3TN_PREC_FP32 use plain stream launches.
 * se3tn_perturb_pairs steps are captured and keyed the same way.
 * se3tn_last_step_was_graph: 1 if the last track_batch / track_render / eval_pairs / perturb_pairs call was a graph launch. */
int se3tn_last_step_was_graph(se3tn_ctx* ctx);
int se3tn_last_launch_count(se3tn_ctx* ctx);

/* Bytes of device scratch the context holds for se3tn_add_adi_sets / se3tn_vocap_sets / se3tn_draw_tracks (0 before the first
 * call). */
size_t se3tn_metrics_scratch_bytes(se3tn_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* SE3TN_H */
