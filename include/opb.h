/*
 * opb.h -- C ABI of libopb.so: the H100-native (sm_90a) OpenPose inference hot path.
 *
 * The reference (DeNA/Chainer_Realtime_Multi-Person_Pose_Estimation) is pure Python and has
 * no FFI layer; its drop-in boundary is the Python module `pose_detector`.  This header is the
 * native boundary *underneath* that module: every entry point replaces one block of
 * reference code (cited as file:line relative to the reference tree) and is what a
 * maintainer of the reference would bind with ctypes (see INTEGRATION.md).
 *
 * Conventions
 *   - plain C types only; no torch / numpy types.
 *   - every function returns 0 on success or a negative opb_status; the message is
 *     available from opb_last_error().  The Python wrapper raises on non-zero.
 *   - `loc` arguments: OPB_HOST (pageable or pinned host memory) or OPB_DEVICE (memory on
 *     the context's device).  Output buffers are caller-allocated with an explicit capacity;
 *     the number of valid rows is returned through an int* argument.
 *   - one context per device; calls on one context are serialised on its stream
 *     (opb_set_stream installs a caller-owned cudaStream_t, e.g. torch's current stream).
 *   - there is NO CPU fallback: every compute entry point launches sm_90a kernels.
 */
#ifndef OPB_H_
#define OPB_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OPB_N_JOINTS 18
#define OPB_N_LIMBS 19
#define OPB_MAX_TAPS 64

typedef enum {
  OPB_OK = 0,
  OPB_ERR_CUDA = -1,          /* CUDA runtime / driver error                                   */
  OPB_ERR_ARG = -2,           /* bad argument                                                  */
  OPB_ERR_STATE = -3,         /* e.g. forward before weights were finalised                    */
  OPB_ERR_CAPACITY = -4,      /* a caller buffer or an internal list overflowed (never silent) */
  OPB_ERR_INDEX = -5,         /* grouping found >=3 matching subsets: the reference raises
                                 IndexError at pose_detector.py:197                            */
  OPB_ERR_UNSUPPORTED = -6
} opb_status;

enum { OPB_HOST = 0, OPB_DEVICE = 1 };
enum { OPB_F32_NCHW = 0, OPB_U8_NHWC_BGR = 1 };          /* opb_forward input formats       */
enum { OPB_PRECISION_FAST = 0, OPB_PRECISION_PARITY = 1, OPB_PRECISION_COMP = 2 };
/* FAST: fp16 operands, fp32 accumulate (map error ~3e-3).  PARITY: split-fp16 (hi+lo, 3 MMAs, two-level accumulation;
 * ~2e-5).  COMP ("compensated"): fp16 main product + 8-bit-float first-order rounding corrections (2 MMAs; ~1e-4),
 * the fastest precision inside north_star's 1e-3 map tolerance. */
enum { OPB_UPSAMPLE_BILINEAR_AC = 0, OPB_UPSAMPLE_BICUBIC = 1 };

/* Constants of entity.py:71-105 (`params`) plus the 21 Gaussian taps of
 * scipy.ndimage.gaussian_filter(sigma=2.5) (pose_detector.py:86), computed by the host in
 * float64 exactly as scipy does, and the capacities of the device-side lists. */
typedef struct opb_params {
  int32_t limbs[OPB_N_LIMBS][2];      /* entity.py:85-105 limbs_point                          */
  double heatmap_peak_thresh;         /* 0.05  entity.py:79                                    */
  double inner_product_thresh;        /* 0.05  entity.py:80                                    */
  double limb_length_ratio;           /* 1.0   entity.py:81                                    */
  double length_penalty_value;        /* 1     entity.py:82                                    */
  double n_subset_limbs_thresh;       /* 3     entity.py:83                                    */
  double subset_score_thresh;         /* 0.2   entity.py:84                                    */
  int32_t n_integ_points;             /* 10    entity.py:77 (only 10 is supported)             */
  int32_t n_integ_points_thresh;      /* 8     entity.py:78                                    */
  int32_t gauss_radius;               /* 10 = int(4.0*2.5+0.5)                                 */
  int32_t reserved0;
  double gauss_taps[OPB_MAX_TAPS];    /* 2*gauss_radius+1 normalised float64 taps              */
  int32_t max_peaks;                  /* per image   (default 8192)                            */
  int32_t max_candidates;             /* per (image, limb) accepted PAF candidates (def 32768) */
  int32_t max_persons;                /* per image subsets alive at any time (default 1024, <= 4096) */
  int32_t reserved1;
} opb_params;

/* Fixed-size per-image result record written by opb_detect_batch (device-resident path) and
 * exchanged between GPUs with one all-gather.  Coordinates are integer peak positions at map
 * resolution so that the host can redo the float64 rescale of pose_detector.py:513-514
 * exactly.  joint id -1 = missing. */
typedef struct opb_person {
  double score;                       /* subsets[:, -2]                                        */
  double count;                       /* subsets[:, -1] (non-integer after a merge, :217)      */
  int32_t peak_id[OPB_N_JOINTS];      /* index into the image's peak table, -1 = none          */
  int32_t x[OPB_N_JOINTS];
  int32_t y[OPB_N_JOINTS];
  int32_t pad[2];
} opb_person;                          /* 16 + 3*72 + 8 = 240 bytes                             */

typedef struct opb_image_header {
  int32_t n_peaks;
  int32_t n_persons;
  int32_t status;                     /* 0 or an opb_status (capacity / index error)           */
  int32_t n_connections;              /* total over the 19 limbs                               */
} opb_image_header;

typedef struct opb_ctx opb_ctx;

/* -- lifetime ---------------------------------------------------------------------------- */
/* replaces PoseDetector.__init__ device selection, pose_detector.py:28-35 */
int opb_create(opb_ctx** out, int device, const opb_params* params);
void opb_destroy(opb_ctx* ctx);
const char* opb_last_error(const opb_ctx* ctx);     /* ctx may be NULL: last create error      */
int opb_set_stream(opb_ctx* ctx, void* cuda_stream); /* cudaStream_t; NULL = context's own     */
int opb_synchronize(opb_ctx* ctx);
int opb_version(void);

/* -- weights: replaces serializers.load_npz(weights_file, model), pose_detector.py:25-26 --- */
/* W is [Cout,Cin,k,k] float32 (Chainer OIHW), b is [Cout]; both host pointers. 92 calls.   */
int opb_load_weights(opb_ctx* ctx, const char* layer, const float* W, const int64_t shape[4],
                     const float* b);
/* repacks to K-major fp16 (and the hi/lo split for OPB_PRECISION_PARITY) and uploads.       */
int opb_finalize_weights(opb_ctx* ctx, int precision_mode);

/* -- CocoPoseNet forward: replaces self.model(x), pose_detector.py:499 / :451
 *    (models/CocoPoseNet.py:132-262).  x: [N,3,H,W] float32 (OPB_F32_NCHW, already
 *    preprocessed as pose_detector.py:426-431) or [N,H,W,3] uint8 BGR (OPB_U8_NHWC_BGR,
 *    /255-0.5 fused into the first conv).  H, W multiples of 8.
 *    paf_out [N,38,H/8,W/8], heat_out [N,19,H/8,W/8] float32.                               */
int opb_forward(opb_ctx* ctx, const void* x, int x_format, int x_loc, int n, int h, int w,
                float* paf_out, float* heat_out, int out_loc);

/* -- upsample: replaces F.resize_images (pose_detector.py:501-502, OPB_UPSAMPLE_BILINEAR_AC:
 *    align-corners bilinear, bit-exact restatement of Chainer's ResizeImages.forward) and one
 *    cv2.resize(INTER_CUBIC) of float maps (pose_detector.py:461-467, OPB_UPSAMPLE_BICUBIC).
 *    in [planes,h,w] -> out [planes,out_h,out_w] float32.  The crop / accumulate / average
 *    steps of detect_precise are inside opb_precise_add_scale.                              */
int opb_upsample(opb_ctx* ctx, int mode, const float* in, int in_loc, int planes, int h, int w,
                 float* out, int out_loc, int out_h, int out_w);

/* -- peaks: replaces compute_peaks_from_heatmaps (CPU branch), pose_detector.py:75-110.
 *    heat [c_plus_1,H,W] float32 (last channel = background, dropped).  peaks_out rows are
 *    (type, x, y, score, id) float64, ordered channel-major then row-major.                 */
int opb_peaks(opb_ctx* ctx, const float* heat, int heat_loc, int c_plus_1, int h, int w,
              double* peaks_out, int peaks_cap, int* n_peaks);

/* -- connections: replaces compute_connections + compute_candidate_connections,
 *    pose_detector.py:135-181.  paf [38,H,W] float32; peaks [n,5] float64 (host).
 *    conn_out rows (id_a, id_b, score) float64, limb after limb; conn_counts[19].           */
int opb_connections(opb_ctx* ctx, const float* paf, int paf_loc, int h, int w, const double* peaks,
                    int n_peaks, double img_len, double* conn_out, int conn_cap, int* conn_counts);

/* -- candidates of ONE limb: replaces compute_candidate_connections, pose_detector.py:135-159.
 *    paf [2,H,W] float32 host; cand_a [n_a,4], cand_b [n_b,4] float64 rows (x, y, score, id).
 *    out rows (id_a, id_b, score) float64, sorted by descending score (stable, :158).          */
int opb_candidates(opb_ctx* ctx, const float* paf, int h, int w, const double* cand_a, int n_a,
                   const double* cand_b, int n_b, double img_len, double* out, int out_cap, int* n_out);

/* -- grouping: replaces grouping_key_points, pose_detector.py:183-250.
 *    subsets_out rows of 20 float64 (18 ids, score, count).                                  */
int opb_group(opb_ctx* ctx, const double* conns, const int* conn_counts, const double* peaks,
              int n_peaks, double* subsets_out, int subsets_cap, int* n_subsets);

/* -- fused device-resident batch path: PoseDetector.__call__ for a batch, pose_detector.py
 *    :493-517 minus the host resize.  imgs [N,H,W,3] uint8 BGR at network-input size.
 *    Runs conv chain -> bilinear upsample to (map_h,map_w) -> peaks -> connections ->
 *    grouping entirely on the device.  headers_out [N], persons_out [N*max_persons]
 *    (host or device per out_loc).  If inject_paf / inject_heat are non-NULL they are
 *    device arrays [N,38,H/8,W/8] / [N,19,H/8,W/8] that REPLACE the network output before
 *    the upsample (the conv chain still runs); used with synthetic 8-person maps because
 *    random weights cannot produce people (SURVEY.md 8d).                                    */
int opb_detect_batch(opb_ctx* ctx, const uint8_t* imgs, int imgs_loc, int n, int h, int w, int map_h,
                     int map_w, double img_len, const float* inject_paf, const float* inject_heat,
                     opb_image_header* headers_out, opb_person* persons_out, int out_loc);

/* -- the post-process half of PoseDetector.__call__ on its own (pose_detector.py:501-512): network outputs
 *    paf_lo [N,38,h8,w8] / heat_lo [N,19,h8,w8] float32 (host or device per maps_loc) -> F.resize_images to
 *    (map_h, map_w) -> peaks -> connections -> grouping, records as in opb_detect_batch.  For callers that run
 *    the network elsewhere, and the entry the no-GPU emulation tests drive (the conv chain cannot be emulated).
 *    With OPB_PAF_LOWRES=1 / OPB_FUSED_PEAKS=1|2 in the environment at opb_create (experimental, also honoured by
 *    opb_detect_batch / opb_detect_image / opb_stream_submit) the PAF line integrals / the peak kernel interpolate
 *    from the low-resolution maps on demand instead of reading materialised full-resolution maps: same results
 *    bit for bit, without the 42 MB per 320x576 image of full-resolution maps going through HBM.            */
int opb_postprocess_batch(opb_ctx* ctx, const float* paf_lo, const float* heat_lo, int maps_loc, int n, int h8,
                          int w8, int map_h, int map_w, double img_len, opb_image_header* headers_out,
                          opb_person* persons_out, int out_loc);

/* -- device-side ingest: replaces cv2.resize(orig_img, (input_w, input_h)) (default INTER_LINEAR on
 *    uint8 BGR, pose_detector.py:493), bit-exact with OpenCV's 8-bit fixed-point path.
 *    src [n,h0,w0,3] -> dst [n,h,w,3] uint8.                                                     */
int opb_resize_linear_u8(opb_ctx* ctx, const uint8_t* src, int src_loc, int n, int h0, int w0,
                         uint8_t* dst, int dst_loc, int h, int w);
/* cv2.resize(orig_img, ..., interpolation=cv2.INTER_CUBIC) on uint8 BGR (detect_precise, pose_detector.py:443):
 * OpenCV's own 8-bit cubic path (int16 Keys taps x 2048, int32 horizontal pass, float32 vertical pass with the
 * fixed-point scalar tail), bit-exact with cv2 when OpenCV does not dispatch to IPP (cv2.ipp.setUseIPP(False), or a
 * build without IPP); IPP's ippiResizeCubic differs from it by 1 LSB in 4-8 % of the pixels.                 */
int opb_resize_cubic_u8(opb_ctx* ctx, const uint8_t* src, int src_loc, int n, int h0, int w0,
                        uint8_t* dst, int dst_loc, int h, int w);
/* PoseDetector.__call__ for ONE frame of arbitrary size (pose_detector.py:484-517): uploads the
 * original frame, resizes it on the device to (in_h, in_w), then runs the same pipeline as
 * opb_detect_batch with n = 1.                                                                  */
int opb_detect_image(opb_ctx* ctx, const uint8_t* img, int img_loc, int orig_h, int orig_w, int in_h,
                     int in_w, int map_h, int map_w, double img_len, opb_image_header* header_out,
                     opb_person* persons_out, int out_loc);

/* -- skeleton overlay: replaces draw_person_pose(orig_img, poses), pose_detector.py:520-553 (the camera loop's
 *    per-frame drawing, camera_pose_demo.py:27).  img [h,w,3] uint8 BGR -> out [h,w,3] = img.copy() with, per person,
 *    the 17 drawn limbs (cv2.line thickness 2; limbs 9 and 13 skipped) and then the joints (cv2.circle radius 3,
 *    filled) in the reference's order and colours, rasterised exactly as OpenCV 4.x does (csrc/overlay.cuh).
 *    poses: host int32 [n_poses,18,3] = poses.round().astype('i') (x, y, visible != 0).  Every drawn joint must lie
 *    inside the image (true for any pose the detector returns); otherwise OPB_ERR_ARG.                           */
int opb_draw_person_pose(opb_ctx* ctx, const uint8_t* img, int img_loc, int h, int w, const int32_t* poses,
                         int n_poses, uint8_t* out, int out_loc);
/* same, taking the persons of image `image_index` of the last detect call straight from the device-resident records
 * (no host round trip of the poses): joint = rint(peak * (sx, sy)) in float64 as :513-514 and :539 compute it
 * (sx = orig_w / map_w, sy = orig_h / map_h; 1, 1 after the precise path).                                        */
int opb_draw_last_result(opb_ctx* ctx, int image_index, const uint8_t* img, int img_loc, int h, int w, double sx,
                         double sy, uint8_t* out, int out_loc);
/* -- the whole-body result picture of demo.py:28-57 in one call: out = cv2.addWeighted(img, 0.6,
 *    draw_person_pose(img, poses), 0.4, 0), then for every part in order its keypoints -- draw_face_keypoints
 *    (face_detector.py:79-97: 70 dots of radius 2, then the 63 face_line_indices segments of thickness 1) or
 *    draw_hand_keypoints (hand_detector.py:89-117: per finger segment dot, dot, line, in the finger's colour) at
 *    (left, top) -- and then cv2.rectangle((left, top), (right, bottom), (255, 255, 255), 1).  Pixel-identical to
 *    those cv2 calls (csrc/overlay.cuh), parts and boxes partly or wholly outside the frame included.
 *    poses: host int32 [n_poses,18,3] as for opb_draw_person_pose (every present joint inside the image).
 *    points: host int32 [n_points,3] = (x, y, present) in crop coordinates; part i reads rows first_point ..
 *    first_point + 69 (face) or + 20 (hand).  One upload of the frame (none with OPB_DEVICE) and one of the tables,
 *    two launches, one download and one synchronisation.  OPB_ERR_ARG (nothing enqueued) for an unknown kind, a
 *    negative count, points past n_points, a present joint outside the image, or a box or drawn keypoint coordinate of
 *    magnitude above 2^20.                                                                                      */
enum { OPB_PART_FACE = 0, OPB_PART_HAND = 1 };
typedef struct opb_part {
  int32_t kind;                       /* OPB_PART_FACE (70 points) or OPB_PART_HAND (21 points)                 */
  int32_t left, top, right, bottom;   /* the crop box of crop_face / crop_hands                                 */
  int32_t first_point;                /* row of the part's first keypoint in points                             */
} opb_part;
int opb_draw_whole_body(opb_ctx* ctx, const uint8_t* img, int img_loc, int h, int w, const int32_t* poses,
                        int n_poses, const opb_part* parts, int n_parts, const int32_t* points, int n_points,
                        uint8_t* out, int out_loc);

/* -- streaming mode: the camera loop of camera_pose_demo.py:20-31, pipelined.  Two slots; submit()
 *    enqueues [pinned staging ->] H2D on a copy stream, the device resize (if orig != in), the whole
 *    pipeline and the D2H of the records, and returns without waiting; collect() blocks until that
 *    slot's records are on the host.  Submitting batch i+1 before collecting batch i overlaps its
 *    upload with batch i's kernels.  frames: [n,orig_h,orig_w,3] uint8 BGR, HOST (pinned or pageable) or DEVICE
 *    (used in place; must stay valid until the slot is collected).
 *    inject_* as in opb_detect_batch (device pointers or NULL).                                 */
int opb_stream_submit(opb_ctx* ctx, const uint8_t* frames, int frames_loc, int n, int orig_h, int orig_w,
                      int in_h, int in_w, int map_h, int map_w, double img_len, const float* inject_paf,
                      const float* inject_heat, int slot);
int opb_stream_collect(opb_ctx* ctx, int slot, opb_image_header* headers_out, opb_person* persons_out);
/* Slot 1 runs on a library-owned stream (its kernels fill the tails and launch gaps of slot 0's).  join makes the
 * context's stream (opb_set_stream) wait for every submitted, uncollected batch -- for callers that time or
 * order other work on that stream.                                                              */
int opb_stream_join(opb_ctx* ctx);

/* -- multi-GPU (SURVEY.md 8e: images shard by rank; the reference has no multi-device path, SURVEY 2a) ------------
 * The ONE collective of the path: an ncclAllGather of the fixed-size result records of a streaming slot's batch,
 * [n opb_image_header | n x max_persons opb_person] = opb_record_block_bytes(ctx, n) bytes per rank, straight from
 * the device-resident record block (no host hop), enqueued on the slot's stream behind its pipeline; gathered_dev
 * (device, world x that many bytes) then holds every rank's block in rank order.  opb_stream_collect / opb_stream_join
 * of that slot afterwards also wait for the collective.  NCCL is resolved at run time (dlopen libnccl.so.2, or
 * $OPB_NCCL_LIB) -- the process that calls this already carries it (torch.distributed, or a program linked to NCCL).
 * opb_nccl_unique_id / opb_nccl_comm_init / opb_nccl_comm_destroy wrap ncclGetUniqueId / ncclCommInitRank /
 * ncclCommDestroy for callers without their own NCCL binding (rank 0 creates the 128-byte id and ships it to the
 * other ranks through whatever channel it has; one communicator per process = per GPU).                        */
int opb_nccl_unique_id(uint8_t id_out[128]);
int opb_nccl_comm_init(opb_ctx* ctx, void** nccl_comm_out, int world, int rank, const uint8_t id[128]);
int opb_nccl_comm_destroy(void* nccl_comm);
size_t opb_record_block_bytes(const opb_ctx* ctx, int n);
int opb_allgather_results(opb_ctx* ctx, void* nccl_comm /* ncclComm_t */, int slot, void* gathered_dev);

/* -- face / hand nets (SURVEY 8f#2).  A context whose loaded layers contain "conv6_2_CPM" is a FaceNet /
 *    HandNet context (models/FaceNet.py:10-76, models/HandNet.py; 52 layers, final 1x1 with 71 / 22 channels):
 *    opb_forward then returns only heat_out [n, 71|22, h/8, w/8] and uint8 input is normalised /256 - 0.5
 *    (face_detector.py:32).
 *    opb_keypoints_detect = FaceDetector.__call__ (face_detector.py:28-41) / HandDetector.__call__
 *    (hand_detector.py:28-51) for one BGR crop [img_h,img_w,3]: device cv2-exact resize to net_size^2,
 *    forward, F.resize_images to the crop size, gaussian_filter(sigma 2.5), per-channel maximum.
 *    out [C-1][3] = (x, y, conf), valid [C-1] = conf > thresh (float32 compare).  mirror = 1 reports positions
 *    in the horizontally flipped maps (hand_type "left": the caller passes the already flipped crop,
 *    hand_detector.py:29-30,46-47).  maps_out (host, may be NULL) receives the unsmoothed upsampled maps.
 *    opb_keypoints_from_heatmaps = compute_peaks_from_heatmaps (face_detector.py:55-67) on caller maps
 *    [planes,h,w] (background channel already dropped).                                          */
int opb_keypoints_detect(opb_ctx* ctx, const uint8_t* img, int img_loc, int img_h, int img_w, int net_size,
                         int mirror, double thresh, double* out, int32_t* valid, float* maps_out);
int opb_keypoints_from_heatmaps(opb_ctx* ctx, const float* heat, int heat_loc, int planes, int h, int w,
                                int mirror, double thresh, double* out, int32_t* valid);

/* -- all face (or hand) crops of one frame in one call: the result for crop i equals opb_keypoints_detect on
 *    flip_i(PoseDetector.crop_image(frame, bbox_i)) with mirror = flip_i, bit for bit at equal conv tile shapes.
 *    The canvas of a crop is (bottom-top) x (right-left); frame pixels outside it are read as 0.  The frame
 *    [frame_h, frame_w, 3] uint8 BGR is uploaded once (or read in place with OPB_DEVICE); crops run through the net
 *    in chunks of at most 16 (full chunks of 16, then the remainder rounded up to a power of two), and the upsample,
 *    smoothing and arg-max of all crops are ragged launches.  One device-to-host copy and one synchronisation per call.
 *    out [n][C-1][3] = (x, y, conf) in crop coordinates, valid [n][C-1].  OPB_ERR_ARG for a crop with a non-positive
 *    width or height (nothing is launched); n == 0 returns at once.                                        */
typedef struct opb_crop {
  int32_t left, top, right, bottom;   /* crop_image bbox; zero fill outside the frame                          */
  int32_t flip;                       /* 1: cv2.flip(crop, 1) before the net, positions reported unflipped     */
  int32_t reserved;
} opb_crop;
int opb_keypoints_detect_crops(opb_ctx* ctx, const uint8_t* frame, int frame_loc, int frame_h, int frame_w,
                               const opb_crop* crops, int n, int net_size, double thresh,
                               double* out /* [n][C-1][3] */, int32_t* valid /* [n][C-1] */);

/* ---- Haar cascade (cv2.CascadeClassifier.detectMultiScale, stump-based HAAR cascades, bit-exact) ----
 * opb_cascade_load: one cascade per context (a second load replaces the first).  Flat tables as the XML holds them:
 *   stage_ntrees / stage_threshold [n_stages] (stageThreshold as stored; the 1e-5f margin is applied here),
 *   stump_feature / stump_threshold / stump_left / stump_right [n_stumps] stage by stage,
 *   rects [n_features][3][4] (x, y, w, h; unused rects zero) and weights [n_features][3] (0: rect absent).
 *   OPB_ERR_ARG for a rect outside the window, a feature index out of range, ntrees that do not add up to n_stumps,
 *   or more than 64 stages. */
int opb_cascade_load(opb_ctx* ctx, int win_w, int win_h, int n_stages, const int32_t* stage_ntrees,
                     const float* stage_threshold, int n_stumps, const int32_t* stump_feature,
                     const float* stump_threshold, const float* stump_left, const float* stump_right, int n_features,
                     const int32_t* rects, const float* weights);
/* opb_cascade_detect: detectMultiScale(gray, scale_factor, min_neighbors, (min_w, min_h), (max_w, max_h)) of an
 *   h x w frame with channels 1 (gray) or 3 (BGR, converted as cvtColor(BGR2GRAY)).  rects_out [cap][4] (x, y, w, h)
 *   sorted by (y, x, w, h).  Per call: one frame upload, five launches (pyramid, row scan, column scan, windows,
 *   compaction), one candidate download and one synchronisation; grouping runs on the host.  Per-shape tables are
 *   uploaded on the first call of a shape.  OPB_ERR_ARG (nothing enqueued) for scale_factor <= 1, a negative
 *   argument or channels other than 1 and 3; OPB_ERR_STATE without a cascade; OPB_ERR_CAPACITY when the result
 *   (or the raw candidate list, 8192 entries) does not fit, never truncation. */
int opb_cascade_detect(opb_ctx* ctx, const uint8_t* img, int img_loc, int h, int w, int channels, double scale_factor,
                       int min_neighbors, int min_w, int min_h, int max_w, int max_h, int32_t* rects_out, int cap,
                       int* n_out);
/* opb_face_detect_frame: the per-frame work of camera_face_demo.py:47-56 -- the cascade on the BGR frame, then for
 *   every face rect its zero-padded square crop (crop_face of that demo, scaled by crop_scale), FaceNet on all crops
 *   in the chunks of opb_keypoints_detect_crops, and the keypoints.  rects_out as opb_cascade_detect; out [cap][C-1][3]
 *   and valid [cap][C-1] as opb_keypoints_detect_crops, in crop coordinates; left_top [cap][2] = (crop_left,
 *   crop_top).  Per call: one frame upload, one candidate download and synchronisation, one crop-table upload, one
 *   keypoint download and synchronisation.  Errors as opb_cascade_detect, and OPB_ERR_STATE without FaceNet. */
int opb_face_detect_frame(opb_ctx* ctx, const uint8_t* frame, int frame_loc, int h, int w, double scale_factor,
                          int min_neighbors, int min_w, int min_h, int max_w, int max_h, double crop_scale,
                          int net_size, double thresh, int32_t* rects_out, int cap, int* n_out, double* out,
                          int32_t* valid, int32_t* left_top);
/* Test hook: the result code (-1 variance test failed, -k rejected by stage k, 1 passed) and final stage sum of every
 *   window of every scale, before the skip rule: layers in scale order, windows row by row (y, x in the layer's
 *   ystep).  *n_out = number of windows; OPB_ERR_CAPACITY when it exceeds cap. */
int opb_test_cascade_windows(opb_ctx* ctx, const uint8_t* img, int img_loc, int h, int w, int channels,
                             double scale_factor, int min_w, int min_h, int max_w, int max_h, int32_t* codes_out,
                             double* sums_out, int cap, int* n_out);

/* ---- the whole-body frame of demo.py:24-57 in one call ----
 * opb_whole_body_frame: pose (CocoPoseNet), face (FaceNet) and hand (HandNet) are three contexts on one device.  In order:
 *   1. one upload of the BGR frame [orig_h, orig_w, 3] to the pose context (none with OPB_DEVICE: read in place), the
 *      device resize to (in_h, in_w) and the pipeline of opb_detect_image; inject_paf / inject_heat as in
 *      opb_detect_batch (device maps that replace the network output, or NULL);
 *   2. the crop-box kernel (csrc/whole_body.cuh) on the device records: per person PoseDetector.get_unit_length,
 *      crop_face and crop_hands of pose_detector.py in float64, bit for bit, with sx = orig_w / map_w and
 *      sy = orig_h / map_h; then one download of the records and the box tables and one synchronisation;
 *   3. FaceNet on the face crops on the face context's stream and HandNet on the hand crops (left hands mirrored) on the
 *      hand context's stream, both reading the frame in place from the pose context's buffer; both are enqueued before
 *      either is collected, so they overlap.  Each equals opb_keypoints_detect_crops on the same boxes; a net without
 *      crops is skipped;
 *   4. with picture_out != NULL, the picture of opb_draw_whole_body on the resident frame -- the skeleton from the
 *      device records (as opb_draw_last_result), then the parts -- and one download of it.
 * Deviation from demo.py, which raises on such persons: a person whose unit length is not finite (no limb of positive
 * length) gets no part, and a box of non-positive width or height is not a part.  Parts come in the demo's order (per
 * person: face, left hand, right hand).  Outputs: header_out and persons_out (max_persons records) as
 * opb_detect_image; parts_out [parts_cap], *n_parts; face_out [parts_cap][70][3] / face_valid [parts_cap][70] and
 * hand_out [parts_cap][21][3] / hand_valid [parts_cap][21] as opb_keypoints_detect_crops, row p.row for part p;
 * picture_out [orig_h, orig_w, 3] host.  What crosses contexts: the frame buffer of the pose context, read by the face
 * and hand streams after the pose stream was synchronised.  No context has work pending on a successful return, and the
 * pose context holds this frame's result (opb_draw_last_result, opb_get_image_detail).
 * OPB_ERR_ARG / OPB_ERR_STATE before anything is enqueued for contexts on different devices, a context that does not
 * hold its net or has no finalised weights, and bad sizes or outputs; the frame's record status (as opb_detect_batch
 * reports it in the header) is returned as the error; OPB_ERR_UNSUPPORTED for a box edge beyond int32;
 * OPB_ERR_CAPACITY when the parts do not fit parts_cap (*n_parts holds the count). */
enum { OPB_SIDE_FACE = 0, OPB_SIDE_LEFT = 1, OPB_SIDE_RIGHT = 2 };
typedef struct opb_wb_part {
  int32_t kind;                       /* OPB_PART_FACE or OPB_PART_HAND                                          */
  int32_t left, top, right, bottom;   /* the crop box of crop_face / crop_hands                                 */
  int32_t row;                        /* the part's keypoint row in face_out / hand_out                         */
  int32_t person;                     /* index of the person in persons_out                                     */
  int32_t side;                       /* OPB_SIDE_FACE / OPB_SIDE_LEFT / OPB_SIDE_RIGHT                        */
} opb_wb_part;
int opb_whole_body_frame(opb_ctx* pose, opb_ctx* face, opb_ctx* hand, const uint8_t* img, int img_loc, int orig_h,
                         int orig_w, int in_h, int in_w, int map_h, int map_w, double img_len, const float* inject_paf,
                         const float* inject_heat, int face_net_size, double face_thresh, int hand_net_size,
                         double hand_thresh, opb_image_header* header_out, opb_person* persons_out,
                         opb_wb_part* parts_out, int parts_cap, int* n_parts, double* face_out, int32_t* face_valid,
                         double* hand_out, int32_t* hand_valid, uint8_t* picture_out);
/* opb_whole_body_batch: opb_whole_body_frame for n >= 1 equally sized BGR frames [n, orig_h, orig_w, 3] (host, or
 * read in place with OPB_DEVICE); opb_whole_body_frame is its n = 1 case.  inject_paf / inject_heat are
 * [n, 38|19, in_h/8, in_w/8].  Per call:
 *   1. one upload of all frames, one device resize of the batch and the pipeline at batch n (the launch sequence of
 *      opb_detect_batch / opb_stream_submit for n frames);
 *   2. one launch of the crop-box kernel for all frames (one block per frame), then one download of the records and
 *      the box tables and one synchronisation;
 *   3. the face crops of all frames, concatenated frame by frame, through FaceNet on the face context's stream and the
 *      hand crops likewise through HandNet on the hand context's stream, both enqueued before either is collected;
 *      forward chunks (full chunks of 16, then the remainder rounded up to a power of two) cross frame boundaries.
 *      Frames go through the nets in groups of whole frames whose crop maps stay under 2^30 floats per net (at least
 *      one frame per group), so that the map workspace stays bounded; each group has its own chunks and download;
 *   4. with pictures_out != NULL: one table upload, at most one records -> poses launch, one raster and one paint
 *      launch for all n pictures, then one download and one synchronisation.
 * Outputs: headers_out [n] and persons_out [n][max_persons] as opb_stream_collect returns them; parts_out [parts_cap]
 * (person counts within its frame, row indexes the batch-wide face / hand tables), *n_parts; frame_parts [n + 1]
 * prefix offsets: frame f owns parts frame_parts[f] .. frame_parts[f+1] - 1, in the demo's order within the frame;
 * face_out / face_valid / hand_out / hand_valid as opb_whole_body_frame with rows over the whole batch;
 * pictures_out [n, orig_h, orig_w, 3] host.  The pose context holds the batch's result (opb_draw_last_result with
 * image_index f).  Errors as opb_whole_body_frame, all checked before anything is enqueued, plus OPB_ERR_ARG for
 * n < 1; the record status of the first frame that carries one is returned after headers_out and persons_out are
 * written; OPB_ERR_UNSUPPORTED for a box edge beyond int32; OPB_ERR_CAPACITY when the parts of the batch exceed
 * parts_cap (*n_parts holds the count). */
int opb_whole_body_batch(opb_ctx* pose, opb_ctx* face, opb_ctx* hand, const uint8_t* frames, int frames_loc, int n,
                         int orig_h, int orig_w, int in_h, int in_w, int map_h, int map_w, double img_len,
                         const float* inject_paf, const float* inject_heat, int face_net_size, double face_thresh,
                         int hand_net_size, double hand_thresh, opb_image_header* headers_out, opb_person* persons_out,
                         opb_wb_part* parts_out, int parts_cap, int* n_parts, int* frame_parts /* [n + 1] */,
                         double* face_out, int32_t* face_valid, double* hand_out, int32_t* hand_valid,
                         uint8_t* pictures_out);
/* Test hook: the crop-box kernel of opb_whole_body_frame on n host person records (all persons of one image).
 *   unit_out [n] float64 unit lengths (NaN without a positive limb), boxes_out [n][3][4] (face, left hand, right hand:
 *   left, top, right, bottom), present_out [n] (bit k: box k exists -- its joint is present and the unit length is
 *   finite -- boxes without the bit are not written), parts_out [3n][2] (person, side) of the kept parts in order,
 *   *n_parts.  OPB_ERR_UNSUPPORTED when a box edge does not fit int32. */
int opb_test_whole_body_boxes(opb_ctx* ctx, const opb_person* persons, int n, double sx, double sy, double* unit_out,
                              int32_t* boxes_out, int32_t* present_out, int32_t* parts_out, int* n_parts);
/* Test hook: the crop-box kernel of opb_whole_body_batch on the host records of n frames, headers [n] and
 *   persons [n][cap] (n * cap <= 65536), in one launch.  Per frame f: counts_out [n][4] (status, n_face, n_hand,
 *   n_parts: a record status error or OPB_ERR_UNSUPPORTED for a box edge beyond int32 is reported here, per frame),
 *   and the frame's sections unit_out [n][cap], boxes_out [n][cap][3][4], present_out [n][cap] as
 *   opb_test_whole_body_boxes, face_out [n][cap] and hand_out [n][2 cap] (the compacted crop tables, flip = 1 for
 *   left hands), parts_out [n][3 cap][4] (side, person, row into the frame's face or hand table, 0).  Entries a frame
 *   does not write are zero. */
int opb_test_whole_body_boxes_batch(opb_ctx* ctx, const opb_image_header* headers, const opb_person* persons, int n,
                                    int cap, double sx, double sy, int32_t* counts_out, double* unit_out,
                                    int32_t* boxes_out, int32_t* present_out, opb_crop* face_out, opb_crop* hand_out,
                                    int32_t* parts_out);

/* device pointers of the last opb_detect_batch outputs/intermediates (valid until the next
 * call with a different shape): 0 paf_lo, 1 heat_lo, 2 pafs (full-res), 3 heatmaps (full-res),
 * 4 headers, 5 persons, 6 peak table ([N,max_peaks] of {int32 type,x,y; float score})       */
void* opb_device_buffer(opb_ctx* ctx, int which);

/* Detail of image `img` of the last opb_detect_batch / opb_precise_finish: the peak table
 * ([n,5] float64 rows type,x,y,score,id), the 19 connection lists and the kept subsets
 * ([P,20] float64), i.e. the reference's all_peaks / all_connections / subsets.  Any output
 * pointer may be NULL.                                                                       */
int opb_get_image_detail(opb_ctx* ctx, int img, double* peaks_out, int peaks_cap, int* n_peaks,
                         double* conn_out, int conn_cap, int* conn_counts, double* subsets_out,
                         int subsets_cap, int* n_subsets);

/* -- multi-scale precise path: replaces detect_precise, pose_detector.py:433-482 -------------
 * begin: allocate/zero the [38|19, orig_h, orig_w] accumulators.
 * add_scale: padded uint8 BGR image [ph,pw,3] (already resized by the host with
 *   cv2.INTER_CUBIC and padded, :443-445) -> forward -> cubic x8 -> crop pad -> cubic to
 *   (orig_h, orig_w) -> accumulate; the last scale also divides by n_scales (:461-470).
 * finish: peaks -> connections -> grouping on the averaged maps (:475-481).                  */
int opb_precise_begin(opb_ctx* ctx, int orig_h, int orig_w);
int opb_precise_add_scale(opb_ctx* ctx, const uint8_t* img, int img_loc, int ph, int pw, int pad_h,
                          int pad_w, int scale_index, int n_scales);
/* same, with pad_image (pose_detector.py:46-55) on the device: img is the resized, UNPADDED frame [h,w,3];
 * the bottom / right margin up to the next multiple of `stride` is filled with pad_value (B,G,R).  */
int opb_precise_add_scale_unpadded(opb_ctx* ctx, const uint8_t* img, int img_loc, int h, int w, int stride,
                                   const uint8_t pad_value[3], int scale_index, int n_scales);
/* same, starting from the ORIGINAL frame [orig_h,orig_w,3]: the per-scale cv2.resize(..., INTER_CUBIC) to (h, w) of
 * :443 also runs on the device (opb_resize_cubic_u8's kernel), so one scale costs one upload of the original frame and
 * no host arithmetic.                                                                                           */
int opb_precise_add_scale_orig(opb_ctx* ctx, const uint8_t* orig, int img_loc, int orig_h, int orig_w, int h, int w,
                               int stride, const uint8_t pad_value[3], int scale_index, int n_scales);
int opb_precise_finish(opb_ctx* ctx, double img_len, opb_image_header* header_out,
                       opb_person* persons_out, int out_loc);
/* copies the full-resolution maps of image 0 of the current post-process workspace
 * (self.pafs / self.heatmaps of the precise path, :469-470) to the caller.                    */
int opb_download_maps(opb_ctx* ctx, float* pafs_out, float* heat_out, int out_loc);

/* -- instrumentation ---------------------------------------------------------------------- */
/* number of kernels launched by this context since creation (bench.py's gpu_launches)      */
int64_t opb_launch_count(const opb_ctx* ctx);
/* Times `reps` launches of one named stage of the cached pipeline of the last
 * opb_detect_batch / opb_forward shape with CUDA events on the context's stream; returns the
 * mean milliseconds per launch in *ms.  stage: "conv7x7" (the Mconv2..5 grouped launch),
 * "conv_chain", "upsample_paf", "peaks", "paf_integral", ...                                 */
int opb_time_stage(opb_ctx* ctx, const char* stage, int reps, float* ms);

/* -- test hooks (tests/ only) ---------------------------------------------------------------
 * single conv layer through the wgmma kernel: x [N,H,W,Cin] fp32 host, W [Cout,Cin,k,k],
 * b [Cout] -> y [N,H,W,Cout] fp32 host (activations are converted to fp16 / split-fp16 on the
 * device exactly as in the chain).  relu: bit 0 = ReLU, bit 1 = fuse the 2x2/2 max-pool (y is
 * then [N,H/2,W/2,Cout]).                                                                    */
int opb_test_conv(opb_ctx* ctx, const float* x, int n, int h, int w, int cin, const float* W,
                  const float* b, int cout, int ksize, int relu, int precision_mode, float* y);
/* conv1_1 alone (preprocess + 3x3 conv 3 -> 64 + ReLU), exactly as the chains run it.  x: uint8
 * BGR [N,H,W,3] (x_is_u8 != 0, normalised as v / u8_denom - 0.5) or preprocessed float32
 * [N,3,H,W]; W [64,3,3,3], b [64].  out receives the raw output tensor, N*H*W pixels of 128 B
 * (fast: 64 fp16) or 256 B (parity: 64 fp16 hi | 64 fp16 lo; compensated: 64 fp16 hi |
 * 64 B fp8(lo * 2^11) | 64 B fp8(v)).  The context's own conv1_1 weights are left untouched.  */
int opb_test_conv_first(opb_ctx* ctx, const void* x, int x_is_u8, int n, int h, int w, float u8_denom,
                        const float* W, const float* b, int precision_mode, uint8_t* out);

/* One problem of a conv launch of a chain: its input and output activation tensors (NHWC, `c` channels per plane,
 * `ctot` = c (fast) or 2c (parity: [hi | lo] fp16; compensated: [hi fp16 | 2c correction bytes]) halves per pixel), the
 * channel offsets it reads and writes, and the packed weights it multiplies.                                        */
typedef struct opb_conv_problem {
  int32_t in_h, in_w, in_c, in_ctot, in_coff;
  int32_t out_h, out_w, out_c, out_ctot, out_coff;   /* out_h, out_w: after the fused max-pool, if any         */
  int32_t cout_valid, relu, pool, has_out32;         /* has_out32: also writes fp32 maps [N][cout_valid][h][w] */
  int32_t cin_pad, cout_pad;
  float acc_scale;
  int32_t reserved;
} opb_conv_problem;
typedef struct opb_conv_record {
  char tag[32];
  char wkey[2][48];                                  /* packed-weight key per problem                          */
  int32_t ks, bn, drain, comp, n_problems, grid;
  int32_t shared_in;                                 /* the problems read one tensor (at their own offsets)    */
  int32_t reserved;
  opb_conv_problem prob[2];
} opb_conv_record;
/* The conv launches of the loaded model's chain at (n, h, w) (built if needed), one record per launch in launch
 * order.  *count = number of launches; OPB_ERR_CAPACITY when it exceeds cap (the first cap records are written). */
int opb_test_chain_convs(opb_ctx* ctx, int n, int h, int w, opb_conv_record* out, int cap, int* count);
/* Runs conv launch `index` of that chain on its own: uploads the raw bytes of each problem's whole input tensor (in0;
 * in1 when problem 1 reads another tensor), out_io as the prior content of the whole output tensor and out32_p as the
 * prior content of problem p's fp32 maps (when it has them), launches the op, and downloads all of them back into
 * out_io / out32_p.  The chain's activations are scratch for this hook.  OPB_ERR_ARG for a bad index or a missing
 * buffer; OPB_ERR_UNSUPPORTED for an op that reads its own output tensor or whose problems write two tensors.     */
int opb_test_chain_conv_run(opb_ctx* ctx, int n, int h, int w, int index, const void* in0, const void* in1,
                            void* out_io, float* out32_0, float* out32_1);

/* One crop of opb_test_keypoint_stages: canvas (bottom-top) x (right-left) at (left, top) of frame `frame`, mirrored
 * when flip = 1; canvas pixels at y >= vh or x >= vw (unmirrored) are zero (vh = h, vw = w: crop_image; smaller: the
 * zero-padded squares of opb_face_detect_frame).                                                                    */
typedef struct opb_kp_stage_crop {
  int32_t left, top, right, bottom, flip, frame, vh, vw;
} opb_kp_stage_crop;
typedef struct opb_channel_max {      /* the arg-max record of one (crop, plane)                                   */
  float value;                        /* maximum of the smoothed map                                              */
  int32_t count;                      /* pixels equal to it                                                       */
  int32_t key0, key1;                 /* row-major index of the first / second of them in the (mirrored) map; key1 = -1
                                         when count < 2                                                           */
} opb_channel_max;
/* The face / hand crop pass of opb_keypoints_detect_crops on its own, with injected network maps instead of a
 * network (no weights needed): frames [n_frames][frame_h][frame_w][3] uint8, maps [n][planes + 1][net/8][net/8]
 * float32 (channel `planes` is the background: it sits in each slot's stride and is never read).  The same crop
 * table, chunks (kp_chunk_slots, padding slots included), crop-resize, ragged upsample, two smoothing passes and
 * arg-max launches as the product.  sizes_out[3] = canvas bytes (16-slot chunks, then a power of two, each slot
 * net x net x 3), ragged map floats (sum of planes * h * w) and records (n * planes).  Outputs, each with the caller's
 * capacity (>= those sizes, else OPB_ERR_CAPACITY before anything runs): canvas_out every slot's canvas; up_out the
 * ragged upsampled maps; tmp_out after the axis-0 pass; smooth_out the smoothed maps; records_out [n][planes];
 * out / valid [n][planes][3] / [n][planes] as opb_keypoints_detect_crops.  Device buffers are filled before the
 * launches with 0x7FA5A5A5 in every 32-bit word (float maps, records) and 0xA5 in every canvas byte, and read back
 * to the full capacity.  OPB_ERR_ARG (nothing enqueued) for a bad crop row, planes outside [1, 1024], net_size not
 * a multiple of 8 in [16, 4096] or a frame index outside [0, n_frames).                                            */
int opb_test_keypoint_stages(opb_ctx* ctx, const uint8_t* frames, int n_frames, int frame_h, int frame_w,
                             const opb_kp_stage_crop* crops, int n, int net_size, int planes, const float* maps,
                             double thresh, uint8_t* canvas_out, size_t canvas_cap, float* up_out, float* tmp_out,
                             float* smooth_out, size_t map_cap, opb_channel_max* records_out, size_t records_cap,
                             double* out, int32_t* valid, int64_t* sizes_out);

#ifdef __cplusplus
}
#endif
#endif /* OPB_H_ */
