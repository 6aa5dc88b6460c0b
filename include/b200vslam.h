/*
 * b200vslam.h -- C ABI of the GPU-native (H100, sm_90a) stella_vslam hot path (ORB extract -> Hamming match -> local BA).
 *
 * The reference has no FFI of its own: its "operator API" for this path is three C++ class surfaces
 * (SURVEY.md section 8b).  Each entry point below names the reference interface it replaces (paths relative to the
 * reference checkout); the C++ adapters in stella_vslam_b200/host/ and INTEGRATION.md show the binding.
 *
 * Conventions: plain pointers and sizes only, caller-allocated outputs, int status (0 = OK, <0 = error, see
 * b200_last_error()), no exceptions cross the boundary.  One opaque handle per instance owns a CUDA stream and its
 * device arenas; handles are not thread-safe, distinct handles are independent (the reference runs the left/right
 * extractors in two threads, system.cc:427-434).  There is NO CPU fallback: every entry point fails with
 * B200_ERR_CUDA when no sm_90 (Hopper) device is usable.
 */
#ifndef B200VSLAM_H
#define B200VSLAM_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_OK 0
#define B200_ERR_INVALID (-1)  /* bad argument (also: image type/size the reference would assert on) */
#define B200_ERR_CUDA (-2)     /* CUDA runtime/driver failure or no device */
#define B200_ERR_CAPACITY (-3) /* caller buffer too small; counts are still written */
#define B200_ERR_ABORTED (-4)  /* local BA: force-stop flag was set before the first solve (no write-back) */

const char* b200_last_error(void);
int b200_device_count(void);
/* bytes of the library's version string: "b200vslam <semver> sm_90a" */
const char* b200_version(void);

/* Pinned host memory helpers (the end-to-end path copies from/to pinned buffers). */
int b200_host_alloc(void** ptr, size_t bytes);
int b200_host_free(void* ptr);

/* ------------------------------------------------------------------------------------------------------------------
 * feature::orb_extractor  (src/stella_vslam/feature/orb_extractor.h:51-61, orb_extractor.cc:16-136)
 * ---------------------------------------------------------------------------------------------------------------- */

/* cv::KeyPoint as the reference fills it (orb_extractor.cc:273-283, 337-345); class_id is always -1. */
typedef struct {
    float x, y;      /* level-0 pixel coordinates (pt * scale_factor[octave]) */
    float size;      /* (unsigned)(31 * scale_factor[octave]) */
    float angle;     /* IC angle, degrees [0,360) */
    float response;  /* FAST score */
    int32_t octave;  /* pyramid level */
} b200_keypoint_t;

/* feature::orb_params (orb_params.cc:12-27) + orb_extractor ctor arguments (orb_extractor.cc:16-20). */
typedef struct {
    float scale_factor;       /* Feature.scale_factor, default 1.2 */
    int32_t num_levels;       /* Feature.num_levels, default 8 (max 16) */
    int32_t ini_fast_thr;     /* Feature.ini_fast_threshold, default 20 */
    int32_t min_fast_thr;     /* Feature.min_fast_threshold, default 7 */
    uint32_t min_area;        /* Preprocessing.min_size (system.cc:95), default 800 */
    int32_t n_mask_rects;     /* mask_rects ctor argument: n x {x_min, x_max, y_min, y_max} as image fractions */
    const float* mask_rects;  /* may be NULL when n_mask_rects == 0 */
    int32_t device;           /* CUDA device ordinal */
    int32_t max_batch;        /* frames per extract call this instance is sized for (>=1); grows on demand */
} b200_orb_params_t;

typedef struct b200_orb_s* b200_orb_t;

void b200_orb_default_params(b200_orb_params_t* p);
int b200_orb_create(const b200_orb_params_t* p, b200_orb_t* out);
int b200_orb_destroy(b200_orb_t h);

/* Upper bound of keypoints one w x h frame can yield (sum over levels of selection-grid cells). */
int b200_orb_max_keypoints(b200_orb_t h, int width, int height);

/* orb_extractor::extract (orb_extractor.cc:28-136) for `batch` same-sized CV_8UC1 frames held in HOST memory.
 *   images      : frame f starts at images + f*frame_stride, rows `pitch` bytes apart.
 *   mask        : optional CV_8UC1 image mask at level-0 resolution shared by the batch (0 = masked), or NULL; when
 *                 NULL the rectangle mask built from mask_rects is used if any (orb_extractor.cc:50-64).
 *   kps/descs   : frame f writes kps[f*cap ..], descs[(f*cap + i)*32 ..]; counts[f] = N_f.
 * width==0 || height==0 || batch==0 -> B200_OK with nothing written (orb_extractor.cc:30-32).
 * Includes the host->device copy of the frames and the device->host copy of the results. */
int b200_orb_extract(b200_orb_t h, const uint8_t* images, int width, int height, size_t pitch, size_t frame_stride,
                     int batch, const uint8_t* mask, size_t mask_pitch, b200_keypoint_t* kps, uint8_t* descs, int cap,
                     int32_t* counts);

/* Same, with frames already resident in device memory (and the mask, if any); results stay on the device until
 * b200_orb_fetch.  Enqueued on the instance's stream (see b200_orb_set_stream) without synchronising. */
int b200_orb_extract_device(b200_orb_t h, const void* d_images, int width, int height, size_t pitch, size_t frame_stride,
                            int batch, const void* d_mask, size_t mask_pitch);
/* Run on the caller's stream (a cudaStream_t, e.g. torch's current stream; NULL is the legacy default stream).
 * use_own != 0 ignores `stream` and restores the instance's own non-blocking stream. */
int b200_orb_set_stream(b200_orb_t h, void* stream, int use_own);
/* Write results into caller-owned DEVICE buffers (e.g. torch tensors) instead of the instance's arenas:
 * keypoints [batch][stride_kps], descriptors [batch][stride_kps][32], counts [batch]; stride_kps must be >=
 * b200_orb_max_keypoints().  d_kps == NULL unbinds. */
int b200_orb_bind_outputs(b200_orb_t h, void* d_kps, void* d_descs, void* d_counts, int stride_kps);
/* Size the arenas for `batch` w x h frames now (otherwise done lazily by the first extract). */
int b200_orb_reserve(b200_orb_t h, int width, int height, int batch);
/* Copy the last extract's results to host buffers (synchronises the instance stream). */
int b200_orb_fetch(b200_orb_t h, b200_keypoint_t* kps, uint8_t* descs, int cap, int32_t* counts);
/* Device views of the last extract's results: keypoints [batch][stride_kps], descriptors [batch][stride_kps][32],
 * counts [batch].  Valid until the next extract on this handle. */
int b200_orb_device_results(b200_orb_t h, const b200_keypoint_t** d_kps, const uint8_t** d_descs, const int32_t** d_counts,
                            int* stride_kps);
int b200_orb_sync(b200_orb_t h);

/* orb_extractor::image_pyramid_ (orb_extractor.h:71; read by match::stereo via system.cc:443): level geometry and a
 * device view / host copy of one level of one frame of the last extract. */
int b200_orb_level_info(b200_orb_t h, int level, int* width, int* height, size_t* pitch, float* scale_factor);
int b200_orb_pyramid_level_device(b200_orb_t h, int frame, int level, const uint8_t** d_ptr);
int b200_orb_pyramid_level_host(b200_orb_t h, int frame, int level, uint8_t* dst, size_t dst_pitch);
/* Every level including 0 (the caller's device image, or the upload staging of b200_orb_extract), with its pitch and size. */
int b200_orb_pyramid_level_view(b200_orb_t h, int frame, int level, const uint8_t** d_ptr, size_t* pitch, int* width, int* height);

/* The per-keypoint steps between extractor and matchers (SURVEY 8f N2), for `n` keypoints in HOST buffers:
 *   camera::perspective::undistort_keypoints     (src/stella_vslam/camera/perspective.cc:245-275: cv::undistortPoints with
 *       TermCriteria(EPS | MAX_ITER, 20, 1e-6), R = I, P = K; also Perspective without distortion, e.g. KITTI)
 *   camera::equirectangular::undistort_keypoints (the identity)
 *   camera::fisheye::undistort_keypoints         (camera/fisheye.cc:281-309: cv::fisheye::undistortPoints with the default
 *       TermCriteria(MAX_ITER + EPS, 10, 1e-8), R = empty, P = K; K and D are CV_32F there, so fx fy cx cy k1..k4 are rounded to
 *       float for the undistortion only; a point that does not converge or whose angle flips sign becomes (-1e6, -1e6))
 *   camera::radial_division::undistort_point     (camera/radial_division.cc:83-98: closed form in double)
 *   camera::base::convert_keypoints_to_bearings  (camera/base.cc:158-162; perspective.cc:117-122, equirectangular.cc:42-49; fisheye and
 *       radial division use the perspective formula with the double intrinsics)
 * model: 0 perspective (k1 k2 p1 p2 k3), 1 equirectangular, 2 fisheye (k1 k2 k3 k4), 3 radial division (distortion).  Model 1 means
 * equirectangular here and in every struct that embeds this one; b200_rectifier_params_t numbers its models differently (1 = fisheye).
 * Models 2 and 3 need finite fx fy cx cy and finite coefficients of their own, else B200_ERR_INVALID.  undist_keypts (n) and bearings
 * (n x 3 doubles) may each be NULL.  response is 0 in the undistorted keypoints of models 0, 2 and 3 (the reference rebuilds them).
 * Runs on the extractor's stream (after the extract whose keypoints it is given). */
typedef struct {
    int32_t model;
    double fx, fy, cx, cy;
    double k1, k2, p1, p2, k3; /* perspective: cv_dist_params_ (k1 k2 p1 p2 k3); fisheye: k1 k2 k3 (p1 / p2 unused) */
    double cols, rows;         /* equirectangular */
    double k4;                 /* fisheye (appended: the fields above keep their offsets) */
    double distortion;         /* radial division */
} b200_camera_intrinsics_t;
int b200_keypoints_undistort(b200_orb_t h, const b200_camera_intrinsics_t* cam, const b200_keypoint_t* keypts, int n,
                             b200_keypoint_t* undist_keypts, double* bearings);

/* data::frame::can_observe (src/stella_vslam/data/frame.cc:59-84) for the `n` local landmarks a frame may see
 * (tracking_module.cc:559-594): reprojection (camera/perspective.cc:130-148, equirectangular.cc:59-73), ORB scale range
 * (data/landmark.h:88-92), viewing angle, predicted pyramid level (data/landmark.cc:336-353).  pose_cw: 4x4 row-major;
 * img_bounds = {min_x, max_x, min_y, max_y} (camera::base::img_bounds_, perspective only); per landmark: pos_w (3 doubles),
 * mean_normal (3 doubles), min / max valid distance (floats).  Out per landmark: observable (0/1) and, when observable, the
 * reprojection (2 doubles), x_right and pred_scale_level -- the inputs of b200_match_guided mode 0.  img_bounds is required for
 * models 0, 2 and 3.  The bound test is strict for perspective and fisheye (min < x < max, perspective.cc:146-147, fisheye.cc:184-186)
 * and inclusive for radial division (x < min || x > max rejects, radial_division.cc:124-130). */
int b200_frame_can_observe(b200_orb_t h, const b200_camera_intrinsics_t* cam, double focal_x_baseline, const float* img_bounds,
                           const double* pose_cw, int n, const double* pos_w, const double* mean_normal, const float* min_valid_dist,
                           const float* max_valid_dist, float ray_cos_thr, unsigned num_levels, float log_scale_factor, uint8_t* observable,
                           double* reproj, float* x_right, uint32_t* pred_scale_level);

/* util::convert_to_grayscale (src/stella_vslam/util/image_converter.cc:8-39; SURVEY 8f N4): cv::cvtColor(COLOR_{RGB,BGR}[A]2GRAY) of
 * 8-bit frames, the step in front of the extractor (system.cc:370-378).  channels: 3 or 4; rgb_order != 0 <=> color_order_t::RGB.
 * The host variant converts one frame; the device variant converts `batch` frames in place on the extractor's stream so that
 * b200_orb_extract_device can follow without a copy (source frames 16-byte aligned, pitches multiples of 4). */
int b200_convert_to_grayscale(b200_orb_t h, const uint8_t* src, int width, int height, size_t src_pitch, int channels, int rgb_order,
                              uint8_t* gray, size_t gray_pitch);
int b200_convert_to_grayscale_device(b200_orb_t h, const void* d_src, int width, int height, size_t src_pitch, size_t src_frame_stride,
                                     int channels, int rgb_order, void* d_gray, size_t gray_pitch, size_t gray_frame_stride, int batch);

/* util::stereo_rectifier (src/stella_vslam/util/stereo_rectifier.cc:12-66): the undistort-and-rectify step in front of the grayscale
 * conversion and the extractor for a stereo rig whose frames are not rectified yet (system::feed_stereo_frame requires rectified input).
 * b200_rectifier_create builds both eyes' maps once, on the host in double with the host libm, as
 *   model 0: cv::initUndistortRectifyMap(K, D, R, K_rect, size, CV_32F)           (D: 4, 5 or 8 coefficients k1 k2 p1 p2 [k3 [k4 k5 k6]])
 *   model 1: cv::fisheye::initUndistortRectifyMap(K, D, R, K_rect, size, CV_32F)  (D: 4 coefficients k1..k4; rays behind the camera map
 *            to an infinity of the sign opposite to the ray's x / y, as OpenCV 4.13 writes them)
 * and converts them once to the fixed-point form cv::remap derives from float maps (source corner + 5-bit fractions).  Every
 * rectify is then cv::remap(..., INTER_LINEAR) with BORDER_CONSTANT 0 in integer arithmetic only, bit-exact by construction.
 * Deviations: the 12- and 14-coefficient models (thin prism, tilt) and model values other than 0 / 1 are B200_ERR_INVALID (the reference
 * throws for equirectangular, stereo_rectifier.cc:52-54); cols and rows are limited to 32766 (the fixed-point corner is a short). */
typedef struct {
    int32_t model;         /* 0 perspective, 1 fisheye (StereoRectifier.model) */
    int32_t cols, rows;    /* Camera.cols / rows: source, map and output size */
    double K_rect[9];      /* camera::perspective::cv_cam_matrix_ of the rectified camera, row-major (CV_32F there: its float values) */
    double K[2][9];        /* StereoRectifier.K_left / K_right, row-major */
    double R[2][9];        /* StereoRectifier.R_left / R_right, row-major */
    double D[2][8];        /* StereoRectifier.D_left / D_right; the first n_dist[eye] entries are read */
    int32_t n_dist[2];
    int32_t device;        /* CUDA device ordinal */
} b200_rectifier_params_t;
typedef struct b200_rectifier_s* b200_rectifier_t;
int b200_rectifier_create(const b200_rectifier_params_t* p, b200_rectifier_t* out);
int b200_rectifier_destroy(b200_rectifier_t h);
/* Same contract as b200_orb_set_stream: run on the caller's stream (NULL = legacy default), use_own != 0 restores the own stream. */
int b200_rectifier_set_stream(b200_rectifier_t h, void* stream, int use_own);
/* The CV_32F maps as built (the reference's undist_map_{x,y}_{l,r}_): eye 0 left, 1 right; rows x cols floats each, tightly packed. */
int b200_rectifier_maps(b200_rectifier_t h, int eye, float* map_x, float* map_y);
/* stereo_rectifier::rectify for one pair of 8-bit frames with `channels` (1, 3 or 4) interleaved channels in HOST memory, rows `*_pitch`
 * bytes apart (pitch >= cols * channels).  Includes the uploads and downloads; returns when the outputs are written. */
int b200_stereo_rectify(b200_rectifier_t h, int channels, const uint8_t* left, size_t left_pitch, const uint8_t* right, size_t right_pitch,
                        uint8_t* out_left, size_t out_left_pitch, uint8_t* out_right, size_t out_right_pitch);
/* Same for `batch` pairs in DEVICE memory, enqueued on the rectifier's stream without synchronising: pair f reads d_left / d_right +
 * f * src_frame_stride and writes d_out_left / d_out_right + f * out_frame_stride.  Interleaving the eyes (d_out_right = d_out_left +
 * one frame, out_frame_stride = two frames) lets ONE b200_orb_extract_device over 2 * batch frames follow on the same stream and feed
 * b200_stereo_compute(h, 2p, h, 2p + 1).  Outputs must not overlap inputs.  Word-wide stores when the output pointers, pitch and frame
 * stride are multiples of 4 bytes, byte stores otherwise.  batch == 0 -> B200_OK with nothing written. */
int b200_stereo_rectify_device(b200_rectifier_t h, int channels, const void* d_left, const void* d_right, size_t src_pitch, size_t src_frame_stride,
                               void* d_out_left, void* d_out_right, size_t out_pitch, size_t out_frame_stride, int batch);

/* Keyframe serialisation (SURVEY 8f N4): the byte layouts in which data::keyframe stores what the extractor produced.
 *   SQLite (data/keyframe.cc:298-347 to_db, :191-235 from_stmt): `undist_keypts` = the std::vector<cv::KeyPoint> as raw bytes (28 bytes per
 *       keypoint: pt.x, pt.y, size, angle, response, octave, class_id), `descs` = cv::Mat rows, 32 bytes each;
 *   JSON / msgpack (data/common.cc:57-81): a descriptor = eight uint32 read through `desc.ptr<uint32_t>()` -- on a little-endian host the
 *       same 32 bytes, so `desc_blob` viewed as uint32[n][8] is convert_descriptors_to_json's payload.
 * Exports frame `frame` of the last extract straight from HBM: the keypoints are undistorted on the device when `cam` is given
 * (camera::*::undistort_keypoints -- the keyframe stores undist_keypts_), re-packed to cv::KeyPoint records (class_id = -1, response = 0
 * for perspective, fisheye and radial-division cameras as perspective.cc:266-272 / fisheye.cc:300-306 / base.cc:124-150 leave it) and
 * copied out with the descriptors.  *n = keypoints of the frame;
 * B200_ERR_CAPACITY if cap is too small. */
typedef struct {
    float x, y, size, angle, response;
    int32_t octave, class_id;
} b200_cv_keypoint_t;
int b200_orb_export_keyframe_blobs(b200_orb_t h, int frame, const b200_camera_intrinsics_t* cam, b200_cv_keypoint_t* keypts_blob,
                                   uint8_t* desc_blob, int cap, int32_t* n);
/* RGB-D frames: system::create_RGBD_frame after the extraction (src/stella_vslam/system.cc:467-530) for the first n_frames frames of the
 * last extract on `h`, whose keypoints are read where they lie in HBM.  The depth maps are HOST buffers (frame f at depth_maps +
 * f * frame_stride, rows `pitch` bytes apart) of type B200_DEPTH_16UC1 (TUM RGB-D) or B200_DEPTH_32FC1, the cv::Mat::type() codes, and
 * exactly the extracted frames' size.  One upload, one launch and one download on the extractor's stream.  Per keypoint:
 *   undist_keypts / bearings : camera::*::undistort_keypoints + convert_keypoints_to_bearings, the device functions of
 *                              b200_keypoints_undistort (bit-identical to it)
 *   depth                    : img_depth.at<float>(y, x) at the DISTORTED keypoint with x, y truncated to int (system.cc:499-503), after
 *                              util::convert_to_true_depth (util/image_converter.cc:41-43) = convertTo(CV_32F, 1.0 / depthmap_factor),
 *                              which OpenCV evaluates as (float)v * (float)(1.0 / depthmap_factor) (a plain copy for 32FC1 with factor 1);
 *                              only the sampled pixels are converted
 *   depths / x_right         : -1 / -1 unless 0 < depth (system.cc:505-507; a NaN is invalid here, the reference's `depth <= 0` lets it
 *                              through), else depth / (float)(undist_x - focal_x_baseline / depth) in double (system.cc:509-510)
 * Frame f writes entries f * cap ..; n_keypoints[f] = its keypoint count.  B200_ERR_CAPACITY when a frame has more than cap keypoints (its
 * first cap are written).  B200_ERR_INVALID: another depth type, a depth map whose size differs from the extracted frames (the reference
 * only warns, system.cc:469-474, and then reads out of bounds), model 1 (equirectangular: data/common.cc:236-238 throws for RGB-D), a
 * depthmap_factor that is not positive and finite, n_frames beyond the last extract. */
#define B200_DEPTH_16UC1 2
#define B200_DEPTH_32FC1 5
int b200_rgbd_depths(b200_orb_t h, int n_frames, const b200_camera_intrinsics_t* cam, double focal_x_baseline, double depthmap_factor, int depth_type,
                     const void* depth_maps, int width, int height, size_t pitch, size_t frame_stride, int cap, b200_keypoint_t* undist_keypts,
                     double* bearings, float* depths, float* x_right, int32_t* n_keypoints);
/* The inverse for a keyframe loaded from a map file (host-only byte shuffling, no GPU work): cv::KeyPoint records -> b200_keypoint_t. */
int b200_keyframe_blob_to_keypoints(const b200_cv_keypoint_t* keypts_blob, int n, b200_keypoint_t* keypts);

/* Raw FAST corners (after NMS, threshold choice and mask tests, before distribute_keypoints) of the first n frames of the last extract:
 * the candidate count of orb_extractor.cc:237-259, which prices the FAST and selection kernels (SURVEY 8d).  Synchronises. */
int b200_orb_raw_corner_counts(b200_orb_t h, int32_t* counts, int n);
/* Per-stage kernel time of the last extract, in ms, measured with CUDA events on the instance stream.
 * stage: 0 pyramid, 1 FAST+NMS+grid arg-max, 2 ordered selection, 3 (unused: the descriptor blur is fused into stage 4),
 * 4 window blur + orientation + rBRIEF, 5 whole extract. */
int b200_orb_stage_ms(b200_orb_t h, int stage, float* ms);
int b200_orb_enable_timing(b200_orb_t h, int enable);

/* ------------------------------------------------------------------------------------------------------------------
 * match::compute_descriptor_distance_32 / match::robust::brute_force_match
 * (src/stella_vslam/match/base.h:15-41, match/robust.cc:232-328)
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct b200_matcher_s* b200_matcher_t;

int b200_matcher_create(int device, b200_matcher_t* out);
int b200_matcher_destroy(b200_matcher_t h);

/* All-pairs 256-bit Hamming distances: dist[i*n2 + j] = popcount(desc1[i] ^ desc2[j])  (host buffers). */
int b200_hamming_matrix(b200_matcher_t h, const uint8_t* desc1, int n1, const uint8_t* desc2, int n2, uint16_t* dist);

/* robust::brute_force_match for `n_problems` independent (frame, keyframe) pairs.  Problem p reads
 *   frame side    (frm_obs):  descriptors desc1 + 32*(off1[p]+i), angle *(float*)((char*)angle1 + (off1[p]+i)*angle1_stride),
 *                             i < cnt1[p]   (angle1_stride = 4 for a float array, sizeof(b200_keypoint_t) for &kps[0].angle)
 *   keyframe side (keyfrm) :  likewise with off2/cnt2; valid2[off2[p]+i] != 0 <=> keypoint i has a live landmark
 *                             (robust.cc:255-262); valid2 == NULL means all valid.
 * and writes (idx_1, idx_2) int32 pairs sorted by idx_1 at pairs + 2*p*pairs_stride, and n_pairs[p].
 * pairs_stride >= max_p cnt1[p].  lowe_ratio / check_orientation: the matcher's ctor arguments (match/base.h:81-91).
 * Host buffers; includes the uploads and the download of the results. */
int b200_match_bruteforce(b200_matcher_t h, int n_problems, const uint8_t* desc1, const void* angle1, size_t angle1_stride,
                          const int32_t* off1, const int32_t* cnt1, const uint8_t* desc2, const void* angle2, size_t angle2_stride,
                          const uint8_t* valid2, const int32_t* off2, const int32_t* cnt2, float lowe_ratio, int check_orientation,
                          int32_t* pairs, int pairs_stride, int32_t* n_pairs);
/* Device-resident variant: every pointer is a device pointer and the work is enqueued on the matcher's stream
 * (see b200_matcher_set_stream) without synchronising.  Problem p reads
 *   frame side    : descriptors d_desc1 + 32*(off1[p]+i), angle *(float*)((char*)d_angle1 + (off1[p]+i)*angle1_stride), i < cnt1[p]
 *   keyframe side : likewise with off2/cnt2 (cnt arrays live on the device, e.g. the extractor's d_counts)
 * and writes its pairs at d_pairs + 2*p*pairs_stride and its count at d_n_pairs[p].  max_n1/max_n2 bound cnt1/cnt2 (host-side
 * upper bounds used to size the launch); pairs_stride >= max_n1. */
int b200_match_bruteforce_device(b200_matcher_t h, int n_problems, const void* d_desc1, const void* d_angle1, size_t angle1_stride,
                                 const void* d_off1, const void* d_cnt1, const void* d_desc2, const void* d_angle2,
                                 size_t angle2_stride, const void* d_valid2, const void* d_off2, const void* d_cnt2, int max_n1,
                                 int max_n2, float lowe_ratio, int check_orientation, void* d_pairs, int pairs_stride,
                                 void* d_n_pairs);
/* Optional: run the sequential resolve pass of b200_match_bruteforce_device on a side stream.  The pass is the reference's greedy loop
 * (robust.cc:253-315) -- one warp per problem, so most SMs sit idle while it runs -- so when it is enabled
 * the caller's NEXT kernels on the matcher's stream (e.g. the next batch's extraction) overlap it.  Contract while enabled: d_pairs /
 * d_n_pairs of a call, and the freedom to overwrite that call's input buffers, are reached on the matcher's stream only after the next
 * b200_match_bruteforce_device call on this handle, b200_matcher_join (stream-ordered: the stream waits, the host does not) or
 * b200_matcher_sync.  Off by default. */
int b200_matcher_set_async_resolve(b200_matcher_t h, int enable);
int b200_matcher_join(b200_matcher_t h);
/* Grid-guided projection matchers
 *   mode 0 (B200_GUIDED_LANDMARKS): match::projection::match_frame_and_landmarks     (src/stella_vslam/match/projection.cc:13-93)
 *   mode 1 (B200_GUIDED_LAST_FRAME): match::projection::match_current_and_last_frames (src/stella_vslam/match/projection.cc:95-207)
 * and, on the same search primitive, the occasional (relocalisation / loop closure / mapping / initialisation) variants:
 *   mode 1 with thr = hamm_dist_thr, t_x_right = NULL:        projection::match_frame_and_keyframe  (projection.cc:217-319)
 *   mode 1 with thr = 50, check_orientation = 0:              projection::match_by_Sim3_transform   (projection.cc:321-416)
 *   mode 2 (B200_GUIDED_INDEPENDENT) once per direction, then b200_match_cross_check:
 *                                                             projection::match_keyframes_mutually  (projection.cc:418-630)
 *   mode 3 (B200_GUIDED_FUSE) with thr = 50:                  fuse::detect_duplication              (match/fuse.cc:12-154)
 *   mode 4 (B200_GUIDED_AREA) with thr = 50, lowe_ratio:      area::match_in_consistent_area        (match/area.cc:8-98); a later
 *        query may take a keypoint over from an earlier one (its match_out entry goes back to -1, area.cc:75-81)
 * including the keypoint grid they search: data::assign_keypoints_to_grid / get_keypoints_in_cell
 * (src/stella_vslam/data/common.cc:83-190).  The caller (the adapter) does what needs the map: it walks the landmarks in the
 * reference's order, reprojects them (camera::base::reproject_to_image), predicts the pyramid level and fills one query per
 * landmark; q_valid[q] == 0 marks a landmark the reference skips before the search (will_be_erased, !is_observable_in_tracking,
 * reprojection failed / outside the image, last-frame outlier).  All pointers are HOST buffers.
 * Result: match_out[q] = index of the frame keypoint landmark q is attached to (frm.add_landmark(lm, idx)) or -1, n_matches;
 * t_occupied is updated in place in modes 0, 1 and 3 (a keypoint that received a landmark is not offered to later landmarks,
 * projection.cc:50-53, 163-166, 292-294, 388-390; fuse.cc:88-90); mode 2 reads it only, mode 4 ignores it.  `n_problems` independent frames are processed in one launch sequence. */
enum { B200_GUIDED_LANDMARKS = 0, B200_GUIDED_LAST_FRAME = 1, B200_GUIDED_INDEPENDENT = 2, B200_GUIDED_FUSE = 3, B200_GUIDED_AREA = 4 };
typedef struct b200_guided_problem {
    int32_t n_train;                  /* keypoints of the frame that is searched */
    const float* t_x;                 /* frm_obs_.undist_keypts_[i].pt.x */
    const float* t_y;
    const uint8_t* t_octave;
    const float* t_angle;             /* needed when mode 1 checks orientation, else may be NULL */
    const float* t_x_right;           /* frm_obs_.stereo_x_right_, NULL when empty (monocular) */
    const uint8_t* t_desc;            /* n_train x 32 */
    uint8_t* t_occupied;              /* in/out, n_train: keypoint already carries a landmark with observations; NULL = none (no write-back) */
    float min_x, max_x, min_y, max_y; /* camera::base::img_bounds_ */
    int32_t grid_cols, grid_rows;     /* camera::base::num_grid_cols_ / num_grid_rows_ (64 x 48) */
    int32_t n_queries;                /* landmarks in the reference's iteration order */
    const uint8_t* q_desc;            /* n_queries x 32 (landmark::get_descriptor) */
    const float* q_x;                 /* reprojection */
    const float* q_y;
    const float* q_margin;            /* margin * scale_factors_[level], evaluated in float like the reference */
    const int8_t* q_min_level;        /* octave window; < 0 = unchecked (data/common.cc:160-173) */
    const int8_t* q_max_level;
    const float* q_x_right;           /* reprojected x_right; read only when t_x_right != NULL */
    const float* q_angle;             /* last-frame keypoint angle; read only in mode 1 with check_orientation */
    const uint8_t* q_valid;           /* NULL = all valid */
    const uint8_t* q_has_observation; /* modes 0 / 1: landmark::has_observation() of the query landmark; NULL = all have.  A keypoint that
                                         receives a landmark WITHOUT observations (a temporal landmark of a stereo / RGBD last frame) stays
                                         open to later landmarks, exactly like the reference's test `lm && lm->has_observation()`
                                         (projection.cc:50-53, 163-166); match_out then lists the keypoint for both and the adapter's
                                         in-order add_landmark leaves the later one, as in the reference */
    const double* q_reproj;           /* mode 3 with do_reprojection_matching: n_queries x 2, the reprojection in double (fuse.cc:96-97) */
    const float* inv_level_sigma_sq;  /* mode 3: orb_params_->inv_level_sigma_sq_, n_levels entries */
    int32_t n_levels;
    int32_t do_reprojection_matching; /* mode 3 (fuse.cc:19, :93) */
    int32_t* match_out;               /* out, n_queries */
    int32_t n_matches;                /* out */
} b200_guided_problem_t;
/* thr: the reference's `best <= thr` acceptance (100 for modes 0-2 in the callers cited, 50 for 3-4); lowe_ratio: modes 0 and 4; max_candidates bounds the
 * keypoints one search window may return (0 = default 256); B200_ERR_CAPACITY reports the size that would have been needed. */
int b200_match_guided(b200_matcher_t h, int n_problems, b200_guided_problem_t* problems, int mode, unsigned thr, float lowe_ratio,
                      int check_orientation, int max_candidates);
/* Closing loop of match_keyframes_mutually (projection.cc:614-627) on two mode-2 results: mutual_out[i] = j iff idx2_in_1[i] == j
 * and idx1_in_2[j] == i, else -1.  Host-side, no device work. */
int b200_match_cross_check(const int32_t* idx2_in_1, int n1, const int32_t* idx1_in_2, int n2, int32_t* mutual_out, int32_t* n_mutual);
/* All-pairs matchers with greedy state, other than brute_force_match:
 *   variant 0 (B200_PAIRS_BOW):           match::bow_tree::match_frame_and_keyframe  (src/stella_vslam/match/bow_tree.cc:169-256)
 *                                         match::bow_tree::match_keyframes           (bow_tree.cc:258-366)
 *   variant 1 (B200_PAIRS_TRIANGULATION): match::robust::match_for_triangulation     (src/stella_vslam/match/robust.cc:14-146)
 *                                         match::bow_tree::match_for_triangulation   (bow_tree.cc:11-167)
 *                                         with match::check_epipolar_constraint      (match/base.h:67-79)
 * Side 1 are the rows the reference's outer loop walks (keyframe / keyframe 1), side 2 the candidates (frame / keyframe 2).
 * node1/node2: the BoW node each keypoint belongs to (the key of bow_feat_vec_ that lists it); a row only sees candidates of its
 * own node.  NULL on both sides = every row sees every candidate (robust::).  valid1/valid2 carry the landmark tests of the
 * variant (BOW: row has a live landmark, bow_tree.cc:192-199 / 284-291, candidate likewise for match_keyframes :303-309;
 * TRIANGULATION: neither has a landmark, robust.cc:44-48, 66-69).  All pointers are HOST buffers.
 * Result: match_out[i] = index on side 2 matched to row i, or -1; n_matches. */
enum { B200_PAIRS_BOW = 0, B200_PAIRS_TRIANGULATION = 1 };
typedef struct b200_pairs_problem {
    int32_t n1;
    const uint8_t* desc1;        /* n1 x 32 */
    const float* angle1;         /* needed when check_orientation */
    const uint8_t* valid1;       /* NULL = all */
    const int32_t* node1;        /* NULL = no BoW gating (then node2 must be NULL too) */
    const double* bearing1;      /* TRIANGULATION: n1 x 3 (frm_obs_.bearings_) */
    const float* scale1;         /* TRIANGULATION: orb_params_->scale_factors_[octave] per row */
    const uint8_t* stereo1;      /* TRIANGULATION: stereo_x_right_[i] >= 0; NULL = monocular */
    int32_t n2;
    const uint8_t* desc2;
    const float* angle2;
    const uint8_t* valid2;
    const int32_t* node2;
    const double* bearing2;
    const uint8_t* stereo2;
    double E_12[9];              /* TRIANGULATION: essential matrix, row-major */
    double epiplane_in_keyfrm_2[3]; /* camera centre of keyframe 1 as a bearing in keyframe 2 (robust.cc:22-27) */
    int32_t valid_epiplane;
    float residual_rad_thr;
    int32_t* match_out;          /* out, n1 */
    int32_t n_matches;           /* out */
} b200_pairs_problem_t;
/* max_candidates bounds the gated candidates kept per row (0 = default 64); B200_ERR_CAPACITY reports the size needed. */
int b200_match_pairs(b200_matcher_t h, int n_problems, b200_pairs_problem_t* problems, int variant, float lowe_ratio,
                     int check_orientation, int max_candidates);
/* match::stereo::compute (src/stella_vslam/match/stereo.cc:20-114, helpers :116-251; constructed at system.cc:443 from the two
 * extractors' image_pyramid_).  `left` / `right` are the extractor handles whose last extract produced the two rectified frames
 * (frame index inside that extract's batch; both eyes may also be frames 0 and 1 of ONE handle): their pyramids are read where
 * they already live on the device.  Keypoints / descriptors are HOST buffers (the caller may have filtered them).
 * scale_factors_ / inv_scale_factors_ are the extractor's own (orb_params.cc:37-48).
 * Out: stereo_x_right[i], depths[i] (-1 = no stereo match), n_matched = keypoints that keep one. */
int b200_stereo_compute(b200_matcher_t h, b200_orb_t left, int frame_left, b200_orb_t right, int frame_right,
                        const b200_keypoint_t* keypts_left, const uint8_t* descs_left, int n_left, const b200_keypoint_t* keypts_right,
                        const uint8_t* descs_right, int n_right, float focal_x_baseline, float true_baseline, float* stereo_x_right,
                        float* depths, int32_t* n_matched);
/* data::landmark::compute_descriptor (src/stella_vslam/data/landmark.cc:199-256; SURVEY 8f N3), for `n_landmarks` landmarks at once
 * (after local BA / fusion every touched landmark is refreshed, local_bundle_adjuster_g2o.cc:387-390, 408).  Landmark l owns the
 * descriptors descs[32 * offsets[l] .. 32 * offsets[l+1]) -- the rows of its observing keyframes that are not about to be erased, in
 * observation order.  best_idx[l] = index (within the landmark) of the descriptor with the smallest median Hamming distance to all of
 * them, first on ties (-1 for a landmark without descriptors); desc_out (optional, n_landmarks x 32) = that descriptor. */
int b200_landmark_descriptors(b200_matcher_t h, int n_landmarks, const uint8_t* descs, const int32_t* offsets, int32_t* best_idx,
                              uint8_t* desc_out);
/* data::landmark::update_mean_normal_and_obs_scale_variance (src/stella_vslam/data/landmark.cc:256-311; SURVEY 8f N3) for
 * `n_landmarks` landmarks.  Landmark l: position pos_w[3l..], observed from the camera centres
 * cam_centers[3 * offsets[l] .. 3 * offsets[l+1]) (keyfrm->get_trans_wc() of its observations in the order the caller walks them);
 * ref_center[3l..] / ref_scale_factor[l] = centre of its reference keyframe and scale_factors_[octave of its keypoint there];
 * inv_scale_factor_last = inv_scale_factors_[num_levels - 1].  Out: mean_normal (n x 3), max_valid_dist, min_valid_dist. */
int b200_landmark_geometry(b200_matcher_t h, int n_landmarks, const double* pos_w, const int32_t* offsets, const double* cam_centers,
                           const double* ref_center, const float* ref_scale_factor, float inv_scale_factor_last, double* mean_normal,
                           float* max_valid_dist, float* min_valid_dist);
/* Device time (ms, CUDA events) of the two passes of the last b200_match_bruteforce[_device] call while timing is enabled:
 * stage 0 = all-pairs distances + per-row top-K lists, stage 1 = sequential resolve.  Synchronises the streams involved. */
int b200_matcher_enable_timing(b200_matcher_t h, int enable);
int b200_matcher_stage_ms(b200_matcher_t h, int stage, float* ms);
/* Run on the caller's stream (a cudaStream_t; NULL is the legacy default stream); use_own != 0 restores the own stream. */
int b200_matcher_set_stream(b200_matcher_t h, void* stream, int use_own);
int b200_matcher_sync(b200_matcher_t h);

/* ------------------------------------------------------------------------------------------------------------------
 * optimize::local_bundle_adjuster  (src/stella_vslam/optimize/local_bundle_adjuster.h:15-24,
 * optimize/local_bundle_adjuster_g2o.cc:36-431).  The host adapter does the pointer-chasing gather (steps 1-4,
 * :41-304) and the write-back under the map mutex (step 8, :379-430); this entry point is steps 5-7: two rounds of
 * Levenberg-Marquardt with Schur complement over the landmarks (g2o BlockSolver_6_3 semantics), outlier marking in
 * between, on a flattened problem.  All arithmetic is fp64.
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct {
    int32_t model;          /* 0: perspective-family edge (Perspective / Fisheye / RadialDivision all use the perspective edges on
                               undistorted keypoints, reproj_edge_wrapper.h:64-188); 1: equirectangular (:129-146) */
    double fx, fy, cx, cy;  /* perspective_reproj_edge.h:34 */
    double fxb;             /* focal_x_baseline_ (stereo rows, perspective_reproj_edge.h:148) */
    double cols, rows;      /* equirectangular_reproj_edge.h */
} b200_camera_t;

typedef struct {
    int32_t n_poses, n_points, n_edges, n_cams;
    const double* pose_cw;           /* K x 16 row-major 4x4: keyfrm->get_pose_cw() (shot_vertex_container.h:103-117) */
    const uint8_t* pose_fixed;       /* K: 1 = fixed keyframe (local_bundle_adjuster_g2o.cc:184-190) */
    const double* points;            /* L x 3: lm->get_pos_in_world() */
    const uint8_t* point_fixed;      /* L or NULL: marker corners of keep_fixed_ markers (:272) */
    const int32_t* e_pose;           /* E: keyframe index of the observation */
    const int32_t* e_point;          /* E: landmark index */
    const uint8_t* e_cam;            /* E: index into cams */
    const float* e_obs;              /* E x 3: undist_keypt.pt.x, .y, stereo_x_right (< 0 => monocular edge, reproj_edge_wrapper.h:62) */
    const float* e_inv_sigma_sq;     /* E: inv_level_sigma_sq_[octave] (:238) */
    const float* e_delta;            /* E: Huber delta = sqrt(chi-square) as float (:205-208, 239-241) */
    const uint8_t* e_robust;         /* E or NULL (=1): Huber kernel in the first round (use_huber_loss, :297-299) */
    const uint8_t* e_can_be_outlier; /* E or NULL (=1): 0 for marker-corner edges, which are never outlier-tested (:251-304) */
    const b200_camera_t* cams;
} b200_lba_problem_t;

typedef struct {
    int32_t iterations[2];   /* LM iterations run in the robust / non-robust round */
    int32_t n_outliers;
    double chi2[2];          /* active robust chi-square after each round */
    double lambda_init;
    double lambda_final[2];
} b200_lba_stats_t;

typedef struct b200_lba_s* b200_lba_t;

int b200_lba_create(int device, b200_lba_t* out);
int b200_lba_destroy(b200_lba_t h);
/* local_bundle_adjuster_g2o::optimize steps 5-7.  iters1/iters2: num_first_iter_/num_second_iter_ (5 / 10,
 * local_bundle_adjuster_g2o.h:25-27).  force_stop: the caller's abort flag (mapping_module.cc:124,199-206), polled
 * between LM iterations; may be NULL.  As in the reference it is also WRITTEN: the gain-threshold terminate action
 * sets it when it stops a round (terminate_action.cc:55-72 via g2o's setOptimizerStopFlag), which is what makes the
 * reference skip the second round after an early first-round stop (:317-321).
 * Returns B200_ERR_ABORTED (nothing written) when *force_stop is already set on entry (:308-310).
 * With force_stop == NULL the gain stop of the first round lands in g2o's own auxiliary flag, which the second optimize() resets:
 * the second round always runs.  Deviation: the reference's terminate_action also CLEARS the caller's flag at iteration -1 of each
 * optimize() (terminate_action.cc:46-51), so an abort raised in the few microseconds between the entry test and the first iteration
 * is lost there; here an externally raised flag is never cleared, it stops the solve at the next iteration boundary.
 * At most 166 FREE keyframes (B200_ERR_INVALID beyond; fixed keyframes are not limited).
 * pose_cw_out: K x 16, points_out: L x 3, outlier_out: E (1 = observation to erase, :354-375).  Same code path as the batch of one. */
int b200_lba_solve(b200_lba_t h, const b200_lba_problem_t* problem, int iters1, int iters2, volatile uint8_t* force_stop,
                   double* pose_cw_out, double* points_out, uint8_t* outlier_out, b200_lba_stats_t* stats);
/* Many independent windows in ONE launch sequence (SURVEY 8d: the batched form is what makes local BA GPU-shaped).  The reference
 * runs one optimize() per new keyframe on the mapping thread (mapping_module.cc:199-206); an integrator with several maps / streams
 * (BASELINE config 5) or a backlog of keyframes hands all pending windows to one call.  The windows advance in lockstep, every
 * kernel serves all of them (window = blockIdx.y, one thread-block cluster per window for the reduced-system Cholesky), the
 * Levenberg-Marquardt decisions are taken on the device per window, and the plan (edges sorted by landmark, per-keyframe edge lists)
 * is built on the device: the host copies the caller's arrays and enqueues.
 *   force_stop[w]  : per-window abort flag as in b200_lba_solve (array may be NULL, entries may be NULL)
 *   pose_cw_out[w] / points_out[w] / outlier_out[w] : per-window outputs (outlier_out or its entries may be NULL)
 *   stats          : n_windows entries or NULL
 *   status[w]      : B200_OK, B200_ERR_ABORTED (flag already set on entry: nothing written for that window) or B200_ERR_INVALID
 * Limits: at most 166 FREE keyframes per window (the reduced system is factored on chip); fixed keyframes, landmarks and
 * observations are limited by memory only.  Returns B200_OK if every window that ran is valid. */
int b200_lba_solve_batch(b200_lba_t h, int n_windows, const b200_lba_problem_t* problems, int iters1, int iters2,
                         volatile uint8_t* const* force_stop, double* const* pose_cw_out, double* const* points_out,
                         uint8_t* const* outlier_out, b200_lba_stats_t* stats, int32_t* status);
/* optimize::global_bundle_adjuster (src/stella_vslam/optimize/global_bundle_adjuster.cc: optimize_impl :26-192, optimize :258-420,
 * optimize_for_initialization :201-256; called by module/loop_bundle_adjuster.cc:54 and module/initializer.cc:281): the same flattened
 * problem and kernels as the local bundle adjuster, ONE Levenberg-Marquardt round of `num_iter` iterations (global_bundle_adjuster.h:20-23:
 * 10) with the terminate action at `gain_threshold` (1e-3 in optimize(), the caller's value in optimize_for_initialization), no outlier
 * pass.  Every keyframe of the map is free except the spanning root (:80-81), so the reduced system has 6 x (keyframes - 1) unknowns: up
 * to 1000 it is factored on chip like a local window; beyond that (limit 4000 free keyframes) the dense Cholesky runs panel by panel over
 * the whole GPU from HBM -- two launches per 24 columns -- where the reference uses g2o's CSparse solver (:42-45).
 * use_huber_kernel is the per-edge e_robust array (NULL = Huber on every edge); marker corners as in b200_lba_problem_t.
 * Returns B200_ERR_ABORTED when the CALLER raised *force_stop (the reference returns false then, :340-342, and uses no result: the
 * output buffers are unspecified); a stop
 * by the gain threshold also sets the flag (terminate_action.cc:66-70) but is a normal return. */
int b200_global_ba_solve(b200_lba_t h, const b200_lba_problem_t* problem, int num_iter, double gain_threshold, volatile uint8_t* force_stop,
                         double* pose_cw_out, double* points_out, b200_lba_stats_t* stats);
/* optimize::pose_optimizer::optimize  (src/stella_vslam/optimize/pose_optimizer.h:24-40, pose_optimizer_g2o.cc:38-175; factory
 * defaults num_trials_robust = 2, num_trials = 2, num_each_iter = 10, pose_optimizer_factory.h:18-47): motion-only bundle adjustment
 * of `n_problems` frames in one launch.  Each problem uses the b200_lba_problem_t layout with exactly ONE pose (free), the landmarks
 * the frame observes (all fixed) and one edge per observation (e_pose = 0; e_obs = undistorted x, y, x_right (< 0: monocular edge);
 * e_inv_sigma_sq = inv_level_sigma_sq_[octave]; e_delta = sqrt(chi-square), :84-88); one camera per problem: every edge must name
 * the same camera (e_cam uniform, any index below n_cams; NULL = camera 0), as the reference optimises one frame of one camera
 * (:38-43).  A problem whose edges name different cameras is refused with B200_ERR_INVALID and nothing is written.
 * Out: pose_cw_out [n_problems][16] row-major (the input pose when a frame has fewer than 5 observations, :116-118),
 * outlier_flags = the problems' edges concatenated (outlier_flags.at(idx), :141-160), n_valid[p] = num_init_obs - num_bad_obs. */
int b200_pose_optimize(b200_lba_t h, int n_problems, const b200_lba_problem_t* problems, int num_trials_robust, int num_trials,
                       int num_each_iter, double* pose_cw_out, uint8_t* outlier_flags, uint32_t* n_valid);

/* ------------------------------------------------------------------------------------------------------------------
 * Device-resident tracking chain: the per-frame steady state of tracking_module::track_local_map for `n_frames` independent
 * frames (one per camera / session / replayed log) in ONE launch sequence, reading the extractor's results where they lie
 * in HBM -- nothing of the frame goes back to the host between the stages:
 *   camera::*::undistort_keypoints            camera/perspective.cc:245-275 (frame construction, system.cc:386-395)
 *   tracking_module::search_local_landmarks   tracking_module.cc:533-606: data::frame::can_observe (data/frame.cc:59-84) over the local
 *                                             landmarks, then projection::match_frame_and_landmarks (match/projection.cc:13-93) with
 *                                             lowe_ratio 0.8 and the margin the caller chose (:599-603), HAMMING_DIST_THR_HIGH
 *   pose_optimizer::optimize                  optimize/pose_optimizer_g2o.cc:38-175 on the landmarks the frame now carries
 *                                             (tracking_module::optimize_current_frame_with_local_map)
 * Frame f is frame `frames[f].frame` of the LAST extract on `orb` (host- or device-image variant).  The landmark table of a frame
 * lists, in the reference's iteration order, every landmark the stage touches: the local landmarks AND the landmarks the frame
 * already carries (those with lm_skip = 1: tracking_module.cc:536-551 puts them into curr_landmark_ids and :561-563 skips them).
 * All pointers are HOST buffers; they go up in one copy and the results come back in one copy.  The three handles' arenas are used
 * and everything is enqueued on the extractor's stream; the call returns when the results are in the caller's buffers.
 * Bit-exact against the stage-by-stage host ABI (b200_keypoints_undistort, b200_frame_can_observe, b200_match_guided mode 0) and
 * within 1e-5 for the pose (b200_pose_optimize): same kernels / same device functions. */
typedef struct b200_track_params {
    b200_camera_intrinsics_t cam;
    double focal_x_baseline;       /* camera::base::focal_x_baseline_ (0 for monocular) */
    int32_t monocular;             /* setup_type_ == Monocular: edge threshold sqrt(chi2_2D), else sqrt(chi2_3D) (pose_optimizer_g2o.cc:84-88) */
    float img_bounds[4];           /* min_x, max_x, min_y, max_y */
    int32_t grid_cols, grid_rows;  /* 64 x 48 */
    uint32_t num_levels;
    float log_scale_factor;
    const float* scale_factors;        /* num_levels */
    const float* inv_level_sigma_sq;   /* num_levels */
    float margin;                  /* margin_local_map_projection_(_unstable_) */
    float lowe_ratio;              /* 0.8 (tracking_module.cc:599) */
    uint32_t hamming_thr;          /* HAMMING_DIST_THR_HIGH = 100 */
    float ray_cos_thr;             /* 0.5 (tracking_module.cc:588) */
    int32_t num_trials_robust, num_trials, num_each_iter; /* 2 / 2 / 10 */
    int32_t max_candidates;        /* 0 = 256 keypoints per search window */
} b200_track_params_t;
typedef struct b200_track_frame {
    int32_t frame;                     /* index into the extractor's last batch */
    const double* pose_cw;             /* 16, row-major: curr_frm_.pose_cw_ entering the stage */
    int32_t n_keypoints_in;            /* entries of kp_x_right / kp_landmark (0 when both are NULL); must equal the frame's keypoint count */
    const float* kp_x_right;           /* frm_obs_.stereo_x_right_, NULL when empty */
    const int32_t* kp_landmark;        /* per keypoint: row of the landmark it already carries (not will_be_erased), -1 none; NULL = none */
    int32_t n_landmarks;
    const double* lm_pos_w;            /* 3 per landmark */
    const double* lm_mean_normal;      /* 3 per landmark */
    const float* lm_min_valid_dist;
    const float* lm_max_valid_dist;
    const uint8_t* lm_desc;            /* 32 per landmark */
    const uint8_t* lm_skip;            /* 1 = not searched (already in the frame, will_be_erased, temporal-ratio test :565-585); NULL = none */
    const uint8_t* lm_has_observation; /* landmark::has_observation(); NULL = all have */
    int32_t kp_cap;                    /* capacity of kp_landmark_out / kp_outlier (>= the frame's keypoint count) */
    uint8_t* lm_observable;            /* out, n_landmarks: searched and can_observe() held (the caller's increase_num_observable, :594) */
    int32_t* kp_landmark_out;          /* out, per keypoint: landmark row after the search (frm.add_landmark applied in order), -1 none */
    uint8_t* kp_outlier;               /* out, per keypoint: outlier_flags of the pose optimisation */
    double pose_cw_out[16];            /* out (the input pose when fewer than 5 observations, :116-118) */
    int32_t n_keypoints;               /* out */
    int32_t n_matches;                 /* out: return value of match_frame_and_landmarks */
    uint32_t n_valid;                  /* out: return value of pose_optimizer::optimize */
} b200_track_frame_t;
int b200_track_local_map(b200_orb_t orb, b200_matcher_t matcher, b200_lba_t opt, const b200_track_params_t* prm, int n_frames,
                         b200_track_frame_t* frames);
/* Device time of the last b200_track_local_map, per stage: 0 undistort + can_observe + query build, 1 grid, 2 candidates, 3 resolve,
 * 4 edge build, 5 pose optimisation + scatter, 6 whole chain (CUDA events on the stream). */
int b200_track_stage_ms(b200_matcher_t matcher, int stage, float* ms);

/* ------------------------------------------------------------------------------------------------------------------
 * Motion-model tracking on the device: module::frame_tracker::motion_based_track (module/frame_tracker.cc:20-59) with
 * match::projection(0.9, true) for `n_frames` independent frames in ONE launch sequence, reading the extractor's results in HBM:
 *   the predicted pose pose_cw = velocity * last_frm.get_pose_cw() (computed by the caller, :24); the frame starts with no landmarks
 *   projection::match_current_and_last_frames (match/projection.cc:95-207): assume_forward / assume_backward from trans_lc (fp64,
 *     reference order) against true_baseline (never for monocular setups), one query per entry of the last-frame table (reproject_to_image
 *     of the camera model, octave window of the last keypoint, margin * scale_factors[last octave], 30-degree orientation gate, stereo
 *     x_right gate, HAMMING_DIST_THR_HIGH)
 *   when fewer than num_matches_thr matches: a second search at twice the margin on a frame without landmarks (:32-36); its result
 *     replaces the first one.  Still short: the frame fails, its pose stays pose_cw and the matches of the last search are reported.
 *   pose_optimizer::optimize (pose_optimizer_g2o.cc:38-175, the < 5 observations early return included) on the keypoints that carry a
 *     landmark, then discard_outliers (:133-150): an outlier keypoint loses its landmark; tracked = n_valid >= num_matches_thr.
 * prm: b200_track_params_t with margin = margin_last_frame_projection (20; 10 in the KITTI example), hamming_thr, max_candidates, the
 * camera / bounds / grid / levels and the optimiser's trials; lowe_ratio, ray_cos_thr and log_scale_factor are not used.  The orientation
 * check is always on (the reference constructs the matcher with it).  true_baseline = camera::base::true_baseline_.
 * Errors as b200_track_local_map: B200_ERR_INVALID for bad parameters, an n_keypoints_in that disagrees with the extractor's count
 * or a missing last_pose_cw in a non-monocular setup; B200_ERR_CAPACITY for a search-window overflow or an undersized kp_cap.
 * One upload, one download and one stream synchronise per call; the retry decision and the choice of search stay on the device. */
typedef struct b200_motion_track_frame {
    int32_t frame;                     /* index into the extractor's last batch */
    const double* pose_cw;             /* 16, row-major, predicted: velocity * last pose */
    const double* last_pose_cw;        /* 16, last_frm pose after update_last_frame; may be NULL when monocular */
    int32_t n_keypoints_in;            /* entries of kp_x_right (0 when NULL); must equal the frame's keypoint count */
    const float* kp_x_right;           /* stereo_x_right_ of the current frame (b200_stereo_compute / b200_rgbd_depths), NULL = monocular */
    int32_t n_landmarks;               /* last-frame table: keypoints with a landmark that is not will_be_erased, last-frame keypoint order */
    const double* lm_pos_w;            /* 3 per entry */
    const uint8_t* lm_desc;            /* 32 per entry: landmark::get_descriptor() */
    const uint8_t* lm_octave;          /* last_frm undist_keypts_[idx].octave */
    const float* lm_angle;             /* last_frm undist_keypts_[idx].angle */
    const uint8_t* lm_has_observation; /* NULL = all have */
    int32_t kp_cap;                    /* capacity of kp_landmark_out (>= the frame's keypoint count) */
    int32_t* kp_landmark_out;          /* out, per keypoint: table row after discard_outliers, -1 none */
    double pose_cw_out[16];            /* out */
    int32_t n_keypoints, n_matches_first, n_matches, retried; /* out; n_matches = count of the search that decided */
    uint32_t n_valid;                  /* out: discard_outliers' count */
    int32_t tracked;                   /* out: motion_based_track's return value */
} b200_motion_track_frame_t;
int b200_motion_based_track(b200_orb_t orb, b200_matcher_t matcher, b200_lba_t opt, const b200_track_params_t* prm, double true_baseline,
                            uint32_t num_matches_thr, int n_frames, b200_motion_track_frame_t* frames);
/* Device time of the last b200_motion_based_track, per stage: 0 undistort + query build, 1 grid, 2 first search, 3 retry set-up + second
 * search + choice, 4 edge build, 5 pose optimisation + scatter + discard, 6 whole chain (CUDA events on the stream). */
int b200_motion_track_stage_ms(b200_matcher_t matcher, int stage, float* ms);

/* ------------------------------------------------------------------------------------------------------------------
 * Robust-match tracking on the device: module::frame_tracker::robust_match_based_track (module/frame_tracker.cc:97-131) with
 * match::robust(lowe_ratio, true)::match_frame_and_keyframe (match/robust.cc:195-230) for `n_frames` independent frames in ONE launch
 * sequence, reading the extractor's results in HBM:
 *   undistortion and bearings of the frame's keypoints (the four camera models of b200_keypoints_undistort)
 *   robust::brute_force_match (robust.cc:232-328): the frame is side 1, the reference keyframe side 2 (its keypoints whose landmark
 *     exists and is not will_be_erased, kf_valid); HAMMING_DIST_THR_LOW, the orientation check on; pairs sorted by frame keypoint
 *   essential_solver::find_via_ransac(1000, true) with the five-point set on the pairs' bearings; its 1 000 minimal sets are drawn on the
 *     device from the frame's engine, bit-identical to b200_draw_min_sets
 *   n_inliers = the inlier count, 0 when the solution is not valid; applied = n_inliers >= num_matches_thr (:105-108)
 *   when applied: set_landmarks (every inlier pair gives its frame keypoint the keyframe keypoint's landmark, every other keypoint none),
 *     the pose last_pose_cw, pose_optimizer::optimize (the < 5 observations early return included), then discard_outliers (:133-150):
 *     an outlier keypoint loses its landmark; tracked = n_valid >= num_matches_thr.
 * prm: b200_track_params_t with lowe_ratio = 0.8 (robust(0.8, true)), the camera, levels and the optimiser's trials; margin,
 * hamming_thr, grid, max_candidates, ray_cos_thr and log_scale_factor are not used.
 * When applied is 0 the reference returns before it touches the frame: kp_landmark_out and pose_cw_out are not written, n_valid and
 * tracked are 0.  B200_ERR_INVALID, with nothing written, for bad parameters, a null required pointer, an n_keypoints_in that
 * disagrees with the extractor's count or a kp_cap below it.  One upload, one download and one stream synchronise per call. */
typedef struct b200_robust_track_frame {
    int32_t frame;                      /* index into the extractor's last batch */
    const double* last_pose_cw;         /* 16, row-major: last_frm.get_pose_cw(), the optimisation's initial pose (:115) */
    int32_t n_keypoints_in;             /* entries of kp_x_right (0 when NULL); must equal the frame's keypoint count */
    const float* kp_x_right;            /* stereo_x_right_ of the current frame, NULL = monocular */
    const struct b200_mt19937* engine;  /* the solver's engine (b200_mt19937_seed); NULL = default-constructed, create_random_engine(true) */
    int32_t n_kf_keypoints;             /* reference keyframe, in its keypoint order: */
    const uint8_t* kf_desc;             /* 32 per keypoint: frm_obs_.descriptors_ */
    const float* kf_angle;              /* undist_keypts_[i].angle */
    const double* kf_bearings;          /* 3 per keypoint: frm_obs_.bearings_ */
    const uint8_t* kf_valid;            /* 1 = the keypoint has a landmark that is not will_be_erased */
    const double* kf_pos_w;             /* 3 per keypoint: its landmark's position (read for valid keypoints only) */
    int32_t kp_cap;                     /* capacity of kp_landmark_out (>= the frame's keypoint count) */
    int32_t* kp_landmark_out;           /* out when applied, per keypoint: the keyframe keypoint whose landmark it carries, -1 none */
    double pose_cw_out[16];             /* out when applied */
    int32_t n_keypoints, n_matches;     /* out; n_matches = brute_force_match's count */
    int32_t essential_valid, status;    /* out: solution_is_valid(), and B200_OK or B200_ERR_INVALID as b200_essential_problem_t.status */
    int32_t n_inliers, applied;         /* out: match_frame_and_keyframe's return value; n_inliers >= num_matches_thr */
    uint32_t n_valid;                   /* out: discard_outliers' count */
    int32_t tracked;                    /* out: robust_match_based_track's return value */
} b200_robust_track_frame_t;
int b200_robust_match_based_track(b200_orb_t orb, b200_matcher_t matcher, b200_lba_t opt, const b200_track_params_t* prm, uint32_t num_matches_thr,
                                  int n_frames, b200_robust_track_frame_t* frames);
/* Device time of the last b200_robust_match_based_track, per stage: 0 undistort + bearings, 1 brute force, 2 sampler, 3 essential,
 * 4 edge build, 5 pose optimisation + discard, 6 whole chain (CUDA events on the stream). */
int b200_robust_track_stage_ms(b200_matcher_t matcher, int stage, float* ms);

/* ------------------------------------------------------------------------------------------------------------------
 * BoW-match tracking on the device: module::frame_tracker::bow_match_based_track (module/frame_tracker.cc:61-95) with
 * match::bow_tree(0.7, true)::match_frame_and_keyframe (match/bow_tree.cc:169-256) for `n_frames` independent frames in ONE launch
 * sequence, reading the extractor's results in HBM:
 *   undistortion of the frame's keypoints (the four camera models of b200_keypoints_undistort) and their angles
 *   match_frame_and_keyframe: the reference keyframe is side 1 (its keypoints whose landmark exists and is not will_be_erased, kf_valid),
 *     the frame side 2; a keyframe keypoint only sees frame keypoints of its own BoW node, a frame keypoint that already received a
 *     landmark is skipped, the 30-degree orientation gate, best <= HAMMING_DIST_THR_LOW and lowe_ratio * second >= best (float).  The
 *     same candidate pass and resolve as b200_match_pairs variant B200_PAIRS_BOW, bit for bit.
 *   applied = n_matches >= num_matches_thr (:69-72)
 *   when applied: set_landmarks (a matched frame keypoint takes the keyframe keypoint's landmark, every other keypoint none), the pose
 *     last_pose_cw, pose_optimizer::optimize (the < 5 observations early return included), then discard_outliers (:133-150): an outlier
 *     keypoint loses its landmark; tracked = n_valid >= num_matches_thr.
 * The BoW vectors stay on the host (curr_frm_.compute_bow, tracking_module.cc:343-345); the chain takes one node id per keypoint on both
 * sides: the key of bow_feat_vec_ that lists the keypoint, or -1 when no node lists it (such a keypoint takes no part).
 * prm: b200_track_params_t with lowe_ratio = 0.7 (bow_tree(0.7, true)), the camera, levels, the optimiser's trials and max_candidates
 * (the gated candidates one keyframe keypoint keeps, 0 = 64 as in b200_match_pairs); margin, hamming_thr, grid, ray_cos_thr and
 * log_scale_factor are not used.
 * When applied is 0 the reference returns before it touches the frame: kp_landmark_out and pose_cw_out are not written, n_valid and
 * tracked are 0.  B200_ERR_INVALID, with nothing written, for bad parameters, a null required pointer, an n_keypoints_in that
 * disagrees with the extractor's count or a kp_cap below it; B200_ERR_CAPACITY, with nothing written, when a keyframe keypoint has more
 * gated candidates than max_candidates.  One upload, one download and one stream synchronise per call. */
typedef struct b200_bow_track_frame {
    int32_t frame;                      /* index into the extractor's last batch */
    const double* last_pose_cw;         /* 16, row-major: last_frm.get_pose_cw(), the optimisation's initial pose (:78) */
    int32_t n_keypoints_in;             /* entries of kp_node and kp_x_right; must equal the frame's keypoint count */
    const int32_t* kp_node;             /* BoW node of every frame keypoint (the key of bow_feat_vec_ that lists it), -1 = none */
    const float* kp_x_right;            /* stereo_x_right_ of the current frame, NULL = monocular */
    int32_t n_kf_keypoints;             /* reference keyframe, in its keypoint order: */
    const uint8_t* kf_desc;             /* 32 per keypoint: frm_obs_.descriptors_ */
    const float* kf_angle;              /* undist_keypts_[i].angle */
    const int32_t* kf_node;             /* BoW node of every keyframe keypoint, -1 = none */
    const uint8_t* kf_valid;            /* 1 = the keypoint has a landmark that is not will_be_erased */
    const double* kf_pos_w;             /* 3 per keypoint: its landmark's position (read for valid keypoints only) */
    int32_t kp_cap;                     /* capacity of kp_landmark_out (>= the frame's keypoint count) */
    int32_t* kp_landmark_out;           /* out when applied, per keypoint: the keyframe keypoint whose landmark it carries, -1 none */
    double pose_cw_out[16];             /* out when applied */
    int32_t n_keypoints, n_matches;     /* out; n_matches = match_frame_and_keyframe's return value */
    int32_t applied;                    /* out: n_matches >= num_matches_thr */
    uint32_t n_valid;                   /* out: discard_outliers' count */
    int32_t tracked;                    /* out: bow_match_based_track's return value */
} b200_bow_track_frame_t;
int b200_bow_match_based_track(b200_orb_t orb, b200_matcher_t matcher, b200_lba_t opt, const b200_track_params_t* prm, uint32_t num_matches_thr,
                               int n_frames, b200_bow_track_frame_t* frames);
/* Device time of the last b200_bow_match_based_track, per stage: 0 undistort + angles, 1 candidate lists, 2 resolve, 3 gate + landmark
 * table, 4 edge build, 5 pose optimisation + discard, 6 whole chain (CUDA events on the stream). */
int b200_bow_track_stage_ms(b200_matcher_t matcher, int stage, float* ms);

/* ------------------------------------------------------------------------------------------------------------------
 * New landmarks of the mapping module: module::two_view_triangulator (src/stella_vslam/module/two_view_triangulator.{h,cc}, with
 * solve::triangulator::triangulate, solve/triangulator.h:77-90, and data::triangulate_stereo, data/common.cc:192-260) and the
 * numeric chain of mapping_module::create_new_landmarks after the baseline test (mapping_module.cc, triangulate_with_two_keyframes).
 * Linear triangulation takes the null vector of the 4x4 system by a two-sided Jacobi SVD in the manner of Eigen::JacobiSVD; all
 * arithmetic follows the CPU restatement's evaluation order (fp64 / fp32 where the reference uses each, no contraction).  atan2 /
 * cos / asin are CUDA's libm (within 1-2 ulp of glibc); they feed accept / reject comparisons only (DESIGN.md section 4).
 * ---------------------------------------------------------------------------------------------------------------- */
/* One keyframe as the triangulator reads it.  b200_camera_t lacks the fields below and keeps its layout. */
typedef struct b200_tri_keyframe {
    double pose_cw[16];             /* keyframe::get_pose_cw(), row-major 4x4 */
    double pose_wc[16];             /* keyframe::get_pose_wc() as the keyframe stores it (camera centre = column 3) */
    int32_t model;                  /* 0: perspective family (perspective / fisheye / radial division), 1: equirectangular */
    double fx, fy, cx, cy, fx_inv, fy_inv; /* camera::perspective (fisheye, radial_division) members */
    double focal_x_baseline, true_baseline; /* camera::base */
    double cols, rows;              /* equirectangular */
    float scale_factor;             /* orb_params_->scale_factor_ */
    int32_t num_levels;             /* entries of the two tables below */
    const float* scale_factors;     /* orb_params_->scale_factors_ */
    const float* level_sigma_sq;    /* orb_params_->level_sigma_sq_ */
    int32_t n_keypoints;
    const float* x;                 /* frm_obs_.undist_keypts_[i].pt.x */
    const float* y;
    const int32_t* octave;          /* undist_keypts_[i].octave */
    const float* x_right;           /* frm_obs_.stereo_x_right_, NULL when empty (monocular) */
    const float* depth;             /* frm_obs_.depths_, NULL when empty */
    const double* bearings;         /* frm_obs_.bearings_, n x 3 */
} b200_tri_keyframe_t;

/* two_view_triangulator(keyfrm_1, keyfrm_2, rays_parallax_deg_thr).triangulate(idx_1, idx_2, pos_w) for every match of every problem,
 * in one upload, one launch and one download.  cos(deg * pi / 180) and ratio_factor_ are taken on the host as the constructor does.
 * Out per match: pos_w (3 doubles; the point computed before the depth / reprojection / scale tests, zeros when neither triangulation
 * branch applied) and ok (1 = the reference returns true); n_ok.  B200_ERR_INVALID (nothing written) for an index or octave out of
 * range and for a stereo keypoint (x_right >= 0) on an equirectangular camera, which the reference does not implement (it throws). */
typedef struct b200_triangulate_problem {
    const b200_tri_keyframe_t* keyfrm_1;
    const b200_tri_keyframe_t* keyfrm_2;
    float rays_parallax_deg_thr;    /* the mapping module passes 1.0 */
    int32_t n_matches;
    const int32_t* matches;         /* n_matches x (idx_1, idx_2) */
    double* pos_w;                  /* out, n_matches x 3 */
    uint8_t* ok;                    /* out, n_matches */
    int32_t n_ok;                   /* out */
} b200_triangulate_problem_t;
int b200_triangulate_pairs(b200_matcher_t h, int n_problems, b200_triangulate_problem_t* problems);

/* mapping_module::create_new_landmarks after the baseline test, for `n_keyframes` current keyframes (several maps / streams, or a
 * backlog) in ONE launch sequence: one upload, one candidate pass of match_for_triangulation (variant B200_PAIRS_TRIANGULATION of
 * b200_match_pairs, check_orientation = false as the mapping module builds it) over every (keyframe, neighbour) problem, then per
 * neighbour rank the sequential resolve and the triangulation of that rank's matches, one download and one synchronisation.
 * Neighbours are processed in the caller's order (get_top_n_covisibilities); every created landmark attaches to its row of the current
 * keyframe, so the later neighbours no longer match that row (robust.cc:44-48) -- the dependency that makes the reference loop
 * sequential, kept on the device.  The caller builds E_12 and the epiplane with the reference's own code, as for b200_match_pairs.
 * Output per keyframe: the landmarks in creation order (neighbour rank, then ascending idx_1), i.e. the order of next_landmark_id_.
 * Deviation: the reference polls abort_create_new_landmarks between neighbours (from the second one on); this chain is not
 * interruptible, so the caller tests the flag before the call and the result is the reference's outcome without an abort (which
 * in the reference depends on timing).  B200_ERR_CAPACITY as b200_match_pairs (max_candidates 0 = 64 gated candidates per row;
 * on-chip occupancy table bounds the neighbours' keypoint counts); B200_ERR_INVALID as b200_triangulate_pairs, checked over every
 * keypoint of the views. */
typedef struct b200_new_landmarks_neighbour {
    const b200_tri_keyframe_t* keyfrm;
    const uint8_t* desc;            /* n_keypoints x 32 */
    const uint8_t* valid;           /* keypoint has no landmark (robust.cc:66-69); NULL = all */
    const int32_t* node;            /* BoW node per keypoint (bow_tree::match_for_triangulation); NULL iff the current keyframe's is NULL */
    double E_12[9];                 /* row-major, essential_solver::create_E_21(keyfrm_1, keyfrm_2) */
    double epiplane_in_keyfrm_2[3];
    int32_t valid_epiplane;
    int32_t* match_out;             /* optional out, current keyframe's n_keypoints: the matcher's result for this neighbour */
    int32_t n_matches;              /* out: the return value of match_for_triangulation */
    int32_t n_created;              /* out: landmarks created with this neighbour */
} b200_new_landmarks_neighbour_t;
typedef struct b200_new_landmarks_problem {
    const b200_tri_keyframe_t* keyfrm; /* the current keyframe (side 1 of every match) */
    const uint8_t* desc;
    const uint8_t* valid;           /* keypoint has no landmark at entry; NULL = all */
    const int32_t* node;
    int32_t n_neighbours;
    b200_new_landmarks_neighbour_t* neighbours; /* ordered */
    int32_t* created_rank;          /* out, capacity n_keypoints: neighbour rank of each created landmark */
    int32_t* created_idx;           /* out, capacity n_keypoints x (idx_1, idx_2) */
    double* created_pos_w;          /* out, capacity n_keypoints x 3 */
    int32_t n_created;              /* out */
} b200_new_landmarks_problem_t;
int b200_create_new_landmarks(b200_matcher_t h, int n_keyframes, b200_new_landmarks_problem_t* problems, float lowe_ratio, float residual_rad_thr,
                              float rays_parallax_deg_thr, int max_candidates);

/* Depth-seeded landmarks of a stereo or RGB-D keyframe, for many keyframes in one upload, one launch (one CTA per problem) and one download
 * on the matcher's stream:
 *   mode 0 (B200_DEPTH_LM_KEYFRAME) : module::keyframe_inserter::create_new_keyframe (module/keyframe_inserter.cc:160-212): the keypoints
 *       with 0 < depth sorted ascending by (depth, idx) as std::sort orders pair<float, unsigned>, walked with `count` = position in that
 *       order; the walk stops at the first count with 100 < count && depth_thr < depth; a keypoint that already has a landmark
 *       (has_landmark[idx] != 0) is skipped but still advances count.  At most B200_DEPTH_LM_MAX_SORT keypoints with 0 < depth per problem
 *       (the sort runs in shared memory): more is B200_ERR_CAPACITY for that problem.
 *   mode 1 (B200_DEPTH_LM_INITIAL)  : module::initializer::create_map_for_stereo (module/initializer.cc:363-387): every keypoint with
 *       0 < depth, in index order; has_landmark is not read.
 * Each created landmark: pos_w = data::triangulate_stereo (data/common.cc:192-260): unproj = (float)((x - cx) * depth * fx_inv) (likewise
 * y) in double, pos_c = (unproj_x, unproj_y, depth), pos_w = R_wc pos_c + t_wc in double with each row summed left to right; then
 * landmark::update_mean_normal_and_obs_scale_variance (data/landmark.cc:256-311) with its one observation, which is also its reference
 * keyframe, at the frame's camera centre (t_wc) and scale_factors[octave]: the device function of b200_landmark_geometry.  Its descriptor
 * (compute_descriptor of one observation) is the keypoint's own row: created_idx gives it.  Outputs are in creation order, i.e. the
 * order of map_database::next_landmark_id_.  try_initialize_for_stereo's count (initializer.cc) is left to the caller.
 * status per problem: B200_OK; B200_ERR_INVALID for model 1 (equirectangular) with a keypoint of 0 < depth (data/common.cc:236-238
 * throws), an octave of a 0 < depth keypoint outside [0, num_levels), a null required pointer or a mode other than 0 / 1;
 * B200_ERR_CAPACITY as above.  Problems whose status is not B200_OK write n_created = 0 and no landmarks; the call returns the first
 * such status (B200_OK when every problem ran). */
#define B200_DEPTH_LM_KEYFRAME 0
#define B200_DEPTH_LM_INITIAL 1
#define B200_DEPTH_LM_MAX_SORT 8192
typedef struct b200_depth_landmarks_problem {
    int32_t mode;                   /* B200_DEPTH_LM_KEYFRAME or B200_DEPTH_LM_INITIAL */
    int32_t model;                  /* model code as in b200_camera_intrinsics_t: 0, 2 or 3; 1 is rejected once a depth is valid */
    double pose_wc[16];             /* frame::get_pose_wc(), row-major: rot_wc, trans_wc (the camera centre) */
    double fx_inv, fy_inv, cx, cy;  /* camera::perspective (fisheye, radial_division) members */
    double depth_thr;               /* camera::base::depth_thr_ (mode 0) */
    int32_t n_keypoints;
    const float* x;                 /* frm_obs_.undist_keypts_[i].pt.x */
    const float* y;
    const int32_t* octave;          /* undist_keypts_[i].octave */
    const float* depth;             /* frm_obs_.depths_ (b200_rgbd_depths or b200_stereo_compute) */
    const uint8_t* has_landmark;    /* mode 0: curr_frm.get_landmark(idx) is set; NULL = none */
    int32_t num_levels;             /* entries of scale_factors */
    const float* scale_factors;     /* orb_params_->scale_factors_ */
    float inv_scale_factor_last;    /* orb_params_->inv_scale_factors_[num_levels - 1] */
    /* out, capacity n_keypoints each */
    int32_t* created_idx;           /* keypoint index of each created landmark */
    double* pos_w;                  /* 3 per landmark */
    double* mean_normal;            /* 3 per landmark */
    float* min_valid_dist;
    float* max_valid_dist;
    int32_t n_created;              /* out */
    int32_t status;                 /* out */
} b200_depth_landmarks_problem_t;
int b200_depth_landmarks(b200_matcher_t h, int n_problems, b200_depth_landmarks_problem_t* problems);

/* Keyframe culling: module::local_map_cleaner::remove_redundant_keyframes (module/local_map_cleaner.cc:68-193) with the observation
 * erasure of keyframe::prepare_for_erasing and landmark::erase_observation (data/keyframe.cc:613-660, data/landmark.cc:124-160), for
 * many maps in one upload, one launch (one CTA per problem), one download and one synchronisation on the matcher's stream.
 * The caller gathers under map_database::mtx_database_:
 *   - the covisibilities, graph_node_->get_top_n_covisibilities(top_n) in that order (a covisibility's position is its rank);
 *   - a landmark table holding every landmark that a covisibility's keypoint lists, once, in CSR form: per landmark its observations
 *     as get_observations() walks them, each with the observer's rank (-1 for any keyframe that is not a listed covisibility, the
 *     current keyframe included), the octave undist_keypts_.at(obs.second).octave and the weight (2 when the observer's
 *     stereo_x_right_ is not empty and stereo_x_right_.at(obs.second) >= 0, else 1: landmark::add_observation, landmark.cc:116-121).
 *     The starting num_observations() of a landmark is the sum of its weights.
 * Ranks run in order.  A rank is skipped (skipped = 1) for the spanning root and (skipped = 2) for the recent window
 * id <= cur_id && cur_id <= id + 2 in uint32_t arithmetic.  Otherwise every keypoint whose landmark is live and whose depth passes
 * (depth == NULL, or !(depth < 0 || depth_thr < depth) in double) counts in n_valid; one whose landmark has num_observations() > 3 and
 * at least 3 live observations by other keyframes at an octave <= its own + 1 counts in n_redundant.  The keypoint's own octave is
 * that of its landmark's observation by this rank.  The rank is removed when
 * redundant_obs_ratio_thr <= (double)((float)n_redundant / (float)n_valid) (so 9/10 against 0.9 is kept and 0/0 is kept), and its
 * observations are then erased before the next rank counts: each live landmark it lists loses that observation and its weight, and a
 * landmark left with no observation is discarded (will_be_erased), so no later rank counts it.
 * The caller makes the reference's early return (redundant_obs_ratio_thr < 0 or top_n <= 0: no call) and applies each removed rank's
 * prepare_for_erasing in rank order.  A keyframe that set_not_to_be_erased() pinned is not erased by prepare_for_erasing although the
 * reference counts it as removed; the device's later ranks assumed it was.  The caller therefore checks will_be_erased() after each
 * prepare_for_erasing, and when a removed keyframe was not erased it gathers again and calls again for the ranks after it: the
 * reference's count is then the removed ranks of the first call up to that keyframe plus the second call's n_removed.
 * B200_ERR_INVALID, with nothing written, for: a negative count; a null required pointer; obs_offsets not starting at 0 or descending;
 * an obs_rank outside [-1, n_covisibilities), an obs_weight other than 1 or 2, or a kp_landmark outside [-1, n_landmarks); and a
 * landmark that a covisibility's keypoints list a number of times other than the number of its observations by that rank, unless
 * both are 0 -- each listed landmark must name the rank exactly once and each observation by a rank must be listed by exactly one
 * keypoint of it. */
typedef struct b200_cull_keyframe {
    uint32_t id;                    /* keyframe::id_ */
    int32_t is_root;                /* graph_node_->is_spanning_root() */
    int32_t n_keypoints;            /* frm_obs_.undist_keypts_.size() */
    const int32_t* kp_landmark;     /* get_landmarks()[idx] as a landmark-table row; -1 when null or will_be_erased() */
    const float* depth;             /* frm_obs_.depths_ when depth_is_available(), else NULL */
    double depth_thr;               /* camera_->depth_thr_ */
    /* out */
    int32_t n_valid, n_redundant;   /* count_redundant_observations; 0 for a skipped rank */
    int32_t skipped;                /* 0, 1 (spanning root) or 2 (recent window) */
    int32_t removed;                /* 1 when the rank is removed */
} b200_cull_keyframe_t;
typedef struct b200_cull_problem {
    uint32_t cur_id;                /* cur_keyfrm->id_ */
    double redundant_obs_ratio_thr; /* local_map_cleaner::redundant_obs_ratio_thr_ (default 0.9) */
    int32_t n_covisibilities;
    b200_cull_keyframe_t* covisibilities; /* in rank order */
    int32_t n_landmarks;
    const int32_t* obs_offsets;     /* n_landmarks + 1 (may be NULL when n_landmarks is 0) */
    const int32_t* obs_rank;        /* obs_offsets[n_landmarks] entries each */
    const int32_t* obs_octave;
    const uint8_t* obs_weight;
    int32_t n_removed;              /* out: the reference's return value */
    int32_t status;                 /* out: B200_OK once the problem has run */
} b200_cull_problem_t;
int b200_remove_redundant_keyframes(b200_matcher_t h, int n_problems, b200_cull_problem_t* problems);

/* ------------------------------------------------------------------------------------------------------------------
 * Relocalisation's PnP: solve::pnp_solver (src/stella_vslam/solve/pnp_solver.{h,cc}) -- EPnP (Lepetit et al., IJCV 2009) inside
 * RANSAC -- for many problems (lost frame x candidate keyframe) in one launch sequence on the b200_lba_t handle's stream, so the pose
 * goes straight on to b200_pose_optimize.  fp64 in the CPU restatement's evaluation order (sums left to right; Eigen's JacobiSVD,
 * ColPivHouseholderQR-preconditioned JacobiSVD::solve and HouseholderQR::solve restated).  Deviations (DESIGN.md section 8): Eigen's
 * vectorised summation order is not reproduced; a hypothesis whose compute_pose writes no pose is rejected (the reference scores the
 * previous hypothesis' pose again, which can never win, and reads uninitialised memory for hypothesis 0); Jacobi sweeps are bounded.
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct b200_pnp_problem {
    int32_t n_matches;
    const double* bearings;         /* n x 3: frm_obs_.bearings_ of the valid matches */
    const double* points;           /* n x 3: landmark::get_pos_in_world() */
    const int32_t* octaves;         /* n: undist_keypts_[i].octave */
    int32_t num_levels;             /* entries of scale_factors */
    const float* scale_factors;     /* orb_params_->scale_factors_ */
    uint32_t min_num_inliers;       /* relocalizer: 10 */
    uint32_t gauss_newton_num_iter; /* constructor default 10 */
    uint32_t max_num_iter;          /* relocalizer: max_num_ransac_iter_ = 30 */
    int32_t recompute;              /* find_via_ransac's recompute */
    const int32_t* min_sets;        /* max_num_iter x 4: the draws of util::create_random_array, in draw order (b200_pnp_draw_min_sets) */
    /* out */
    int32_t status;                 /* B200_OK, or B200_ERR_INVALID when a Jacobi SVD hit its sweep bound (the results are then unreliable) */
    int32_t valid;                  /* solution_is_valid() */
    int32_t best_iter;              /* hypothesis that won (-1 none) */
    int32_t num_inliers;            /* of the winning hypothesis */
    double min_cost;                /* of the winning hypothesis (DBL_MAX when none) */
    double rot_cw[9];               /* row-major; written only when valid (get_best_rotation) */
    double trans_cw[3];             /* written only when valid */
    uint8_t* inlier_flags;          /* n: get_inlier_flags(); all 0 when not valid; untouched on the early return (n < 4 or n < min_num_inliers) */
} b200_pnp_problem_t;
/* find_via_ransac(max_num_iter, recompute) for every problem: one upload, the hypothesis and selection launches, one download.
 * B200_ERR_INVALID (nothing written) for a negative count, a null required pointer, an octave outside [0, num_levels) or a min_sets index
 * outside [0, n) of a problem that runs RANSAC. */
int b200_pnp_ransac(b200_lba_t h, int n_problems, b200_pnp_problem_t* problems);

typedef struct b200_epnp_problem {
    int32_t n;                      /* >= 1 */
    const double* bearings;         /* n x 3 */
    const double* points;           /* n x 3 */
    uint32_t num_iter;              /* Gauss-Newton iterations (the reference's default argument: 5) */
    /* in / out: kept as given unless a candidate N reaches reproj_error < DBL_MAX, as the reference writes rot_cw / trans_cw */
    double rot_cw[9];
    double trans_cw[3];
    /* out */
    double reproj_error;            /* return value of compute_pose */
    int32_t wrote;                  /* rot_cw / trans_cw were written */
    int32_t status;                 /* B200_OK, or B200_ERR_INVALID when a Jacobi SVD hit its sweep bound */
} b200_epnp_problem_t;
/* pnp_solver::compute_pose (static; also marker_detector::base's per-marker pose) for every problem in one launch. */
int b200_epnp_compute_pose(b200_lba_t h, int n_problems, b200_epnp_problem_t* problems);

/* std::mt19937 as libstdc++ implements it, and util::create_random_array(4, 0, n - 1, engine) as find_via_ransac draws its minimal
 * sets (std::uniform_int_distribution<unsigned>, sort, unique, std::shuffle), on the host (b200_draw_min_sets_batch: the same sampler on
 * the device).  The draws reproduce a reference built
 * against libstdc++ (GCC 11 or later: Lemire's nearly divisionless uniform_int_distribution). */
typedef struct b200_mt19937 {
    uint32_t state[624];
    uint32_t index;
} b200_mt19937_t;
/* n_seed == 0: a default-constructed engine (seed 5489, util::create_random_engine(true)); otherwise std::seed_seq over the words. */
int b200_mt19937_seed(b200_mt19937_t* engine, const uint32_t* seed_seq, int n_seed);
/* The next 32-bit output of the engine (the raw stream). */
uint32_t b200_mt19937_next(b200_mt19937_t* engine);
/* max_num_iter minimal sets (out: max_num_iter x 4) from one engine, continuing its state; n_matches >= 4. */
int b200_pnp_draw_min_sets(b200_mt19937_t* engine, uint32_t n_matches, uint32_t max_num_iter, int32_t* out);
/* max_num_iter calls of util::create_random_array(set_size, 0, n_matches - 1, engine) (out: max_num_iter x set_size), continuing the
 * engine's state.  B200_ERR_INVALID for a null engine, set_size outside [1, 65535] or n_matches < set_size. */
int b200_draw_min_sets(b200_mt19937_t* engine, uint32_t set_size, uint32_t n_matches, uint32_t max_num_iter, int32_t* out);
/* The device sampler of b200_robust_match_based_track for n_engines engines on the handle's stream: engine p (engines NULL: every
 * engine default-constructed) makes max_num_iter calls of util::create_random_array(set_size, 0, n_matches[p] - 1) into
 * out + p * max_num_iter * set_size, the same draws as b200_draw_min_sets; the engines are not advanced.  B200_ERR_INVALID for
 * set_size outside [1, 8] or an n_matches below set_size. */
int b200_draw_min_sets_batch(b200_lba_t h, int n_engines, const b200_mt19937_t* engines, uint32_t set_size, const uint32_t* n_matches,
                             uint32_t max_num_iter, int32_t* out);

/* ------------------------------------------------------------------------------------------------------------------
 * Robust matching's essential matrix: solve::essential_solver::find_via_ransac (src/stella_vslam/solve/essential_solver.cc) with the
 * five-point minimal set (Stewenius et al.), for many problems (frame x keyframe, or an equirectangular initialisation) in one launch
 * sequence on the b200_lba_t handle's stream.  fp64 in the CPU restatement's evaluation order; the pieces of Eigen it uses (FullPivLU,
 * EigenSolver, JacobiSVD with its QR preconditioners) restated.  Deviations (DESIGN.md section 8): Eigen's vectorised summation and
 * blocked triangular-solve order are not reproduced; a RealSchur that does not converge gives no candidates (the reference reads
 * uninitialised eigenvalues) and sets status; Jacobi sweeps are bounded.
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct b200_essential_problem {
    int32_t n_matches;
    const double* bearings_1;       /* n x 3: bearings_1[matches_12[i].first] */
    const double* bearings_2;       /* n x 3: bearings_2[matches_12[i].second] */
    uint32_t min_set_size;          /* must be 5 (every caller in the reference passes the default) */
    uint32_t max_num_iter;          /* robust matcher: 1000 */
    int32_t recompute;              /* find_via_ransac's recompute */
    const int32_t* min_sets;        /* max_num_iter x min_set_size: util::create_random_array's draws in draw order (b200_draw_min_sets) */
    /* out */
    int32_t status;                 /* B200_OK, or B200_ERR_INVALID when a RealSchur did not converge or a Jacobi SVD hit its sweep bound */
    int32_t valid;                  /* solution_is_valid() */
    int32_t best_iter;              /* iteration of the RANSAC winner (-1 none) */
    int32_t best_candidate;         /* its candidate, in eigenvalue order (-1 none) */
    int32_t num_inliers;            /* of the RANSAC winner (before the recompute) */
    float best_cost;                /* get_best_cost(): FLT_MAX when no winner; 0 on the early return (the member's initial value) */
    double E_21[9];                 /* row-major get_best_E_21(); written only when valid */
    uint8_t* inlier_flags;          /* n: get_inlier_matches(); all 0 when not valid; untouched on the early return (n < min_set_size) */
} b200_essential_problem_t;
/* find_via_ransac(max_num_iter, recompute, 5) for every problem: one upload, the hypothesis, scoring and selection launches, one
 * download.  B200_ERR_INVALID (nothing written) for a negative count, a null required pointer, min_set_size != 5 or a min_sets index
 * outside [0, n) of a problem that runs RANSAC. */
int b200_essential_ransac(b200_lba_t h, int n_problems, b200_essential_problem_t* problems);

/* ------------------------------------------------------------------------------------------------------------------
 * Monocular initialisation's two-view RANSAC: solve::homography_solver::find_via_ransac (src/stella_vslam/solve/homography_solver.cc)
 * and solve::fundamental_solver::find_via_ransac (fundamental_solver.cc), with solve::normalize (solve/common.cc) over all keypoints of
 * each frame, for many problems of either model in one launch sequence on the b200_lba_t handle's stream.  initialize::perspective
 * runs one H and one F problem per attempt (recompute = false); both go into one call.  Float exactly where the reference stores
 * float, fp64 elsewhere, in the CPU restatement's evaluation order (csrc/twoview_core.h).  Deviations (DESIGN.md section 8): sums run
 * left to right (Eigen's vectorised reductions are not reproduced); Jacobi sweeps are bounded, and an H coefficient matrix whose sweeps
 * hit the bound counts as degenerate and sets status.
 * ---------------------------------------------------------------------------------------------------------------- */
#define B200_TWOVIEW_H 0
#define B200_TWOVIEW_F 1
typedef struct b200_twoview_problem {
    int32_t model;                  /* B200_TWOVIEW_H (minimal set 4) or B200_TWOVIEW_F (minimal set 8) */
    int32_t n_keypts_1;             /* all undistorted keypoints of frame 1: normalize runs over every one, matched or not */
    const float* keypts_1;          /* n_keypts_1 x 2: undist_keypts_1[i].pt (x, y) */
    int32_t n_keypts_2;
    const float* keypts_2;          /* n_keypts_2 x 2 */
    int32_t n_matches;
    const int32_t* matches_12;      /* n_matches x 2: (index into keypts_1, index into keypts_2) in the reference's order */
    float sigma;                    /* initialize::perspective passes 1.0f */
    uint32_t max_num_iter;          /* initialize::perspective: num_ransac_iterations (default 100) */
    int32_t recompute;              /* find_via_ransac's recompute (initialize::perspective passes false) */
    const int32_t* min_sets;        /* max_num_iter x (4 or 8): util::create_random_array's draws in draw order (b200_draw_min_sets) */
    /* out */
    int32_t status;                 /* B200_OK, or B200_ERR_INVALID when a Jacobi SVD hit its sweep bound */
    int32_t valid;                  /* solution_is_valid() */
    int32_t best_iter;              /* iteration of the RANSAC winner (-1 none) */
    int32_t num_inliers;            /* of the RANSAC winner (before the recompute) */
    float best_cost;                /* get_best_cost(): FLT_MAX when no winner; 0 on the early return (the member's initial value) */
    double M_21[9];                 /* row-major get_best_H_21() / get_best_F_21(); written only when valid */
    uint8_t* inlier_flags;          /* n_matches: get_inlier_matches(); all 0 when not valid; untouched on the early return (n < 8) */
} b200_twoview_problem_t;
/* find_via_ransac(max_num_iter, recompute) for every problem: one upload, the normalisation, hypothesis, scoring and selection
 * launches, one download.  Early return (nothing drawn, flags untouched) when n_matches < 8 for either model.  B200_ERR_INVALID
 * (nothing written) for a negative count, a null required pointer, a model other than H / F, a match index outside its frame's
 * keypoints or a min_sets entry outside [0, n_matches) of a problem that runs RANSAC. */
int b200_twoview_ransac(b200_lba_t h, int n_problems, b200_twoview_problem_t* problems);

/* ------------------------------------------------------------------------------------------------------------------
 * Monocular initialisation: initialize::perspective::initialize (src/stella_vslam/initialize/perspective.cc) and
 * initialize::bearing_vector::initialize (bearing_vector.cc) for many frame pairs in one launch sequence on the b200_lba_t handle's
 * stream: the H and F RANSAC of b200_twoview_ransac (perspective, fisheye, radial division) or the E RANSAC of b200_essential_ransac
 * (equirectangular), all with recompute = false; the rel_cost_H choice; homography_solver::decompose (8 hypotheses) or the
 * essential_solver::decompose of E = K2^T F K1 or of E (4 hypotheses); base::triangulate with the midpoint triangulation for every
 * hypothesis; base::find_most_plausible_pose.  Float exactly where the reference stores float, fp64 elsewhere, in the CPU
 * restatement's evaluation order (csrc/initialize_core.h).  Deviations (DESIGN.md section 8): sums run left to right; Jacobi sweeps
 * are bounded and set status; points that are not triangulated are zeros (the reference leaves them uninitialised); a point behind
 * a camera whose parallax is small is scored with its projection (the reference reads an unset pixel there).
 * ---------------------------------------------------------------------------------------------------------------- */
#define B200_INIT_MODEL_NONE 0
#define B200_INIT_MODEL_H 1
#define B200_INIT_MODEL_F 2
#define B200_INIT_MODEL_E 3
/* Where an attempt stopped.  NO_MODEL and DECOMPOSE leave rot / trans untouched; the rejections of find_most_plausible_pose zero them
 * (base.cc:59-60), as the reference does. */
#define B200_INIT_STAGE_NO_MODEL 0          /* neither RANSAC gave a usable model */
#define B200_INIT_STAGE_DECOMPOSE 1         /* homography_solver::decompose's rank test failed */
#define B200_INIT_STAGE_MIN_VALID 2         /* the largest nums_valid is below min_num_valid_pts */
#define B200_INIT_STAGE_AMBIGUOUS 3         /* more than one hypothesis has 0.8 * max < nums_valid */
#define B200_INIT_STAGE_PARALLAX 4          /* the winner's parallax_cos exceeds cos(parallax_deg_thr) */
#define B200_INIT_STAGE_MIN_TRIANGULATED 5  /* the winner triangulated fewer than min_num_triangulated points */
#define B200_INIT_STAGE_SUCCEEDED 6
typedef struct b200_init_problem {
    b200_camera_intrinsics_t cam_ref, cam_cur; /* models 0, 2, 3: perspective path (K = fx fy cx cy); 1 (both views): bearing_vector */
    float img_bounds_ref[4], img_bounds_cur[4]; /* min_x, max_x, min_y, max_y (unused by model 1) */
    int32_t n_ref, n_cur;                       /* keypoints of each frame */
    const float* undist_ref;                    /* n_ref x 2: frm_obs_.undist_keypts_[i].pt */
    const double* bearings_ref;                 /* n_ref x 3: frm_obs_.bearings_ */
    const float* undist_cur;                    /* n_cur x 2 */
    const double* bearings_cur;                 /* n_cur x 3 */
    const int32_t* ref_matches_with_cur;        /* n_ref: the current keypoint matched to ref keypoint i, negative for none */
    uint32_t num_ransac_iters;                  /* default 100 (module/initializer.cc) */
    uint32_t min_num_triangulated;              /* default 50 */
    uint32_t min_num_valid_pts;                 /* default 50 */
    float parallax_deg_thr;                     /* default 1.0; cos(parallax_deg_thr / 180 * pi) is taken in double on the host */
    float reproj_err_thr;                       /* default 4.0 */
    /* minimal sets of util::create_random_array in draw order (b200_draw_min_sets), each drawn from its solver's own engine; needed
     * only by a problem whose RANSAC runs (8 or more matches on the perspective path, 5 or more on the bearing-vector path) */
    const int32_t* min_sets_H;                  /* num_ransac_iters x 4 (perspective path) */
    const int32_t* min_sets_F;                  /* num_ransac_iters x 8 (perspective path) */
    const int32_t* min_sets_E;                  /* num_ransac_iters x 5 (bearing-vector path) */
    /* out */
    int32_t status;                             /* B200_OK, or B200_ERR_INVALID when a RealSchur or a Jacobi SVD did not converge */
    int32_t succeeded;                          /* initialize()'s return value */
    int32_t model;                              /* B200_INIT_MODEL_*: the model reconstructed with (NONE when no model was usable) */
    int32_t stage;                              /* B200_INIT_STAGE_* */
    int32_t n_matches;                          /* ref_cur_matches_.size() */
    float cost_H, cost_F, cost_E;               /* get_best_cost() of each solver that was constructed (0 otherwise) */
    int32_t valid_H, valid_F, valid_E;          /* solution_is_valid() */
    int32_t num_inliers_H, num_inliers_F, num_inliers_E;
    int32_t n_hypotheses;                       /* 8 (H), 4 (F, E); 0 when find_most_plausible_pose did not run */
    int32_t nums_valid[8];                      /* per hypothesis: base::triangulate's return value */
    int32_t num_triangulated[8];
    float parallax_cos[8];
    double rot_ref_to_cur[9];                   /* row-major get_rotation_ref_to_cur(); see the stages above */
    double trans_ref_to_cur[3];
    double* triangulated_pts;                   /* n_ref x 3, written when succeeded: get_triangulated_pts() */
    uint8_t* triangulated_flags;                /* n_ref, written when succeeded: get_triangulated_flags() */
    uint8_t* inlier_flags;                      /* NULL or n_ref entries: the chosen solver's get_inlier_matches() in its first n_matches,
                                                   written when a model was chosen */
} b200_init_problem_t;
/* initialize(cur_frm, ref_matches_with_cur) for every problem: one upload, the RANSAC launches, the model choice and decomposition,
 * the triangulation of every hypothesis and the selection, one download.  B200_ERR_INVALID (nothing written) for a null handle or
 * required pointer, a negative count, a camera model outside 0-3, model 1 on one view only, non-finite intrinsics of models 2 and 3, a
 * match index at or above n_cur, num_ransac_iters above INT_MAX or a minimal-set index outside [0, n_matches). */
int b200_initialize(b200_lba_t h, int n_problems, b200_init_problem_t* problems);

/* ----------------------------------------------------------------------------------------------------------------
 * Pose-graph optimisation (optimize::graph_optimizer, optimize/graph_optimizer.cc:254-302): the Sim3 essential graph of a loop
 * closure, g2o's Levenberg-Marquardt with numeric central-difference Jacobians (delta 1e-9) and the terminate action, on the handle's
 * stream.  The vertices and edges are built by the caller as :45-250 does (stella_vslam_b200.optimize.build_essential_graph restates
 * it).  The linear solve is an envelope (skyline) Cholesky over 32x32 tiles in a reverse Cuthill-McKee ordering of the free vertices
 * instead of CSparse: both are exact SPD solves and differ in rounding only (DESIGN.md section 8).
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct b200_sim3 {
    double q[4];                    /* g2o::Sim3::rotation().coeffs(): x y z w */
    double t[3];                    /* translation() */
    double s;                       /* scale() */
} b200_sim3_t;
typedef struct b200_pose_graph {
    int32_t n_vertices, n_edges, fix_scale;   /* fix_scale: shot_vertex::fix_scale_ (stereo / RGBD) */
    const b200_sim3_t* estimate;    /* n_vertices: Sim3_cw before the optimisation, in the reference's vertex order */
    const uint8_t* fixed;           /* n_vertices: loop keyframe, current keyframe and spanning root are fixed */
    const int32_t* e_v1;            /* n_edges, insertion order: vertex 0 (id1) */
    const int32_t* e_v2;            /* vertex 1 (id2) */
    const b200_sim3_t* e_meas;      /* Sim3_21 = Sim3_2w * Sim3_w1; information I_7, no robust kernel */
    int32_t n_points;               /* landmarks to correct (may be 0) */
    const double* points;           /* n_points x 3: pos_w */
    const int32_t* point_ref;       /* n_points: vertex index of found_lm_to_ref_keyfrm_id[lm] or lm->get_ref_keyframe() */
    b200_sim3_t* estimate_out;      /* n_vertices: corrected Sim3_cw (fixed vertices bit-unchanged) */
    double* pose_cw_out;            /* n_vertices x 16 row-major: [R | t / s] with s rounded to float (:265-268) */
    double* points_out;             /* n_points x 3 or NULL: corrected_Sim3_wc[ref].map(Sim3_cw[ref].map(pos_w)) (:283-300) */
} b200_pose_graph_t;
typedef struct b200_pgo_stats {
    int32_t iterations;             /* LM iterations run */
    int32_t trials;                 /* linear solves over all iterations */
    double chi2_init, chi2_final, lambda_init, lambda_final;
    int64_t envelope_doubles;       /* size of the envelope factor (32x32 tiles) */
    int64_t factor_flops;           /* floating-point operations of one envelope factorisation, counted from the structure */
    int32_t launches;               /* kernel launches of the whole call (graph nodes counted per replay) */
    float lin_ms, factor_ms, solve_ms, total_ms; /* device time of the linearisations, of envelope assembly + factorisation and of
                                                    substitution + trial oplus + chi2, summed over the call; host wall time of the call */
} b200_pgo_stats_t;
/* Bound on the envelope, in doubles (2 GiB).  A chain-like essential graph (spanning tree plus covisibilities of neighbouring
 * keyframes) needs roughly 2 000 doubles per keyframe and fits up to about 100 000 keyframes; a map that revisits its ground once
 * needs about twice that.  Measured sizes are in DESIGN.md section 8. */
#define B200_PGO_MAX_ENVELOPE_DOUBLES ((int64_t)1 << 28)
/* graph_optimizer::optimize steps 4-5: optimize(max_iter) (50 in the reference) with terminate_action(gain_threshold) (1e-3), then
 * the write-back of the poses and the landmark correction.  The caller still runs update_mean_normal_and_obs_scale_variance().
 * B200_ERR_INVALID (nothing written): a null required pointer, a negative count, an edge with an endpoint out of range or v1 == v2, a
 * point_ref out of range, a non-finite value, a scale <= 0 or a quaternion whose norm is not within [0.5, 2] in an estimate or a
 * measurement, a non-finite point, no free vertex.
 * B200_ERR_CAPACITY (nothing written, nothing allocated): the envelope exceeds B200_PGO_MAX_ENVELOPE_DOUBLES (checked on the host). */
int b200_graph_optimize(b200_lba_t h, const b200_pose_graph_t* g, int max_iter, double gain_threshold, b200_pgo_stats_t* stats);
/* Host only: the reverse Cuthill-McKee order of the free vertices (order_out: n_free vertex indices, position 0 first; may be NULL),
 * the number of free vertices and the envelope b200_graph_optimize would factor.  Same validation as b200_graph_optimize. */
int b200_pgo_envelope(const b200_pose_graph_t* g, int32_t* n_free, int32_t* order_out, int64_t* envelope_doubles);

/* ----------------------------------------------------------------------------------------------------------------
 * Sim3 refinement of a loop candidate (optimize::transform_optimizer::optimize, optimize/transform_optimizer.cc:20-158): one Sim3_12
 * vertex, a forward and a backward reprojection edge per matched pair (internal/sim3/mutual_reproj_edge_wrapper.h) with Huber delta
 * sqrt(chi_sq), g2o's Levenberg-Marquardt with numeric central-difference Jacobians (delta 1e-9) and no terminate action:
 * optimize(5), the outlier test, optimize(num_iter) on the surviving pairs, the inlier count.  One CTA per problem, the whole protocol in
 * one launch on the handle's stream.  The caller gathers the pairs as :58-94 does (stella_vslam_b200.optimize.gather_mutual_edges
 * restates it).  The 7x7 system is solved by a dense Cholesky instead of SimplicialLDLT (DESIGN.md section 8).
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct b200_transform_problem {
    int32_t n_matches;              /* gathered pairs, in ascending idx1 */
    int32_t fix_scale;              /* transform_vertex::fix_scale_ (stereo / RGBD) */
    b200_sim3_t sim3_12;            /* initial Sim3_12 as the caller built it: g2o::Sim3(rot_12, trans_12, scale_12) */
    double rot_1w[9], trans_1w[3];  /* keyfrm_1->get_rot_cw() row-major, get_trans_cw() */
    double rot_2w[9], trans_2w[3];  /* keyfrm_2 */
    b200_camera_t cam_1, cam_2;     /* model 0 (perspective / fisheye / radial division) or 1 (equirectangular); fxb unused */
    const float* obs_1;             /* n x 2: keyfrm_1's undistorted keypoint idx1 (observation of edge_12) */
    const float* inv_sigma_sq_1;    /* n: keyfrm_1's inv_level_sigma_sq_[octave] */
    const double* pos_w_2;          /* n x 3: lm_2->get_pos_in_world() (point of edge_12) */
    const float* obs_2;             /* n x 2: keyfrm_2's undistorted keypoint idx2 (observation of edge_21) */
    const float* inv_sigma_sq_2;    /* n */
    const double* pos_w_1;          /* n x 3: lm_1->get_pos_in_world() (point of edge_21) */
    /* out */
    b200_sim3_t sim3_12_out;        /* optimised Sim3_12; the input when the second round did not run */
    uint8_t* keep;                  /* n: 1 = the entry stays non-null in matched_lms_in_keyfrm_2 */
    uint32_t num_inliers;           /* return value of optimize() */
    int32_t n_outliers_round1;      /* pairs nulled by the first outlier test */
    int32_t iterations[2];          /* LM iterations of optimize(5) and optimize(num_iter) */
    int32_t trials[2];              /* linear solves of each round */
    double chi2[2];                 /* active robust chi2 of the state each round leaves */
    double lambda_init[2];          /* computeLambdaInit of each round */
} b200_transform_problem_t;
/* transform_optimizer(fix_scale, num_iter)::optimize(..., chi_sq) for every problem.  Results are independent of the batch.
 * B200_ERR_INVALID (nothing written): a null handle or required pointer, a negative count, chi_sq <= 0 or non-finite, num_iter < 0,
 * a non-finite value, a scale <= 0 or a quaternion whose norm is not within [0.5, 2] in sim3_12, a camera model other than 0 or 1, an
 * inv_sigma_sq <= 0. */
int b200_transform_optimize(b200_lba_t h, int n_problems, b200_transform_problem_t* problems, float chi_sq, int num_iter);

/* Profiling mode: an event after every launch of the following solves (adds a few microseconds per launch; off by default).
 * b200_lba_kernel_ms reports, for the LAST batch, the summed device time and the number of intervals of
 *   kernel 0 plan (5 launches, one interval), 1 landmark pass / build, 2 keyframe rows, 3 Schur rows, 4 reduced-system Cholesky,
 *   5 back-substitution + chi2 of the trial state, 6 (unused since the trial pass was fused into 5), 7 everything after the last
 *   repetition (round tails, outliers, export). */
int b200_lba_enable_profile(b200_lba_t h, int enable);
int b200_lba_kernel_ms(b200_lba_t h, int kernel, float* total_ms, int* launches);
/* Device time (ms, CUDA events) spent in the kernels of the last solve, and the number of kernel launches. */
int b200_lba_last_profile(b200_lba_t h, float* gpu_ms, int* launches);

#ifdef __cplusplus
}
#endif
#endif /* B200VSLAM_H */
