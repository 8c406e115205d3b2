/*
 * hybvio_b200.h -- C ABI of libhybvio_b200.so: the H100 (sm_90a) implementation of HybVIO's per-frame hot path.
 *
 * Boundary (SURVEY.md 8(b)). Each entry point names the reference interface it replaces (paths relative to the
 * reference root; OCV = 3rdparty/mobile-cv-suite/opencv/modules). The reference-side C++ adapter classes
 * (CudaImagePyramid / CudaOpticalFlow / CudaEKF, hybvio_b200/host/) sit on top of exactly these calls.
 *
 * Conventions: every function returns HV_OK (0) or a negative hv_status; nothing throws across the boundary;
 * handles are opaque; the caller owns host buffers, the library owns device buffers; matrices are fp64
 * COLUMN-MAJOR with leading dimension = rows (Eigen's default layout). All work of a context is issued on one
 * CUDA stream; calls taking host output buffers synchronise that stream before returning, `_device`/`_async`
 * variants do not. A context must be used from one thread at a time (the reference drives Tracker and EKF from
 * a single thread, src/api/api.cpp:425-428).
 *
 * There is NO CPU fallback: hv_ctx_create fails with HV_ERR_NO_DEVICE when no sm_90 GPU is present.
 */
#ifndef HYBVIO_B200_H_
#define HYBVIO_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum hv_status {
    HV_OK = 0,
    HV_ERR_INVALID = -1,      /* bad argument (NULL handle, n < 0, unsupported window size ...) */
    HV_ERR_NO_DEVICE = -2,    /* no CUDA device / not sm_90 */
    HV_ERR_CUDA = -3,         /* a CUDA runtime call failed; see hv_last_error */
    HV_ERR_OOM = -4,
    HV_ERR_UNSUPPORTED = -5,  /* e.g. pyrLKWindowSize not in {11,15,21,31}, maxLevel > 5 */
    HV_ERR_STATE = -6         /* call order violated (e.g. unaugment with no augmented pose) */
} hv_status;

typedef struct hv_ctx hv_ctx;
typedef struct hv_pyr hv_pyr;
typedef struct hv_ekf hv_ekf;

/* ---------------------------------------------------------------- context ------------------------------- */
const char* hv_version(void);
/* Last error text of this thread (valid until the next failing call). */
const char* hv_last_error(void);
int hv_device_count(void);
/* Creates a context on `device` with its own non-blocking stream. */
int hv_ctx_create(int device, hv_ctx** out);
/* Same, but issues all work on a caller-owned cudaStream_t (e.g. torch.cuda.current_stream().cuda_stream). */
int hv_ctx_create_on_stream(int device, void* cuda_stream, hv_ctx** out);
int hv_ctx_destroy(hv_ctx* ctx);
/* Waits for everything issued through the context: its stream and the library's side stream (hv_ekf_run_device_results). */
int hv_ctx_sync(hv_ctx* ctx);
/* The stream as a cudaStream_t (for event timing by the caller). */
void* hv_ctx_stream(hv_ctx* ctx);
/* Number of kernels this context has launched so far (bench.py's gpu_launches). */
long long hv_ctx_launch_count(hv_ctx* ctx);

/* ---------------------------------------------------------------- image pyramid ------------------------- */
/* Replaces tracker::ImagePyramid + CpuImagePyramidFactory (src/tracker/image_pyramid.hpp:18-42,
 * image_pyramid.cpp:28-48): one object per camera frame, recycled through a pool like util::Allocator.
 * win = tracker.pyrLKWindowSize, max_level = tracker.pyrLKMaxLevel. Level sizes follow
 * cv::buildOpticalFlowPyramid (OCV/video/src/lkpyramid.cpp:726-822): ((w+1)/2, (h+1)/2), stopping early when
 * the next level would be <= win. */
int hv_pyr_create(hv_ctx* ctx, int width, int height, int win, int max_level, hv_pyr** out);
int hv_pyr_release(hv_pyr* pyr);
int hv_pyr_levels(const hv_pyr* pyr);
int hv_pyr_level_size(const hv_pyr* pyr, int level, int* width, int* height);
/* Replaces ImagePyramid::Factory::compute -> cv::buildOpticalFlowPyramid. `gray` is a HOST 8-bit image
 * (accelerated::Image CPU storage, row stride in bytes). Asynchronous: H2D copy + one fused kernel on the
 * context stream; the host buffer must stay valid until the next synchronising call (use pinned memory for
 * a truly asynchronous copy). */
int hv_pyr_build(hv_pyr* pyr, const uint8_t* gray, size_t stride_bytes);
/* Same for `n` images in ONE kernel launch (stereo pair: n = 2). src_is_device != 0: `gray[i]` are device
 * pointers (frame already in HBM). All pyramids must belong to one context and have equal level-0 size. */
int hv_pyr_build_batch(hv_pyr* const* pyrs, const uint8_t* const* gray, const size_t* stride_bytes, int n,
                       int src_is_device);
/* Test/debug accessors, replacing ImagePyramid::getGrayLevel/getGradientLevel/getOpenCv: copy one level to the
 * host. gray: w*h u8; deriv: w*h*2 int16 interleaved (Ix,Iy), GRADIENT_SCALE_0_255 = 1/32
 * (image_pyramid.hpp:19-26). Either pointer may be NULL. Synchronises. */
int hv_pyr_download_level(hv_pyr* pyr, int level, uint8_t* gray, int16_t* deriv);
/* Same, laid out exactly like the reference's cv::Mat level *with* its win-pixel padding (gray REFLECT_101,
 * deriv CONSTANT 0; lkpyramid.cpp:761-808): (w+2win) x (h+2win). The device stores levels unpadded; the
 * border is materialised on the host by this accessor only. */
int hv_pyr_download_level_padded(hv_pyr* pyr, int level, uint8_t* gray, int16_t* deriv);

/* ---------------------------------------------------------------- Lucas-Kanade -------------------------- */
/* Replaces tracker::OpticalFlow::compute -> cv::calcOpticalFlowPyrLK (src/tracker/optical_flow.cpp:10-59,
 * 78-102; OCV/video/src/lkpyramid.cpp:1236-1401, 183-724) with TermCriteria(COUNT|EPS, max_iter, eps),
 * flags = use_initial ? OPTFLOW_USE_INITIAL_FLOW : 0, minEigThreshold = min_eig, `err` requested.
 *   prev_xy   n x (x,y) float32, host
 *   next_xy   n x (x,y) float32, host; in: initial guesses when use_initial, out: tracked end points
 *   status    n x uint8, OpenCV status (1 tracked, 0 failed); may be NULL
 *   track_status  n x int32 tracker::Feature::Status (src/tracker/track.hpp:9-20): TRACKED=0, FAILED_FLOW=2,
 *             FLOW_OUT_OF_RANGE=4, exactly as optical_flow.cpp:52-58 derives it; may be NULL
 * Synchronises. */
int hv_lk_track(hv_ctx* ctx, hv_pyr* prev, hv_pyr* next, const float* prev_xy, float* next_xy, uint8_t* status,
                int32_t* track_status, int n, int use_initial, int max_iter, double eps, double min_eig);
/* Device-resident variant: all pointers are device pointers, nothing is copied, no synchronisation. */
int hv_lk_track_device(hv_ctx* ctx, hv_pyr* prev, hv_pyr* next, const float* d_prev_xy, float* d_next_xy,
                       uint8_t* d_status, int32_t* d_track_status, int n, int use_initial, int max_iter,
                       double eps, double min_eig);
/* The same launch on a stream of the CALLER instead of the context's own (cuda_stream: a cudaStream_t of the same device). For pipelines
 * that keep the tracker and the filter on ONE stream, so that the optical flow of a frame, its visual updates and the next propagation
 * follow each other without cross-stream events, while the pyramid builds keep the context's stream. The caller orders the call
 * behind the builds of both pyramids (an event recorded on hv_ctx_stream(ctx)) and the next build of either pyramid behind this call.
 * d_init_xy (n x 2, may be NULL = start at d_prev_xy): the predicted end points (OPTFLOW_USE_INITIAL_FLOW) are READ from there and the
 * results written to d_next_xy -- a predictor's output buffer is used as it is, no copy into the result buffer first. */
int hv_lk_track_device_on_stream(hv_ctx* ctx, void* cuda_stream, hv_pyr* prev, hv_pyr* next, const float* d_prev_xy, const float* d_init_xy,
                                 float* d_next_xy, uint8_t* d_status, int32_t* d_track_status, int n, int max_iter, double eps, double min_eig);
/* Several independent LK calls (e.g. one per stream) in one launch; device pointers. */
typedef struct hv_lk_job {
    hv_pyr* prev; hv_pyr* next;
    const float* d_prev_xy; float* d_next_xy; uint8_t* d_status; int32_t* d_track_status;
    int n; int use_initial;
} hv_lk_job;
int hv_lk_track_batch_device(hv_ctx* ctx, const hv_lk_job* jobs, int njobs, int max_iter, double eps, double min_eig);

/* ---------------------------------------------------------------- corner detection (SURVEY.md 8(f) N2) ---- */
/* Device part of tracker::FeatureDetector::detect on CPU images (src/tracker/feature_detector.cpp:566-682, the default "GPU-GFTT"
 * detector without OpenGL images): CpuCornerResponse = cv::cornerMinEigenVal(gray, block_size, 3) (feature_detector.cpp:281-310,
 * OCV/imgproc/src/corner.cpp:238-320) and CollectMax::cpuImplementation (feature_detector.cpp:393-417: the best response of every
 * cell x cell block, x GAIN 16, kept if > min_response), on the level-0 gray image of `pyr`, which hv_pyr_build has already put into
 * HBM. cell = the detector's block size (32 for tracker.gfttMinDistance >= 32, feature_detector.cpp:425-433), block_size =
 * tracker.gfttBlockSize (3), min_response = tracker.gfttMinResponse.
 *   kp    (w / cell) * (h / cell) x (x, y, response) float32 in row-major cell order; a cell without a qualifying pixel reports
 *         (0, 0, -1e10) exactly as the reference does. The sort by response, the reference's resize quirk and applyMinDistance
 *         (feature_detector.cpp:625-638) follow either on the host (hybvio_b200/host/cuda_feature_detector.cpp runs the reference's
 *         own code) or on the device (hv_gftt_select_device / hv_gftt_corners below).
 * hv_gftt_detect: host output, synchronises. hv_gftt_detect_device: device output, no synchronisation. */
int hv_gftt_cells(const hv_pyr* pyr, int cell, int* cells_x, int* cells_y);
int hv_gftt_detect(hv_ctx* ctx, hv_pyr* pyr, int block_size, int cell, float min_response, float* kp);
int hv_gftt_detect_device(hv_ctx* ctx, hv_pyr* pyr, int block_size, int cell, float min_response, float* d_kp);

/* Corner selection: the rest of FeatureDetector::detect after CollectMax (feature_detector.cpp:625-638) on the device --
 * std::stable_sort of the key points by response (descending), the `corners.resize(n)` + push_back quirk (n points at (0, 0) in front
 * of the sorted ones), and, when mask_radius > 0, applyMinDistance (src/tracker/feature_detector_legacy.cpp): in list order a point is
 * kept iff no previous corner and no point kept before it lies within the radius ((c.x - p.x)^2 + (c.y - p.y)^2 < (float)(r * r),
 * fp32), stopping once max_tracks points are kept. mask_radius <= 0 returns all 2 nkp points and does not apply max_tracks.
 * Bit-identical to the reference's list for any key points without NaN responses.
 *   kp        nkp x (x, y, response) float32, as hv_gftt_detect(_device) writes them
 *   prev_xy   nprev x (x, y) float32: the corners already tracked (prevCorners)
 *   corners   capacity x (x, y) float32: the first *count entries are the list; slots [count, capacity) are set to
 *             (HV_CORNER_NONE, HV_CORNER_NONE), which hv_subpix_refine_device leaves unchanged (outside the image) and hv_lk_track_device
 *             reports as status 0 / FLOW_OUT_OF_RANGE, so a device pipeline can run both over `capacity` without reading the count.
 * capacity must hold the worst case: mask_radius > 0 ? min(max_tracks, 2 nkp) : 2 nkp.
 * Errors, before anything is launched: HV_ERR_INVALID for a NULL context / pyramid / buffer (kp and prev_xy may be NULL when their
 * count is 0), a pyramid of another context, nkp < 0, nprev < 0, max_tracks < 1 or a capacity below the worst case;
 * HV_ERR_UNSUPPORTED for more than 16384 key points (one CTA sorts them in shared memory: 1280 x 720 at cell 8 is 14400) or a
 * mask_radius above 46340 (r * r overflows the reference's int).
 * hv_gftt_select_device: device buffers, asynchronous, one launch (nkp = 0 writes count 0 and the padding only); composes on the
 * context's stream as hv_gftt_detect_device -> hv_gftt_select_device -> hv_subpix_refine_device -> hv_lk_track_device.
 * hv_gftt_corners: hv_gftt_detect + selection on the level-0 image of pyr with host prev_xy / corners / count and ONE synchronisation;
 * the key points stay in a device buffer of the context. nkp = 0 (image smaller than a cell) launches nothing. */
#define HV_CORNER_NONE (-1.0e6f)
int hv_gftt_select_device(hv_ctx* ctx, const float* d_kp, int nkp, const float* d_prev_xy, int nprev, int mask_radius, int max_tracks,
                          float* d_corners, int capacity, int* d_count);
int hv_gftt_corners(hv_ctx* ctx, hv_pyr* pyr, int block_size, int cell, float min_response, const float* prev_xy, int nprev,
                    int mask_radius, int max_tracks, float* corners, int capacity, int* count);

/* ---------------------------------------------------------------- sub-pixel corner refinement --------------- */
/* cv::cornerSubPix(level 0 of pyr, xy, Size(win_w, win_h), Size(zero_w, zero_h), TermCriteria(criteria_type, max_count, epsilon))
 * (OCV/imgproc/src/cornersubpix.cpp): the SubPixelAdjuster step of the reference's detection (src/tracker/image.cpp:76-79) on the
 * level-0 image that hv_pyr_build / hv_pyr_build_batch / hv_ingest_frame has already put into HBM. criteria_type: 1 COUNT, 2 EPS,
 * 3 both (cv::TermCriteria values). Bit-identical to cv::cornerSubPix built without IPP.
 *   xy        n x (x, y) float32, refined in place
 * Errors: HV_ERR_UNSUPPORTED for a half-window outside 1..15 on either axis; HV_ERR_INVALID for NULL arguments, a pyramid of another
 * context, or an image smaller than (2 win_w + 5) x (2 win_h + 5). hv_subpix_refine also returns HV_ERR_INVALID, before anything is
 * launched, for a corner outside [0, w) x [0, h) (cv::cornerSubPix asserts); hv_subpix_refine_device cannot inspect its input and
 * leaves such a corner unchanged. n = 0 launches nothing. */
int hv_subpix_refine(hv_ctx* ctx, hv_pyr* pyr, float* xy, int n, int win_w, int win_h, int zero_w, int zero_h,
                     int criteria_type, int max_count, double epsilon);          /* host xy in/out, synchronises */
int hv_subpix_refine_device(hv_ctx* ctx, hv_pyr* pyr, float* d_xy, int n, int win_w, int win_h, int zero_w, int zero_h,
                            int criteria_type, int max_count, double epsilon);   /* device xy, asynchronous */

/* ---------------------------------------------------------------- the new-corner step of many sessions -------- */
/* hv_gftt_detect_device, hv_gftt_select_device and hv_subpix_refine_device for up to HV_CORNER_BATCH_MAX independent lists (one per
 * session sharing the context) in ONE launch each: every job's outputs are bit-identical to the per-session call's. Device buffers,
 * asynchronous, on the context's stream; composes as
 *   hv_gftt_detect_batch_device -> hv_gftt_select_batch_device -> hv_subpix_refine_batch_device -> hv_lk_track_batch_device
 * (the stereo LK over every job's d_corners and capacity: one launch per 8 jobs). The parameters that shape a launch
 * (block size, cell, response threshold; the sub-pixel window, zero zone and criteria) are the batch's; the rest is per job.
 *   pyr          detect / refine: level 0 is the frame; pyramids may differ in size and pitch (select does not read it)
 *   d_kp, nkp    (x, y, response) per cell: detect writes hv_gftt_cells' cells_x * cells_y of them (nkp unused), select reads nkp
 *   d_prev_xy, nprev, mask_radius, max_tracks, d_corners, capacity, d_count: as hv_gftt_select_device (d_corners padded with
 *                HV_CORNER_NONE up to capacity)
 * Errors, for every job and before anything is launched: HV_ERR_INVALID for njobs outside 1..HV_CORNER_BATCH_MAX, a NULL context / jobs /
 * pyramid / buffer (d_kp, d_prev_xy, d_xy may be NULL when their count is 0; select's d_kp is never written), a pyramid of another
 * context, a negative count, max_tracks < 1, a capacity below the worst case, an image smaller than the sub-pixel window needs, or more
 * than 2^31 - 1 points in a refine batch; HV_ERR_UNSUPPORTED for what the per-session calls refuse as such (block size other than 3, cell
 * outside 2..32, more than 16384 key points in a job, a mask_radius above 46340, a half-window outside 1..15).
 * Each call is one launch (ctx's launch count + 1); a detect batch in which no image holds a cell and a refine batch without points
 * launch nothing. One session alone is served as well by the per-session calls (DESIGN.md 4.6 has the measured times). */
#define HV_CORNER_BATCH_MAX 64
typedef struct hv_corner_job {
    hv_pyr* pyr;
    float* d_kp; int nkp;
    const float* d_prev_xy; int nprev;
    int mask_radius, max_tracks;
    float* d_corners; int capacity;
    int* d_count;
} hv_corner_job;
int hv_gftt_detect_batch_device(hv_ctx* ctx, const hv_corner_job* jobs, int njobs, int block_size, int cell, float min_response);
int hv_gftt_select_batch_device(hv_ctx* ctx, const hv_corner_job* jobs, int njobs);
/* d_xy: n x (x, y) float32 on level 0 of pyr, refined in place (a point outside the image stays as it is, HV_CORNER_NONE padding too) */
typedef struct hv_subpix_job { hv_pyr* pyr; float* d_xy; int n; } hv_subpix_job;
int hv_subpix_refine_batch_device(hv_ctx* ctx, const hv_subpix_job* jobs, int njobs, int win_w, int win_h, int zero_w, int zero_h,
                                  int criteria_type, int max_count, double epsilon);

/* ---------------------------------------------------------------- FAST corner detection ----------------------- */
/* cv::FAST(level 0 of pyr, keypoints, threshold, nonmax, FastFeatureDetector::TYPE_9_16) (OCV/features2d/src/fast.cpp, fast_score.cpp):
 * the detector the reference's FeatureDetector::build hands out for featureDetector = FAST (src/tracker/feature_detector_legacy.cpp;
 * how that adapter post-processes the keypoints is not restated here), on the level-0 image that hv_pyr_build / hv_pyr_build_batch /
 * hv_ingest_frame(s) has already put into HBM. threshold is clamped to [0, 255] as FAST_t clamps it; nonmax != 0 keeps a corner only when
 * its score is strictly above its 8 neighbours'. Bit-identical to cv::FAST built without or with IPP for thresholds in [0, 255].
 *   xy        capacity x (x, y) float32: the keypoints in OpenCV's order (rows top to bottom, columns left to right); slots
 *             [count, capacity) are set to (HV_CORNER_NONE, HV_CORNER_NONE), so hv_subpix_refine_device and hv_lk_track_device can
 *             run over `capacity` without the count reaching the host (as with hv_gftt_select_device)
 *   response  capacity x float32 or NULL: the keypoint's score with suppression (cornerScore<16>), 0 without it (the KeyPoint
 *             response cv::FAST reports); 0 in the slots [count, capacity)
 *   count     the full count, which may exceed capacity: only the first `capacity` keypoints are written
 * Errors, before anything is launched (buffers and the context's launch count untouched): HV_ERR_INVALID for a NULL context / pyramid /
 * count, a NULL xy with capacity > 0, a pyramid of another context or a negative capacity.
 * Every call is two launches (ctx's launch count + 2); an image smaller than 7 x 7 yields count 0. */
int hv_fast_detect(hv_ctx* ctx, hv_pyr* pyr, int threshold, int nonmax, float* xy, float* response, int capacity, int* count);   /* host, synchronises */
int hv_fast_detect_device(hv_ctx* ctx, hv_pyr* pyr, int threshold, int nonmax, float* d_xy, float* d_response, int capacity,
                          int* d_count);                                                                             /* device, asynchronous */
/* hv_fast_detect_device for up to HV_CORNER_BATCH_MAX pyramids (one per session sharing the context) in the two launches of one call:
 * every job's outputs are bit-identical to the per-frame call's. Pyramids may differ in size and pitch; threshold and nonmax are the
 * batch's. Errors as hv_fast_detect_device's for every job, and HV_ERR_INVALID for a NULL jobs array or njobs outside
 * 1..HV_CORNER_BATCH_MAX, all before anything is launched. */
typedef struct hv_fast_job { hv_pyr* pyr; float* d_xy; float* d_response; int capacity; int* d_count; } hv_fast_job;
int hv_fast_detect_batch_device(hv_ctx* ctx, const hv_fast_job* jobs, int njobs, int threshold, int nonmax);

/* ---------------------------------------------------------------- Shi-Tomasi corner detection ----------------- */
/* cv::goodFeaturesToTrack(level 0 of pyr, corners, max_corners, quality_level, min_distance, mask, cornersQuality, block_size = 3,
 * gradientSize = 3, useHarrisDetector = false) (OCV/imgproc/src/featureselect.cpp, the CPU path): the primitive of the reference's
 * featureDetector = GFTT setting (how its legacy detector post-processes the list is not restated here), on the level-0 image that
 * hv_pyr_build / hv_pyr_build_batch / hv_ingest_frame(s) has already put into HBM. Not GPU-GFTT's response (hv_gftt_*): this one is
 * cv::cornerMinEigenVal's, bit for bit. In order: the minimum-eigenvalue response; maxVal = its maximum over the mask's non-zero pixels
 * (0 when the mask selects none); the response kept where it is > (float)(maxVal * quality_level); the candidates are the pixels of
 * [1, w - 1) x [1, h - 1) under the mask whose kept response is non-zero and the maximum of its 3 x 3 neighbourhood; they are listed by
 * response, descending, ties by descending pixel address (y w + x); with min_distance >= 1 a candidate is dropped when a corner kept
 * before it lies at (float)dx^2 + (float)dy^2 < min_distance^2; the list stops at max_corners. Bit-identical to cv::goodFeaturesToTrack
 * built without IPP and run on its baseline code path (cv::setUseOptimized(false)); DESIGN.md 4.10 says what the other paths change.
 *   mask      NULL or w x h u8 with row stride mask_stride bytes (host memory for hv_good_features, device memory otherwise)
 *   xy        capacity x (x, y) float32, integer-valued: the list; slots [count, capacity) are set to (HV_CORNER_NONE, HV_CORNER_NONE), so
 *             hv_subpix_refine_device and hv_lk_track_device can run over `capacity` without the count reaching the host
 *   response  capacity x float32 or NULL: the corner's response (OpenCV's cornersQuality); 0 in the slots [count, capacity)
 *   count     the list's length, at most max_corners
 * Errors, before anything is launched (buffers and the context's launch count untouched): HV_ERR_INVALID for a NULL context / pyramid /
 * xy / count, a pyramid of another context, capacity < max_corners, quality_level <= 0 or NaN, min_distance < 0 or not finite, or a mask stride
 * below the width; HV_ERR_UNSUPPORTED for block_size other than 3 or max_corners < 1 (OpenCV's "no limit").
 * Every call is three launches (ctx's launch count + 3) whatever the image holds; an image smaller than 3 x 3 yields count 0. The
 * response map, the candidate keys (8 bytes per interior pixel) and the min-distance grid live in scratch memory of the context, which
 * only grows. */
int hv_good_features(hv_ctx* ctx, hv_pyr* pyr, int block_size, int max_corners, double quality_level, double min_distance,
                     const uint8_t* mask, size_t mask_stride, float* xy, float* response, int capacity, int* count);      /* host, synchronises */
int hv_good_features_device(hv_ctx* ctx, hv_pyr* pyr, int block_size, int max_corners, double quality_level, double min_distance,
                            const uint8_t* d_mask, size_t mask_stride, float* d_xy, float* d_response, int capacity, int* d_count);
/* hv_good_features_device for up to HV_CORNER_BATCH_MAX pyramids (one per session sharing the context) in the three launches of one
 * call: every job's outputs are bit-identical to the per-frame call's. Pyramids may differ in size and pitch; max_corners, the mask and
 * the outputs are per job, block_size, quality_level and min_distance the batch's. Errors as hv_good_features_device's for every job,
 * and HV_ERR_INVALID for a NULL jobs array or njobs outside 1..HV_CORNER_BATCH_MAX, all before anything is launched. */
typedef struct hv_good_features_job {
    hv_pyr* pyr; int max_corners;
    const uint8_t* d_mask; size_t mask_stride;
    float* d_xy; float* d_response; int capacity;
    int* d_count;
} hv_good_features_job;
int hv_good_features_batch_device(hv_ctx* ctx, const hv_good_features_job* jobs, int njobs, int block_size, double quality_level,
                                  double min_distance);

/* ---------------------------------------------------------------- essential-matrix RANSAC (SURVEY.md 8(f) N3) -- */
/* cv::findEssentialMat(xy1[used], xy2[used], K, RANSAC, prob, threshold, max_iters, mask) (OCV/calib3d/src/five-point.cpp, ptsetreg.cpp):
 * the five-point RANSAC that the reference's RANSAC-5 stage is built on (how its modified copy differs from OpenCV is not restated here),
 * K = [[fx, 0, cx], [0, fy, cy], [0, 0, 1]]. The used points are those with status != 0 (all n when status is NULL), in index order; m is
 * their count. RANSAC replays OpenCV's: cv::RNG seeded with ~0 draws the subsets, a count above max(best, 4) wins, the iteration bound
 * shrinks through RANSACUpdateNumIters, an error is an inlier when (float)Sampson <= (float)((threshold / ((fx + fy) / 2))^2).
 * The five-point solver is this library's own (DESIGN.md 4.11): the same essential matrices as OpenCV's up to rounding, the solutions
 * of one subset in ascending order of their hidden variable. Where two solutions of one subset reach the same winning inlier count, OpenCV
 * keeps the first in its own root order, which is not restated, so its E (rarely its mask) can then be the other one.
 *   xy1, xy2  n x (x, y) float32: the correspondences (the layout the LK calls write)
 *   status    n x u8 or NULL; LK's status over a padded capacity (HV_CORNER_NONE slots report 0) can be passed as it is
 *   E         10 column-major fp64 3 x 3 slots: m < 5: none; m == 5: every solution of the five points (nsol <= 10);
 *             m > 5: the best one (nsol = 1), or none (nsol = 0) where OpenCV returns none. Slots [nsol, 10) are 0.
 *   mask      n x u8: 1 for the used points that are inliers of the result (m == 5: the five points when nsol > 0), 0 elsewhere
 *   inliers   the number of ones in mask
 * max_iters <= 0 runs one iteration, as OpenCV does; threshold may be any value OpenCV accepts (it is squared; NaN finds no inlier).
 * Errors, before anything is launched (buffers and the context's launch count untouched): HV_ERR_INVALID for a NULL context / E / nsol /
 * inliers, a NULL xy1 / xy2 / mask with n > 0, n < 0, or prob outside (0, 1) or NaN (what cv::findEssentialMat 4.13 refuses);
 * HV_ERR_UNSUPPORTED for n above HV_ESSENTIAL_MAX_POINTS, max_iters above HV_ESSENTIAL_MAX_ITERS, and intrinsics that are not finite or
 * have a zero focal length (OpenCV accepts them and returns NaN-laden results).
 * Every call is one launch (ctx's launch count + 1) whatever the data holds. The normalised points and their indices live in scratch
 * memory of the context (36 bytes per point), which only grows. */
#define HV_ESSENTIAL_MAX_POINTS 4096
#define HV_ESSENTIAL_MAX_ITERS 4096
int hv_find_essential(hv_ctx* ctx, const float* xy1, const float* xy2, const uint8_t* status, int n, double fx, double fy, double cx,
                      double cy, double prob, double threshold, int max_iters, double* E, int* nsol, uint8_t* mask, int* inliers); /* host, synchronises */
int hv_find_essential_device(hv_ctx* ctx, const float* d_xy1, const float* d_xy2, const uint8_t* d_status, int n, double fx, double fy,
                             double cx, double cy, double prob, double threshold, int max_iters, double* d_E, int* d_nsol, uint8_t* d_mask,
                             int* d_inliers);                                                                      /* device, asynchronous */
/* hv_find_essential_device for up to HV_ESSENTIAL_BATCH_MAX jobs (one per session sharing the context) in the one launch of one call:
 * every job's outputs are bit-identical to the per-call function's. Points, status, n, intrinsics and outputs are per job; prob,
 * threshold and max_iters the batch's. Errors as hv_find_essential_device's for every job, and HV_ERR_INVALID for a NULL jobs array or
 * njobs outside 1..HV_ESSENTIAL_BATCH_MAX, all before anything is launched. */
#define HV_ESSENTIAL_BATCH_MAX 64
typedef struct hv_essential_job {
    const float* d_xy1; const float* d_xy2; const uint8_t* d_status;
    int n;
    double fx, fy, cx, cy;
    double* d_E; int* d_nsol; uint8_t* d_mask; int* d_inliers;
} hv_essential_job;
int hv_find_essential_batch_device(hv_ctx* ctx, const hv_essential_job* jobs, int njobs, double prob, double threshold, int max_iters);

/* ---------------------------------------------------------------- relative pose from E (SURVEY.md 8(f) N3) -- */
/* cv::recoverPose(E, xy1, xy2, K, R, t, distance_thresh, mask) (OCV/calib3d/src/five-point.cpp): decomposeEssentialMat's four
 * candidates [R1 | t], [R2 | t], [R1 | -t], [R2 | -t]; every point triangulated (DLT) under each; a point is good for a candidate when
 * its depth in both cameras is positive and below distance_thresh, and mask_in (if any) is non-zero there; the candidate with the most
 * good points wins, ties going to the first in that order, as in OpenCV. K = [[fx, 0, cx], [0, fy, cy], [0, 0, 1]]. Both SVDs are this
 * library's own (DESIGN.md 4.12), so where two candidates tie at the winning count, OpenCV's choice between them (its SVD's sign
 * conventions) can be the other one; wherever one candidate wins alone the result is OpenCV's.
 *   E         column-major fp64 3 x 3 (host call: one matrix). d_nsol (device calls) NULL: d_E is one matrix; otherwise the count
 *             hv_find_essential_device wrote: 0 gives good 0, a zero mask and R = t = 0; above 1 the first slot is used, which is
 *             cv::recoverPose(E[0:3]) (OpenCV refuses the stacked matrix)
 *   xy1, xy2  n x (x, y) float32, as hv_find_essential takes them; every point is triangulated
 *   mask_in   n x u8 or NULL (every point used); mask_out n x u8: 1 where the point is good for the winner (0 where mask_in is 0);
 *             mask_out may be mask_in, so hv_find_essential_device's d_mask can be refined in place
 *   R, t      the winner, column-major fp64 3 x 3 and 3; good its count
 * distance_thresh may be any value OpenCV accepts (50 is its default); NaN passes no point.
 * Errors, before anything is launched (buffers and the context's launch count untouched): HV_ERR_INVALID for a NULL context / E / R /
 * t / good, a NULL xy1 / xy2 / mask_out with n > 0, n < 0; HV_ERR_UNSUPPORTED for n above HV_ESSENTIAL_MAX_POINTS and intrinsics that
 * are not finite or have a zero focal length, and (host call) an E that is not finite. Every call is one launch. */
int hv_recover_pose(hv_ctx* ctx, const double* E, const float* xy1, const float* xy2, const uint8_t* mask_in, int n, double fx, double fy,
                    double cx, double cy, double distance_thresh, double* R, double* t, uint8_t* mask_out, int* good); /* host, synchronises */
int hv_recover_pose_device(hv_ctx* ctx, const double* d_E, const int* d_nsol, const float* d_xy1, const float* d_xy2,
                           const uint8_t* d_mask_in, int n, double fx, double fy, double cx, double cy, double distance_thresh, double* d_R,
                           double* d_t, uint8_t* d_mask_out, int* d_good);                                   /* device, asynchronous */
/* hv_recover_pose_device for 1..HV_ESSENTIAL_BATCH_MAX jobs in the one launch of one call: every job's outputs are bit-identical to the
 * per-call function's. Everything but distance_thresh is per job. Errors as hv_recover_pose_device's for every job, and HV_ERR_INVALID
 * for a NULL jobs array or njobs outside 1..HV_ESSENTIAL_BATCH_MAX, all before anything is launched. */
typedef struct hv_pose_job {
    const double* d_E; const int* d_nsol;
    const float* d_xy1; const float* d_xy2; const uint8_t* d_mask_in;
    int n;
    double fx, fy, cx, cy;
    double* d_R; double* d_t; uint8_t* d_mask_out; int* d_good;
} hv_pose_job;
int hv_recover_pose_batch_device(hv_ctx* ctx, const hv_pose_job* jobs, int njobs, double distance_thresh);

/* ---------------------------------------------------------------- frame ingest (SURVEY.md 8(f) N4) -------- */
/* Device part of tracker::Image::Factory::build / buildStereo (src/tracker/image.cpp:243-308): colour -> gray
 * (accelerated-arrays pixelwiseAffine, image.cpp:360-366) and undistortion / rectification (UndistorterImplementation::undistort,
 * src/tracker/undistorter.cpp:77-118), with the result written straight into level 0 of the frame's pyramid, followed by the fused
 * pyramid kernel -- the frame crosses PCIe once, as it arrives.
 *   hv_remap_entry: per OUTPUT pixel the source position the reference's cameras map it to, as undistorter.cpp:93-94 forms it:
 *   x0 = floor(px), y0 = floor(py), xfrac = (float)(px - x0), yfrac = (float)(py - y0); x0 = HV_REMAP_INVALID_X0 where pixelToRay /
 *   rayToPixel fail or (px, py) lies outside [0, w) x [0, h). The table belongs to a (rectified camera, original camera) pair and is
 *   computed once by the adapter with the reference's own Camera classes (hybvio_b200/host/cuda_undistorter.cpp).
 * hv_ingest_frame: src = HOST frame (w x h, `channels` interleaved 8-bit channels, row stride in bytes). channels > 1: gray =
 * sum_j coeff[j] * channel_j in the reference's fixed-point arithmetic (coeff NULL: 0.299, 0.587, 0.114, 0). table (device handle from
 * hv_ingest_set_remap) optional. dst: the pyramid to build from the ingested frame. gray_out (host, optional, w x h, tightly packed)
 * receives the ingested gray image (the tracker::Image keeps it on the host for cornerSubPix / SLAM); asynchronous like hv_pyr_build:
 * synchronise (hv_ctx_sync or any synchronising call) before reading it. */
#define HV_REMAP_INVALID_X0 (-32768)
typedef struct hv_remap_entry { int16_t x0, y0; float xfrac, yfrac; } hv_remap_entry;
typedef struct hv_ingest hv_ingest;
int hv_ingest_create(hv_ctx* ctx, int width, int height, hv_ingest** out);
int hv_ingest_destroy(hv_ingest* ing);
int hv_ingest_set_remap(hv_ingest* ing, const hv_remap_entry* table);     /* width * height entries, host; NULL removes the table */
int hv_ingest_frame(hv_ingest* ing, const uint8_t* src, size_t stride_bytes, int channels, const double* coeff, hv_pyr* dst, uint8_t* gray_out);
/* hv_ingest_frames: hv_ingest_frame for up to HV_INGEST_BATCH_MAX frames (a stereo pair, or the pairs of many sessions sharing the
 * context) with the launches of one. Every job leaves the same bytes as hv_ingest_frame(job.ing, job.src, ...) would: every level of
 * dst (gray and gradients) and gray_out. Asynchronous, on the context's stream.
 *   src_is_device != 0: every src is a device pointer, read in place (no copy; e.g. a frame decoded on the GPU). Otherwise every src is
 *     host memory, copied once into its own hv_ingest's staging buffer up to the last pixel (no byte past it), as hv_ingest_frame does;
 *     it must stay valid until the next synchronising call.
 *   Jobs that need colour conversion or a remap run in ceil(k / 64) launches of one kernel (k such jobs). Gray jobs without a table skip
 *   it, as hv_ingest_frame does: a host source is copied into level 0, a device source is read in place by the pyramid kernel, as in
 *   hv_pyr_build_batch(..., 1). The pyramids are then built with one pyramid launch per 32 frames of one level-0 size (pyramids of
 *   different depth share a launch). A rectified stereo pair takes 2 launches, and so do 16 such pairs of one size.
 * Errors, checked for every job before anything is copied or launched (a refused call leaves every pyramid and gray_out untouched and
 * the context's launch count unchanged): HV_ERR_INVALID for njobs outside 1..HV_INGEST_BATCH_MAX; a NULL jobs, ing, src or dst;
 * channels outside 1..4 or a stride below w * channels; an ing or dst of another context than jobs[0].ing, or a dst whose size differs
 * from its ing; the same hv_ingest twice (it has one staging buffer and one table) or the same pyramid twice; a device source whose
 * bytes [src, src + stride * (h - 1) + w * channels) overlap the memory of any job's pyramid (the call writes it while it reads the
 * source). */
#define HV_INGEST_BATCH_MAX 128            /* 64 stereo sessions, matching the 64-session corner and EKF batches */
typedef struct hv_ingest_job {
    hv_ingest* ing;                        /* size and remap table (may have none) */
    const uint8_t* src; size_t stride_bytes; int channels;
    const double* coeff;                   /* NULL: 0.299, 0.587, 0.114, 0 (as hv_ingest_frame) */
    hv_pyr* dst;
    uint8_t* gray_out;                     /* host, optional, w x h tightly packed */
} hv_ingest_job;
int hv_ingest_frames(const hv_ingest_job* jobs, int njobs, int src_is_device);

/* ---------------------------------------------------------------- EKF ----------------------------------- */
/* Replaces odometry::EKF / EKFImplementation (src/odometry/ekf.hpp:62-174, ekf.cpp). State m (N) and
 * covariance P (N x N) are fp64 and live in HBM; N = 20 + 7*trail + 3*map (ekf.cpp:156-158). */
typedef struct hv_ekf_params {          /* the odometry::Parameters fields EKFImplementation reads */
    int camera_trail_length;            /* odometry.cameraTrailLength */
    int hybrid_map_size;                /* odometry.hybridMapSize */
    double noise_scale;                 /* odometry.noiseScale (the EKF uses its square, ekf.cpp:154) */
    double gravity;                     /* odometry.gravity */
    double noise_initial_pos, noise_initial_vel, noise_initial_ori;
    double noise_initial_bga, noise_initial_baa, noise_initial_bat, noise_initial_sft;
    double noise_initial_pos_trail, noise_initial_ori_trail;
    double noise_process_acc, noise_process_gyro;
    double noise_process_baa, noise_process_baa_rev, noise_process_bga, noise_process_bga_rev;
    double augment_r, init_zupt_r, rotation_zupt_r;
} hv_ekf_params;
/* Fills `p` with the defaults of codegen/parameter_definitions.c. */
void hv_ekf_default_params(hv_ekf_params* p);

/* EKF::build (ekf.cpp:153-296, 1087-1092) */
int hv_ekf_create(hv_ctx* ctx, const hv_ekf_params* params, hv_ekf** out);
int hv_ekf_destroy(hv_ekf* ekf);
/* EKF::clone (ekf.cpp:1074-1079): device-to-device copy of m, P, Q and the host-side time bookkeeping */
int hv_ekf_clone(const hv_ekf* src, hv_ekf** out);
int hv_ekf_state_dim(const hv_ekf* ekf);                       /* getStateDim */
int hv_ekf_pose_count(const hv_ekf* ekf);                      /* getPoseCount = augmentCount + 1 */
double hv_ekf_platform_time(const hv_ekf* ekf);                /* getPlatformTime */
double hv_ekf_history_time(const hv_ekf* ekf, int i);          /* historyTime (ekf.cpp:556-562) */
int hv_ekf_was_stationary(const hv_ekf* ekf);                  /* getWasStationary */
int hv_ekf_set_first_sample_time(hv_ekf* ekf, double t);       /* setFirstSampleTime (ekf.cpp:1035-1041) */

/* setState / setStateCovariance / getState / getStateCovariance (ekf.cpp:950-981). NULL = skip. download
 * synchronises. */
int hv_ekf_upload(hv_ekf* ekf, const double* m, const double* P);
int hv_ekf_download(hv_ekf* ekf, double* m, double* P);
/* getInertialState / setInertialState (ekf.cpp:679-690): first 20 entries / top-left 20x20 block. */
int hv_ekf_download_inertial(hv_ekf* ekf, double* m20, double* P20x20);
int hv_ekf_set_inertial_state(hv_ekf* ekf, const double* m20, const double* P20x20);
int hv_ekf_set_process_noise(hv_ekf* ekf, const double* Q12x12);   /* setProcessNoise */
int hv_ekf_get_dydx(hv_ekf* ekf, double* dydx20x20);               /* getDydx's non-identity block (tests) */

int hv_ekf_initialize_orientation(hv_ekf* ekf, const double acc[3]);          /* ekf.cpp:299-317 */
/* predict (ekf.cpp:320-514): mean propagation, Jacobians and the structured covariance update all run on the
 * device; the host only keeps the sample-time bookkeeping (first sample / dt <= 0 are no-ops). Asynchronous. */
int hv_ekf_predict(hv_ekf* ekf, double t, const double gyro[3], const double acc[3]);
/* IMU samples are DEFERRED: consecutive predict() calls -- each optionally followed by normalize_quaternions(ekf, 1), as in
 * the reference's sample loop (src/odometry/backend.cpp:734-735) -- are queued on the host (up to max_samples, default and
 * maximum 16) and issued as ONE launch by the next call that needs the state, or by hv_ekf_flush. Results are identical
 * to issuing every sample on its own (max_samples = 1). Likewise hv_ekf_symmetrize directly followed by hv_ekf_augment
 * (backend.cpp:1267 -> 805) is one launch. */
int hv_ekf_flush(hv_ekf* ekf);
/* The 20 inertial states (position, velocity, orientation, biases: ekf.hpp:26-50) that the QUEUED IMU samples lead to, written to
 * d_mean20 (device, 20 doubles) by a small launch of its own on the context's stream -- the mean part of predict() alone, a quarter of
 * the full launch, which stays queued. For consumers that need the propagated pose but not the covariance: the optical-flow predictor
 * (src/odometry/backend.cpp:547-600 reads ekf->position() / orientation() and the pose trail, which predict() does not change), so that
 * the tracker can start while the covariance is still being propagated. Bit-identical to what the full launch leaves in the state. */
int hv_ekf_predicted_mean_device(hv_ekf* ekf, double* d_mean20);
/* The same into host memory (launch, 160-byte read-back, one synchronisation): what odometry::EKF::position() / orientation() / velocity()
 * cost behind a burst of predict() calls -- the flow predictor's reads -- instead of the full launch plus a read-back of the whole mean. */
int hv_ekf_predicted_mean(hv_ekf* ekf, double* mean20);
/* After this call the queued FULL launch (hv_ekf_flush, or whatever issues the queue next) goes to a stream of the library instead of the
 * context's stream, and the next call that touches the filter waits for it there: work the caller puts on the context's stream in between
 * without touching the filter -- the optical flow of a pipeline that keeps tracker and filter on one stream -- does not queue behind the
 * covariance propagation. (Not in throughput mode, HV_EKF_NO_PDL=1.) */
int hv_ekf_set_imu_batching(hv_ekf* ekf, int max_samples);

/* The fixed-H updates (ekf.cpp:573-677); rate limits and early-outs as in the reference. Asynchronous. */
int hv_ekf_update_zupt(hv_ekf* ekf, double r);
int hv_ekf_update_zupt_initialization(hv_ekf* ekf);
int hv_ekf_update_zrupt(hv_ekf* ekf, const double gyro[3]);
int hv_ekf_update_pseudo_velocity(hv_ekf* ekf, double default_speed, double r);
int hv_ekf_update_position(hv_ekf* ekf, const double pos[3], double r);
int hv_ekf_update_zero_height(hv_ekf* ekf, double r);
int hv_ekf_update_orientation(hv_ekf* ekf, const double q[4], double r);

/* visualTrackOutlierCheck (ekf.cpp:787-819). H is n x l column-major (host), f and y length n (host).
 * *vu_status: odometry::VuOutlierStatus (ekf.hpp:54-59) INLIER=0, NOT_COMPUTED=1, RMSE=2, CHI2=3.
 * *chi2 (optional) receives noiseScale * v' S^-1 v. Synchronises (the caller branches on the result,
 * src/odometry/backend.cpp:1158-1161). */
int hv_ekf_visual_check(hv_ekf* ekf, const double* H, int n, int l, const double* f, const double* y, double r,
                        double track_rmse_threshold, int* vu_status, double* chi2);
/* updateVisualTrack (ekf.cpp:829-844). Asynchronous. */
int hv_ekf_visual_update(hv_ekf* ekf, const double* H, int n, int l, const double* f, const double* y, double r);
/* Fused check + conditional update in one kernel and ONE host round trip: applies updateVisualTrack iff the
 * check returns INLIER, and (if m_out != NULL) returns the updated state mean, which the caller needs to
 * build the next track's H (backend.cpp:1054-1056). Equivalent to check followed by update. Synchronises. */
int hv_ekf_visual_check_update(hv_ekf* ekf, const double* H, int n, int l, const double* f, const double* y,
                               double r, double track_rmse_threshold, int* vu_status, double* chi2, double* m_out);
/* Device-resident variant of the two calls above (H, f, y already in HBM; result words written to
 * d_result[0] = status, d_result[1] = chi2 as doubles); mode: 0 = check only, 1 = update only,
 * 2 = check then update-if-inlier. Asynchronous. */
int hv_ekf_visual_device(hv_ekf* ekf, const double* d_H, int n, int l, const double* d_f, const double* d_y,
                         double r, double track_rmse_threshold, int mode, double* d_result);

/* Batch submission: executes `nops` EKF calls in order with ONE crossing of the language boundary (what
 * Session::process issues per frame: the IMU predicts, the per-track checks/updates, symmetrise, augment;
 * src/odometry/backend.cpp:716-867). Each op is exactly the single call of the same name. */
typedef enum hv_ekf_op_kind {
    HV_EKF_OP_PREDICT = 0,        /* t, gyro, acc */
    HV_EKF_OP_VISUAL = 1,         /* H, n, l, f, y, r, rmse_thr, mode (0 check, 1 update, 2 check+update-if-inlier) */
    HV_EKF_OP_SYMMETRIZE = 2,
    HV_EKF_OP_AUGMENT = 3,        /* index = discarded pose */
    HV_EKF_OP_UNAUGMENT = 4,
    HV_EKF_OP_NORMALIZE = 5       /* index = only_current */
} hv_ekf_op_kind;
typedef struct hv_ekf_op {
    int kind;
    int n, l, mode, index;
    double t, r, rmse_thr;
    double gyro[3], acc[3];
    const double* H; const double* f; const double* y;
} hv_ekf_op;
/* H/f/y are DEVICE pointers; fully asynchronous. Consecutive independent outlier checks (mode 0) are issued as one launch, one
 * cluster per measurement. The measurement inputs of a list are PREPARED inputs: the kernels read them while their predecessor on the
 * stream may still be running (programmatic dependent launch), so they must not be produced by work queued on this stream after that
 * predecessor. For H produced by the caller's own kernel right before the call use hv_ekf_visual_device, which reads its inputs only
 * after the dependency on all earlier work of the stream has been resolved. The inputs must stay valid until hv_ctx_sync or
 * hv_ekf_run_device_results has returned (synchronising the context's STREAM alone is not enough, see below). */
int hv_ekf_run_device(hv_ekf* ekf, const hv_ekf_op* ops, int nops);
/* What the VISUAL ops of the most recent hv_ekf_run_device list decided: VuOutlierStatus / chi2 into vu_status[i] / chi2[i] for the ops
 * [0, nops) of that list (entries of other ops untouched; lists of up to 256 ops report). The list itself returns nothing and does not
 * wait: a run of outlier checks that is followed by the pose augmentation (the end of a frame, backend.cpp:1012-1270) is issued on a side
 * stream of the library -- the checks only read the state and the augmentation writes second buffers that are swapped in -- so that
 * the augmentation, the next IMU burst and the next visual updates do not queue behind them. This call waits for all of it. */
int hv_ekf_run_device_results(hv_ekf* ekf, int nops, int* vu_status, double* chi2);
/* H/f/y are HOST pointers; every VISUAL op with mode 0 or 2 returns its VuOutlierStatus / chi2 into
 * vu_status[i] / chi2[i] (arrays of length nops, entries of other ops untouched) -- i.e. each such op is a host
 * round trip, as in the reference interface. m_out (optional, N doubles) receives the final state mean. */
int hv_ekf_run_host(hv_ekf* ekf, const hv_ekf_op* ops, int nops, int* vu_status, double* chi2, double* m_out);

/* Many independent filters of ONE context stepped together (several sessions per process): for every i, the effect of
 * hv_ekf_run_device(ekfs[i], ops[i], nops[i]), called for each i in turn -- m, P, the pose count, the time bookkeeping and the result
 * words hv_ekf_run_device_results(ekfs[i], ...) returns afterwards are bit-identical -- with the launches of one filter: each list is
 * cut into steps (an IMU burst; one visual update; a run of outlier checks, with the augmentation that follows them as one more
 * cluster; an augmentation), and step k of every filter goes into one launch per kernel. Asynchronous, on the context's stream; never
 * on the library's side stream (throughput-mode stream policy); HV_EKF_NO_PDL keeps its meaning. H, f, y are DEVICE pointers and
 * prepared inputs, as for hv_ekf_run_device. Work queued for a filter by earlier calls is issued first; IMU samples at the end of a
 * list stay queued, as with hv_ekf_run_device.
 * The lists may only hold the ops of a device-resident frame:
 *   - PREDICT, each optionally followed by NORMALIZE with a non-zero index that folds into the sample before it (bursts of up to
 *     hv_ekf_set_imu_batching samples, 16 by default; a longer run of PREDICTs takes several launches -- a NORMALIZE right after the
 *     sample that completes a burst, or after a PREDICT that adds no sample, would be a launch of its own and is refused);
 *   - VISUAL in modes 0, 1, 2 whose measurement fits the cluster kernel whole (n <= 84 at N = 160);
 *   - AUGMENT, or SYMMETRIZE directly followed by AUGMENT, where the augmentation fits the cluster kernel (N <= 200).
 * Refused before anything is issued, every filter untouched: HV_ERR_UNSUPPORTED for any other op (UNAUGMENT, a standalone SYMMETRIZE or
 * NORMALIZE, a measurement or augmentation that does not fit); HV_ERR_INVALID for NULL arrays, a NULL filter, list or measurement
 * pointer, count outside 1..HV_EKF_GROUP_MAX, filters of different contexts or state dimensions, a filter that appears twice, a bad
 * mode or shape, an unknown op kind or a discarded-pose index out of range. The caller falls back to per-filter calls.
 * The visual-update chains of a group (hv_ekf_visual_tracks) have their own group call, hv_ekf_group_visual_tracks, below. */
#define HV_EKF_GROUP_MAX 64
int hv_ekf_group_run_device(hv_ekf* const* ekfs, int count, const hv_ekf_op* const* ops, const int* nops);

int hv_ekf_augment(hv_ekf* ekf, int discarded_pose_index);     /* updateVisualPoseAugmentation (ekf.cpp:848-885) */
int hv_ekf_unaugment(hv_ekf* ekf);                             /* updateUndoAugmentation (ekf.cpp:888-903) */
int hv_ekf_symmetrize(hv_ekf* ekf);                            /* maintainPositiveSemiDefinite (ekf.cpp:1059-1067) */
int hv_ekf_normalize_quaternions(hv_ekf* ekf, int only_current);   /* ekf.cpp:1024-1032 */
int hv_ekf_translate_to(hv_ekf* ekf, const double pos[3]);     /* ekf.cpp:696-702 */
int hv_ekf_transform_to(hv_ekf* ekf, const double pos[3], const double q[4], int pose_index); /* ekf.cpp:704-758 */
int hv_ekf_insert_map_point(hv_ekf* ekf, int idx, const double pf[3]);   /* ekf.cpp:911-921 */
int hv_ekf_condition_on_last_pose(hv_ekf* ekf);                /* ekf.cpp:928-942 */
int hv_ekf_lock_biases(hv_ekf* ekf);                           /* ekf.cpp:944-947 */
/* ---- Per-track measurement model on the device (next hot-path row, SURVEY.md 8(f) N1) --------------------------------
 * What Session::trackerVisualUpdate computes on the host for every track before it can call the EKF
 * (src/odometry/backend.cpp:1050-1160): extractCameraPoseTrail (src/odometry/triangulation.cpp:65-103) ->
 * Triangulator::triangulate with derivatives (:120-407, two-view start :610-710) -> per-pose sum of the two cameras
 * (backend.cpp:1105-1116) -> prepareVisualUpdate(truncated) (:897-987). Here it runs on the device from the resident state
 * mean; H, f (and the measurement vector y = the observations) stay in HBM, where hv_ekf_visual_device / hv_ekf_run_device
 * read them, so H is neither built on nor uploaded from the host. */
typedef struct hv_camera_model {
    double imu_to_camera[16];            /* odometry::Parameters::imuToCamera, 4x4 column-major (Eigen) */
    double second_imu_to_camera[16];     /* ...::secondImuToCamera (ignored unless use_stereo) */
    int use_stereo;                      /* tracker.useStereo */
    int estimate_imu_camera_time_shift;  /* odometry.estimateImuCameraTimeShift */
    unsigned gauss_newton_iterations;    /* odometry.triangulationGaussNewtonIterations (10) */
    double convergence_threshold;        /* odometry.triangulationConvergenceThreshold (1e-2) */
    double convergence_r;                /* odometry.triangulationConvergenceR (11) */
    double rcond_threshold;              /* odometry.triangulationRcondThreshold (1e-8) */
    double min_dist, max_dist;           /* odometry.triangulationMinDist / MaxDist (0, 1e300): BAD_DEPTH gate, backend.cpp:1095-1098 */
} hv_camera_model;
void hv_camera_model_defaults(hv_camera_model* c);     /* the reference defaults above; the two matrices are zeroed */
int hv_ekf_set_camera_model(hv_ekf* ekf, const hv_camera_model* c);
#define HV_TRACK_MAX_POSES 21            /* pose-trail indices per track (cameraTrailLength 20 + the current pose) */
typedef struct hv_track_obs {
    int npose;                           /* 2 .. HV_TRACK_MAX_POSES */
    const int* pose_trail_index;         /* npose indices as EkfStateIndex::createTrackIndex gives them: 0 = current pose, k = trail slot k - 1 */
    const double* ip;                    /* normalised image points x,y: npose of the first camera [, npose of the second] */
    const double* velocities;            /* their velocities, same layout (TriangulationArgsIn::featureVelocities) */
} hv_track_obs;
typedef struct hv_track_model {
    int triangulator_status;             /* odometry::TriangulatorStatus (output.hpp:21-29): OK 0, BEHIND 2, BAD_COND 3, NO_CONVERGENCE 4, BAD_DEPTH 5, UNKNOWN_PROBLEM 6 */
    int prepare_vu_status;               /* odometry::PrepareVuStatus (output.hpp:15-19), -1 if triangulation failed */
    int rows, cols;                      /* of H: 2 n_obs x l (truncated at the last pose the track touches) */
    double pf[3], depth;                 /* triangulated point, |pf - first camera| */
    const double* d_H;                   /* DEVICE: rows x cols, column-major, ld = rows */
    const double* d_f;                   /* DEVICE: predicted observations, rows */
    const double* d_y;                   /* DEVICE: the observations, rows (the y of visualTrackOutlierCheck / updateVisualTrack) */
} hv_track_model;
/* All tracks are evaluated against the CURRENT state mean in one launch (one CTA per track); the device pointers in out[]
 * stay valid until the next call on this ekf. Synchronises (the caller branches on the statuses). */
int hv_ekf_track_models(hv_ekf* ekf, const hv_track_obs* tracks, int ntracks, hv_track_model* out);
/* visualTrackOutlierCheck (mode 0) / updateVisualTrack (mode 1) / check then update-if-inlier (mode 2) (ekf.cpp:787-844) on
 * the device-resident H, f, y of one track of the last hv_ekf_track_models call. Modes 0 and 2 return the VuOutlierStatus and
 * chi2 (one host round trip, like hv_ekf_visual_check); mode 1 is asynchronous. Note that an update changes the state: the
 * models of the other tracks of that call were evaluated against the state before it (as in the reference's batch mode,
 * backend.cpp:1170-1183; per-track mode re-evaluates the next track with a new hv_ekf_track_models call). */
int hv_ekf_visual_track(hv_ekf* ekf, const hv_track_model* t, double r, double track_rmse_threshold, int mode, int* vu_status,
                        double* chi2);
/* The per-track loop of Session::trackerVisualUpdate in per-track mode (src/odometry/backend.cpp:1012-1252) as ONE chain on the
 * stream, with the control flow on the device: for every track, in order,
 *     measurement model against the CURRENT state (the previous track's update included)
 *  -> visualTrackOutlierCheck(chi_outlier_r, track_rmse_threshold)       if the model is valid
 *  -> updateVisualTrack(visual_r)                                         if the check says INLIER,
 * and nothing more once max_successful_updates updates have been applied (backend.cpp:1240-1247). Check and update of a track
 * run as ONE kernel (H P and H P H' formed once, factorised with each of the two noise levels; HV_CHAIN_SEPARATE=1 in the
 * environment issues two gated launches instead), so a track costs two launches. Each kernel is gated by
 * words its predecessors wrote, so the host does not synchronise per track but once per `lookahead` tracks (0: once). The
 * caller applies its own pre-filters (track score, trackMinFrames, blacklist, maxVisualUpdates: backend.cpp:1020-1047, 1241)
 * by choosing which tracks to submit. Results are those of the per-track calls hv_ekf_track_models ->
 * hv_ekf_visual_track(mode 0) -> hv_ekf_visual_track(mode 1) issued track by track.
 * State sizes: a track whose measurement does not fit the cluster kernel whole (long trails, hybrid maps: at N = 202 tracks of more
 * than 71 rows, N = 301 more than 41, N = 400 more than 16) runs in its row-chunked form, still one kernel for check and update.
 * Every track of up to 84 rows (21 stereo poses) runs for N <= 424 (8-row tracks up to N = 432, 4-row up to 448); a chain with a track
 * beyond that is refused with HV_ERR_UNSUPPORTED before anything is issued, the filter state untouched.
 * Not covered: trackOutlierThresholdGrowthFactor != 1 (the thresholds are fixed for the chain), hybrid map-point tracks. */
typedef struct hv_visual_update_params {
    double chi_outlier_r;            /* r of the check: odometry.trackChiTestOutlierR / focal length (backend.cpp:996) */
    double track_rmse_threshold;     /* odometry.trackRmseThreshold / focal length (backend.cpp:995); < 0: off */
    double visual_r;                 /* r of the update: odometry.visualR / focal length (backend.cpp:997) */
    int max_successful_updates;      /* odometry.maxSuccessfulVisualUpdates; <= 0: unlimited */
    int lookahead;                   /* tracks issued per host synchronisation; 0 = all */
} hv_visual_update_params;
typedef struct hv_track_result {
    int triangulator_status;         /* odometry::TriangulatorStatus; -1: not attempted (enough successful updates before it) */
    int prepare_vu_status;           /* odometry::PrepareVuStatus, -1 if triangulation failed / not attempted */
    int outlier_status;              /* odometry::VuOutlierStatus (INLIER 0, NOT_COMPUTED 1, RMSE 2, CHI2 3) */
    int updated;                     /* 1: updateVisualTrack was applied with this track */
    double chi2, pf[3], depth;
} hv_track_result;
int hv_ekf_visual_tracks(hv_ekf* ekf, const hv_track_obs* tracks, int ntracks, const hv_visual_update_params* params,
                         hv_track_result* out, int* successful_updates);
/* The visual-update chains of many independent filters of ONE context (several sessions per process; the counterpart of
 * hv_ekf_group_run_device): for every i, the effect of hv_ekf_visual_tracks(ekfs[i], tracks[i], ntracks[i], &params[i], out[i],
 * &successful_updates[i]) -- m, P, the pose count, the hv_track_result records and the successful-update count are bit-identical,
 * lookahead included -- with the launches of one chain: step k is track k of every filter that still has tracks to issue, as one
 * launch of the model kernel (a CTA per filter), one of the cluster kernel (a cluster per filter: check + update) and, in a step where
 * a filter uses the separate form (chi_outlier_r < 0 or visual_r <= 0), one more for the updates of those filters. A group costs the
 * launches of its longest chain. The host synchronises once per `lookahead` steps for all filters together (with different lookaheads:
 * whenever a filter reaches the end of one of its windows); a filter with max_successful_updates reached at a synchronisation is not
 * issued further, and its later tracks get the records of tracks the per-filter call never issues. Synchronises before it returns;
 * HV_EKF_NO_PDL keeps its meaning. Work queued for a filter by earlier calls is issued first.
 * Per filter: ntracks[i] (0: the filter is left untouched, its count is 0; tracks[i] and out[i] may then be NULL), params[i] and the
 * camera model (mono or stereo) may differ. successful_updates: count entries, or NULL.
 * Refused before anything is issued, every filter untouched: HV_ERR_INVALID for NULL arrays, a NULL filter, a NULL tracks[i] / out[i]
 * where ntracks[i] > 0, a negative ntracks[i], count outside 1..HV_EKF_GROUP_MAX, filters of different contexts or state dimensions, a
 * filter that appears twice, a malformed track (as hv_ekf_track_models checks them); HV_ERR_STATE for a filter without
 * hv_ekf_set_camera_model; HV_ERR_UNSUPPORTED for a track whose measurement does not fit the cluster kernel whole (the group has no
 * row-chunked form: every track of up to 84 rows fits at N = 160 and at N = 62); the message names the filter and the track, and the
 * caller falls back to per-filter calls. An innovation covariance that is not positive definite in any filter returns HV_ERR_STATE after
 * every result has been written, as the per-filter call does; the message names the (first such) filter. A single filter is faster
 * through hv_ekf_visual_tracks (DESIGN.md 4.5b). */
int hv_ekf_group_visual_tracks(hv_ekf* const* ekfs, int count, const hv_track_obs* const* tracks, const int* ntracks,
                               const hv_visual_update_params* params, hv_track_result* const* out, int* successful_updates);
/* Test / debug: copies H (rows x cols), f (rows) and d pf / d (poses, t) (3 x (7 npose + 1), column-major, after the stereo
 * sum) of track `track` of the last hv_ekf_track_models call to the host; any pointer may be NULL. */
int hv_ekf_track_model_download(hv_ekf* ekf, int track, double* H, double* f, double* dpf);

/* Measurement aid (bench): repeats the kernel of the last hv_ekf_track_models call `reps` times between two CUDA events on the
 * context's stream and returns the average device time per launch in milliseconds. */
int hv_ekf_track_models_time(hv_ekf* ekf, int reps, float* ms_per_launch);
/* Debug: the 32 result words of the last update kernel ([0] status, [1] chi2, [2] flag, [8..] phase timestamps when
 * the library is built with -DHV_EKF_TIMING). */
int hv_ekf_debug_result_words(hv_ekf* ekf, double* out32);
/* Host wall time of the most recent hv_ekf_run_host list that had something to hand back: out4 = {issuing the list, waiting in its one
 * synchronisation, total} in microseconds and the number of ops (bench.py reports them next to `e2e`). */
int hv_ekf_debug_host_times(hv_ekf* ekf, double* out4);

#ifdef __cplusplus
}
#endif
#endif /* HYBVIO_B200_H_ */
