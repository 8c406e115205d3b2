// hybvio_b200 -- shared device-side types for the sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/hybvio_b200.h"     // the limits of the C ABI (HV_CORNER_BATCH_MAX, HV_ESSENTIAL_*, HV_PNP_*, ...)

#define HV_MAX_LEVELS 6      // pyrLKMaxLevel <= 5 (HybVIO default 3, codegen/parameter_definitions.c:334-344)
#define HV_PYR_TILE 64       // level-0 tile edge of the fused pyramid kernel; must be divisible by 2^maxLevel

// One pyramid level in HBM. Levels are stored UNPADDED (the reference pads every level by winSize on all
// sides, OCV/video/src/lkpyramid.cpp:761-808; here the reflect-101 / zero border is applied by index
// arithmetic in the LK kernel instead, which saves 0.79 MB of writes per 752x480 image).
struct HvLevel {
    uint8_t* gray;    // w x h, row pitch gpitch bytes (multiple of 4; level 0: w when w % 4 == 0, else / coarser levels: multiple of 128)
    short2*  deriv;   // w x h (Ix, Iy) Scharr x32, row pitch dpitch elements (multiple of 32 => 128 B)
    int w, h;
    int gpitch;
    int dpitch;
};

struct HvPyrDesc {
    HvLevel lv[HV_MAX_LEVELS];
    int nlevels;
    int win;
};

// BORDER_REFLECT_101 (OCV/core/src/copy.cpp:1136-1181)
__host__ __device__ __forceinline__ int hv_reflect101(int p, int len)
{
    if ((unsigned)p < (unsigned)len) return p;
    if (len == 1) return 0;
    do {
        if (p < 0) p = -p;
        else p = 2 * len - 2 - p;
    } while ((unsigned)p >= (unsigned)len);
    return p;
}

// Completion signal of a host-buffer launch whose results land in mapped pinned host memory: every CTA makes its results visible
// system-wide (__threadfence_system) and calls hv_signal_done; the last of the launch's `target` counts stores seq into *hostFlag,
// which the host polls instead of a D2H copy + stream synchronisation. hostFlag NULL: no signal.
struct HvDoneSignal {
    unsigned* counter;
    unsigned target, seq;
    volatile unsigned* hostFlag;
};

#if defined(__CUDACC__) || defined(HV_EMU)      // (a plain host compiler that reads the argument blocks has no device intrinsics)
__device__ __forceinline__ void hv_signal_done(const HvDoneSignal& d)
{
    const unsigned old = atomicAdd(d.counter, 1u);
    if (old + 1u == d.target) { __threadfence_system(); *d.hostFlag = d.seq; }
}
#endif

// ---- Lucas-Kanade launch description (lk.cu)
#define LK_WARPS_PER_CTA 4
#define LK_MAX_JOBS 8

struct LkJob {
    int prevIdx, nextIdx;       // pyramid descriptor indices
    int n;                      // number of features
    int useInitial;             // OPTFLOW_USE_INITIAL_FLOW
    const float2* prevPts;      // device
    float2* nextPts;            // device; in: initial guess (if useInitial), out: end point
    uint8_t* status;            // device; OpenCV status 1 = ok, 0 = failed
    int32_t* trackStatus;       // device, optional; tracker::Feature::Status (src/tracker/track.hpp:9-20)
    const float2* initPts;      // device, optional: the initial guess lives here instead of in nextPts (which is then only written)
};

struct LkLaunch {
    const HvPyrDesc* table;
    LkJob jobs[LK_MAX_JOBS];
    int njobs;
    int maxLevel;
    int maxIter;                // already clamped to [0,100]
    double eps2;                // already clamped and squared
    float minEig;
    HvDoneSignal done;          // host-buffer API (single job, CTA-per-feature kernel): one count per CTA
    int prefetch;               // CTA-per-feature kernel: request the search region of a level with cp.async before the template patch is loaded
};


// Kernel choice of hv_launch_lk: up to 640 features in a launch (one session) a CTA of 4 warps per feature (minimal latency; the
// only kernel that raises the host flag of the polled path), above that a warp per feature (throughput). Both produce identical bits.
inline bool hv_lk_uses_cta_kernel(long long totalFeatures) { return totalFeatures <= 640; }
cudaError_t hv_launch_lk(const LkLaunch& L, int win, cudaStream_t stream);

// ---- corner detection launch description (gftt.cu)
struct GfttArgs {
    const uint8_t* gray; int pitch, w, h;
    int cell;                 // bs
    float k0, k1;             // [1 2 1] * scale as the fp32 kernel OpenCV builds (k0 = 2 s, k1 = s)
    float minResponse;
    float* kp;                // cellsX * cellsY * (x, y, response * 16); may be mapped pinned host memory
    HvDoneSignal done;        // host-buffer API: one count per CTA
};

cudaError_t hv_launch_gftt(const GfttArgs& a, cudaStream_t stream);

// Batches of the corner step (detect, select, refine): one job per session, at most HV_CORNER_BATCH_MAX per launch. Every argument
// block travels as a __grid_constant__ kernel parameter (at most 32764 bytes on sm_90).
#define HV_KERNEL_PARAM_MAX 32764

// The job of CTA b in a flattened grid: the last j with first[j] <= b, where first[] is the prefix sum of the jobs' CTA counts (a job
// without CTAs repeats its successor's start) padded with the grid size up to HV_CORNER_BATCH_MAX. Six steps whatever the batch size.
__host__ __device__ __forceinline__ int hv_batch_job(const int* first, int b)
{
    int j = 0;
#pragma unroll
    for (int step = HV_CORNER_BATCH_MAX / 2; step > 0; step >>= 1)
        if (first[j + step] <= b) j += step;
    return j;
}
struct GfttBatchArgs {
    GfttArgs job[HV_CORNER_BATCH_MAX];        // done.hostFlag NULL
    int first[HV_CORNER_BATCH_MAX + 1];       // first CTA (cell) of job j in the flattened grid; first[njobs ..] = the grid
    int cellsX[HV_CORNER_BATCH_MAX];
};
static_assert(sizeof(GfttBatchArgs) <= HV_KERNEL_PARAM_MAX, "detect batch arguments exceed the kernel-parameter space");
cudaError_t hv_launch_gftt_batch(const GfttBatchArgs& b, int njobs, cudaStream_t stream);

// ---- corner selection launch description (gftt_select.cu): the detector's sort, resize quirk and applyMinDistance
#define HV_GFTT_SELECT_MAX_KP 16384   // key points per call: one CTA, the sort keys in opt-in shared memory (128 KB)
#define HV_GFTT_SELECT_MAX_RADIUS 46340   // mask_radius^2 still fits the reference's int product
#define HV_CORNER_NONE_F (-1.0e6f)    // padding slots [count, capacity) (HV_CORNER_NONE of the header)
struct GfttSelectArgs {
    const float* kp; int nkp;         // (x, y, response) per cell, as hv_launch_gftt writes them
    const float* prev; int nprev;     // previous corners (x, y)
    int maskRadius, maxTracks;
    float r2;                         // (float)(mask_radius * mask_radius), formed on the host as the reference does
    int pow2;                         // sort width: the smallest power of two >= nkp (>= 2)
    float* out; int capacity;         // (x, y) per slot; may be mapped pinned host memory
    int* count;                       // may be mapped pinned host memory
    HvDoneSignal done;        // host-buffer API: one count per CTA
};

cudaError_t hv_launch_gftt_select(const GfttSelectArgs& a, cudaStream_t stream);

struct GfttSelectBatchArgs {
    GfttSelectArgs job[HV_CORNER_BATCH_MAX];  // CTA j is list j; done.hostFlag NULL
};
static_assert(sizeof(GfttSelectBatchArgs) <= HV_KERNEL_PARAM_MAX, "select batch arguments exceed the kernel-parameter space");
// maxPow2: the largest job[j].pow2, which sizes the dynamic shared memory of every CTA
cudaError_t hv_launch_gftt_select_batch(const GfttSelectBatchArgs& b, int njobs, int maxPow2, cudaStream_t stream);

// ---- sub-pixel corner refinement launch description (subpix.cu)
#define HV_SUBPIX_MAX_HALF 15        // half-window per axis: a 31 x 31 window at most
struct SubpixArgs {
    const uint8_t* gray; int pitch, w, h;
    float2* xy; int n;                // refined in place; may be mapped pinned host memory
    int hw, hh;                       // half-window (win.width, win.height)
    int maxIters;                     // already clamped as cv::cornerSubPix does
    double eps2;                      // already clamped and squared
    float mask[(2 * HV_SUBPIX_MAX_HALF + 1) * (2 * HV_SUBPIX_MAX_HALF + 1)];    // (2 hh + 1) x (2 hw + 1), built on the host, zero zone applied
    HvDoneSignal done;                // host-buffer API: one count per CTA
};

cudaError_t hv_launch_subpix(const SubpixArgs& a, cudaStream_t stream);

struct SubpixJob { const uint8_t* gray; int pitch, w, h; float2* xy; int n; };
struct SubpixBatchArgs {
    SubpixArgs s;                             // window, criteria and mask of the whole batch (gray, xy, n and done unused)
    SubpixJob job[HV_CORNER_BATCH_MAX];
    int first[HV_CORNER_BATCH_MAX + 1];       // first CTA (point) of job j in the flattened grid; first[njobs ..] = the grid
};
static_assert(sizeof(SubpixBatchArgs) <= HV_KERNEL_PARAM_MAX, "sub-pixel batch arguments exceed the kernel-parameter space");
cudaError_t hv_launch_subpix_batch(const SubpixBatchArgs& b, int njobs, cudaStream_t stream);

// ---- FAST corner detection (fast.cu): cv::FAST, TYPE_9_16, on level 0
struct FastArgs {
    const uint8_t* gray; int pitch, w, h;
    int threshold;                    // already clamped to [0, 255]
    int nonmax;
    int tilesX, tilesY;               // ceil(w / 32) x ceil(h / 8) tiles
    unsigned* mask;                   // scratch: 8 tilesY x tilesX keypoint masks, row-major over (row, tile)
    int* tileCount;                   // scratch: tilesY x tilesX keypoint counts
    float2* xy; float* response;      // capacity slots each; response may be NULL
    int capacity;
    int* count;                       // the full count, which may exceed capacity
};
cudaError_t hv_launch_fast(const FastArgs& a, cudaStream_t stream);         // two launches: mark + count, then scan + scatter

struct FastBatchArgs {
    FastArgs job[HV_CORNER_BATCH_MAX];
    int firstTile[HV_CORNER_BATCH_MAX + 1];   // first CTA (tile) of job j in the mark grid; firstTile[njobs ..] = that grid
    int firstBand[HV_CORNER_BATCH_MAX + 1];   // first CTA (band of 8 rows) of job j in the scatter grid; firstBand[njobs ..] = that grid
};
static_assert(sizeof(FastBatchArgs) <= HV_KERNEL_PARAM_MAX, "FAST batch arguments exceed the kernel-parameter space");
cudaError_t hv_launch_fast_batch(const FastBatchArgs& b, int njobs, cudaStream_t stream);

// ---- Shi-Tomasi corner detection (good_features.cu): cv::goodFeaturesToTrack with the minimum-eigenvalue response, block size 3
#ifndef HV_GF_CHUNK                   // (a power of two; the emulator test builds with a small one to run many rounds on small images)
#define HV_GF_CHUNK 8192              // sorted keys per selection round: 64 KB of dynamic shared memory
#endif
struct GoodFeaturesArgs {
    const uint8_t* gray; int pitch, w, h;
    const uint8_t* mask; int maskPitch;   // NULL: no mask
    int tilesX, tilesY;               // ceil(w / 32) x ceil(h / 8) tiles
    int maxCorners;
    double quality;                   // qualityLevel
    double md2;                       // minDistance^2
    int useGrid;                      // minDistance >= 1: the greedy distance filter
    int cell, reach, gridW, gridH;    // its grid: cell side (at most one kept corner per cell), +-reach pixels searched, cells per axis
    float* eig;                       // scratch: w x h response map
    unsigned long long* keys;         // scratch: maxCand = max(1, (w - 2)(h - 2)) candidate keys
    int maxCand;
    int* grid;                        // scratch: gridW x gridH, the pixel index of the cell's kept corner or -1
    unsigned* maxWord;                // scratch: the masked maximum as order-preserving bits, 0: no pixel
    int* nCand;                       // scratch: the candidate count (maxWord and nCand are zeroed before the first launch)
    float2* xy; float* response;      // capacity slots each; response may be NULL
    int capacity;
    int* count;
};
cudaError_t hv_launch_good_features(const GoodFeaturesArgs& a, cudaStream_t stream);     // three launches: response, candidates, select

struct GoodFeaturesBatchArgs {
    GoodFeaturesArgs job[HV_CORNER_BATCH_MAX];
    int firstStrip[HV_CORNER_BATCH_MAX + 1];  // first CTA (32 columns) of job j in the response grid; firstStrip[njobs ..] = that grid
    int firstTile[HV_CORNER_BATCH_MAX + 1];   // first CTA (tile) of job j in the candidate grid; firstTile[njobs ..] = that grid
};
static_assert(sizeof(GoodFeaturesBatchArgs) <= HV_KERNEL_PARAM_MAX, "good-features batch arguments exceed the kernel-parameter space");
cudaError_t hv_launch_good_features_batch(const GoodFeaturesBatchArgs& b, int njobs, cudaStream_t stream);

// ---- essential-matrix RANSAC (essential.cu): cv::findEssentialMat(..., RANSAC, prob, threshold, maxIters) on the used points
struct EssentialArgs {
    const float2* xy1; const float2* xy2;
    const uint8_t* status;            // NULL: every point is used
    int n;
    double fx, fy, cx, cy;
    double* E;                        // 10 column-major 3 x 3 slots
    int* nsol; uint8_t* mask; int* inliers;
    double* q;                        // scratch: n normalised used points (x1, y1, x2, y2), 32-byte aligned
    int* idx;                         // scratch: their original indices
};
struct EssentialBatchArgs {
    EssentialArgs job[HV_ESSENTIAL_BATCH_MAX];
    double prob, threshold;
    int maxIters;
};
static_assert(sizeof(EssentialBatchArgs) <= HV_KERNEL_PARAM_MAX, "essential batch arguments exceed the kernel-parameter space");
cudaError_t hv_launch_essential(const EssentialBatchArgs& b, int njobs, cudaStream_t stream);     // one launch, one CTA per job

// ---- relative pose (pose.cu): cv::recoverPose(E, xy1, xy2, K, R, t, distanceThresh, mask), up to HV_ESSENTIAL_BATCH_MAX jobs
struct PoseArgs {
    const double* E;                  // column-major 3 x 3 slots; the first is used
    const int* nsol;                  // NULL: E is one matrix; *nsol == 0: no result (R, t, mask and good zero)
    const float2* xy1; const float2* xy2;
    const uint8_t* maskIn;            // NULL: every point is used
    int n;
    double fx, fy, cx, cy;
    double* R; double* t;             // column-major 3 x 3, 3
    uint8_t* maskOut; int* good;      // maskOut 0/1, may be maskIn
};
struct PoseBatchArgs {
    PoseArgs job[HV_ESSENTIAL_BATCH_MAX];
    double dist;
};
static_assert(sizeof(PoseBatchArgs) <= HV_KERNEL_PARAM_MAX, "pose batch arguments exceed the kernel-parameter space");
cudaError_t hv_launch_pose(const PoseBatchArgs& b, int njobs, cudaStream_t stream);     // one launch, one CTA per job

// ---- absolute-pose RANSAC (pnp.cu): cv::solvePnPRansac(..., SOLVEPNP_P3P) on the used points, up to HV_ESSENTIAL_BATCH_MAX jobs
struct PnpArgs {
    const float* xyz;                 // n x 3
    const float2* xy;
    const uint8_t* status;            // NULL: every point is used
    int n;
    double fx, fy, cx, cy;
    double* rvec; double* tvec;       // 3 each
    uint8_t* mask; int* inliers; int* ok;
    float* P; float2* Q; int* idx;    // scratch: the used points (world, image) and their original indices
    double* pws; double* us;          // scratch: EPnP's inliers (world, image after OpenCV's undistort round trip)
    double* al; double* pcs;          // scratch: their barycentric coordinates and camera points
};
struct PnpBatchArgs {
    PnpArgs job[HV_ESSENTIAL_BATCH_MAX];
    double confidence;
    float reprojError;
    int iterations;
};
static_assert(sizeof(PnpBatchArgs) <= HV_KERNEL_PARAM_MAX, "pnp batch arguments exceed the kernel-parameter space");
cudaError_t hv_launch_pnp(const PnpBatchArgs& b, int njobs, cudaStream_t stream);     // one launch, one CTA per job

// ---- two-view triangulation (triangulate.cu): cv::triangulatePoints + convertPointsFromHomogeneous, up to HV_ESSENTIAL_BATCH_MAX jobs
struct TriArgs {
    double P1[12], P2[12];            // row-major 3 x 4
    const float2* xy1; const float2* xy2;
    const uint8_t* status; const uint8_t* status2;     // NULL: all non-zero
    int n;
    float* X4;                        // 4 x n (row r at X4 + r n) or NULL
    float* xyz;                       // n x 3 or NULL
    uint8_t* used;                    // n, 0/1, or NULL; may be status or status2
};
struct TriBatchArgs {
    TriArgs job[HV_ESSENTIAL_BATCH_MAX];
};
static_assert(sizeof(TriBatchArgs) <= HV_KERNEL_PARAM_MAX, "triangulation batch arguments exceed the kernel-parameter space");
cudaError_t hv_launch_triangulate(const TriBatchArgs& b, int njobs, int maxn, cudaStream_t stream);   // one launch: grid (points, jobs)

// ---- frame ingest (ingest.cu)
#define HV_REMAP_INVALID (-32768)
struct HvRemapEntry { short x0, y0; float xfrac, yfrac; };      // 12 bytes per output pixel (hv_remap_entry of the C ABI)
cudaError_t hv_launch_gray(const uint8_t* src, int srcPitch, int channels, int w, int h, const float coeff[4], uint8_t* dst, int dstPitch, cudaStream_t s);
cudaError_t hv_launch_remap(const uint8_t* src, int srcPitch, int w, int h, const HvRemapEntry* table, uint8_t* dst, int dstPitch, cudaStream_t s);

// Frames that need colour conversion and / or a remap, HV_CORNER_BATCH_MAX per launch (hv_ingest_frames)
struct IngestJob {
    const uint8_t* src; int srcPitch, channels;     // channels > 1: colour -> gray
    float coeff[4];                                 // resolved as hv_ingest_frame resolves them
    const HvRemapEntry* table;                      // NULL: no remap
    uint8_t* dst; int dstPitch;                     // level 0 of the pyramid
    int w, h;
};
struct IngestBatchArgs {
    IngestJob job[HV_CORNER_BATCH_MAX];
    int first[HV_CORNER_BATCH_MAX + 1];             // first CTA of job j: prefix sum of ceil(w / 256) * h; first[njobs ..] = the grid
};
static_assert(sizeof(IngestBatchArgs) <= HV_KERNEL_PARAM_MAX, "ingest batch arguments exceed the kernel-parameter space");
cudaError_t hv_launch_ingest_batch(const IngestBatchArgs& b, int njobs, cudaStream_t s);
