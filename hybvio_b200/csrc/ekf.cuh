// hybvio_b200/csrc/ekf.cuh -- device-side EKF state layout and kernel argument blocks (ekf.cu, ekf_capi.cu).
#pragma once
#include <cuda_runtime.h>

// State layout of odometry::EKF (src/odometry/ekf.hpp:26-50)
#define EKF_POS 0
#define EKF_VEL 3
#define EKF_ORI 6
#define EKF_BGA 10
#define EKF_BAA 13
#define EKF_BAT 16
#define EKF_SFT 19
#define EKF_CAM 20
#define EKF_INER 20
#define EKF_POSE 7
#define EKF_MAP_POINT 3
#define EKF_Q_ACC 0
#define EKF_Q_GYRO 3
#define EKF_Q_BGA_DRIFT 6
#define EKF_Q_BAA_DRIFT 9
#define EKF_Q_DIM 12

#define EKF_NT 512          // threads of the single-CTA kernels
#define EKF_SMALL_MAXN 8    // rows of the built-in (selector) measurement models
#define EKF_SMALL_MAXL 32

// Device buffers of one filter. P is fp64 COLUMN-MAJOR with leading dimension N (Eigen layout).
struct EkfBufs {
    double* m;        // N
    double* P;        // N x N   (current)
    double* P2;       // N x N   (target of out-of-place shifts/transforms; host swaps after the launch)
    double* work;     // global fallback for the elimination tableau when it does not fit shared memory
    double* cwork;    // cluster kernel exchange buffers through L2: gathered Z | reduced S | 8 partial S  (10 x N x N)
    double* Hs;       // EKF_SMALL_MAXN x EKF_SMALL_MAXL built-in measurement matrix
    double* Q;        // 12 x 12 process noise
    double* dydx;     // 20 x 20 last predict Jacobian (getDydx)
    double* res;      // [0] VuOutlierStatus, [1] chi2, [2] numeric flag (0 ok, 1 non-positive pivot)
    int N;
    int trail;        // camPoseCount
    int mapDim;       // hybridMapDim
};

// mode of ekf_update_kernel
#define EKF_MODE_CHECK 0          // visualTrackOutlierCheck
#define EKF_MODE_UPDATE 1         // updateVisualTrack / update()
#define EKF_MODE_CHECK_UPDATE 2   // check, then update iff inlier (one launch)

// built-in measurement models (ekf.cpp:573-677, 848-885)
#define EKF_OP_DENSE 0            // H given (visual update)
#define EKF_OP_ZUPT 1
#define EKF_OP_ZRUPT 2
#define EKF_OP_PSEUDO_VELOCITY 3
#define EKF_OP_POSITION 4
#define EKF_OP_ZERO_HEIGHT 5
#define EKF_OP_ORIENTATION 6
#define EKF_OP_AUGMENT 7

struct EkfUpdateArgs {
    EkfBufs b;
    const double* H;      // device, n x l column-major (ld n); unused for built-in ops
    const double* f;      // device, n (may be NULL: residual is y - H m)
    const double* y;      // device, n (may be NULL: use ysmall)
    double ysmall[EKF_SMALL_MAXN];
    int n, l;
    int op;
    int mode;
    double Rdiag;         // R = Rdiag * I (noiseScale already applied)
    double noiseScale;    // multiplies the chi2 statistic (ekf.cpp:815)
    double rmseThr;       // < 0: disabled
    double chi2Thr;       // chi2inv95[n]
    int skipChi2;         // r < 0: the check returns INLIER without computing (ekf.cpp:803)
    int normalizeAll;     // normalizeQuaternions() vs only the current orientation (updateCommon)
    int symmetrize;       // maintainPositiveSemiDefinite afterwards
    int dropIdx;          // EKF_OP_AUGMENT: discarded pose index
    double augNoisePos, augNoiseOri;   // visAugQ diagonal (noiseScale applied)
    double defaultSpeed;  // EKF_OP_PSEUDO_VELOCITY
    int useGlobalWork;    // tableau in b.work instead of shared memory (set by ekf_launch_update)
    int symFirst;         // EKF_OP_AUGMENT: a deferred maintainPositiveSemiDefinite() is applied while P is read
    // Result words for a polling host (both update kernels, ekf_report): sig[0..2] = res[0..2], then sig[3] = sigSeq, written to
    // mapped pinned host memory at decision time (a check+update continues with the update afterwards). NULL: none.
    double* sig;
    double sigSeq;
    // Device-side control flow (ekf_cluster2.cuh only) for chains that are issued without host round trips
    // (hv_ekf_visual_tracks): the kernel does its work only if
    //   (gateI == NULL || *gateI == gateIExpect) && (gateD == NULL || *gateD == gateDExpect) && (counter == NULL || *counter < counterMax),
    // otherwise it reports NOT_COMPUTED and leaves the filter alone. slot (3 doubles, device; both update kernels) receives the
    // result words as well; *bump is incremented once an update has been applied. lateH: the measurement model is produced by
    // the preceding kernel of the stream, so it may only be read after griddepcontrol.wait.
    const int* gateI; int gateIExpect;
    const double* gateD; double gateDExpect;
    const int* counter; int counterMax;
    int* bump;
    double* slot;
    int lateH;
    // Row-chunked form (ekf_cluster2.cuh, dense visual ops only; 0: off): the measurement is processed rowChunk rows at a time
    // next to the resident P blocks, for measurements whose whole tableau does not fit shared memory (ek2_geom_chunked)
    int rowChunk;
    // Results into the second buffers (ekf_cluster2.cuh; NULL: off): the updated covariance blocks and state mean are written to
    // specP / specM instead of P / m, which stay untouched -- the host adopts them by swapping pointers. Used by the speculative
    // update (dense check+update: adopted if the caller's updateVisualTrack(H, f, y, r) really follows the INLIER check with the same
    // measurement, hv_ekf_visual_update) and by the augmentation that shares a launch with outlier checks reading (m, P).
    double* specP; double* specM;
    // EKF_MODE_CHECK_UPDATE with two noise levels (ekf_cluster2.cuh only; 0: off): the outlier check uses Rdiag, the update that
    // follows an INLIER decision uses Rdiag2 -- visualTrackOutlierCheck(trackChiTestOutlierR) then updateVisualTrack(visualR),
    // backend.cpp:1158-1185, in one kernel: H P and S0 = H P H' are formed once, S0 + R is factorised twice.
    double Rdiag2;
};

// Result words (VuOutlierStatus, chi2, numeric flag), written by one thread of an update kernel at each decision: device copy,
// optional device slot, optional mapped-host copy whose sequence word follows the other three
__device__ __forceinline__ void ekf_report(const EkfUpdateArgs& a, double st, double chi2, double flag)
{
    a.b.res[0] = st; a.b.res[1] = chi2; a.b.res[2] = flag;
    if (a.slot) { a.slot[0] = st; a.slot[1] = chi2; a.slot[2] = flag; }
    if (a.sig) {
        a.sig[0] = st; a.sig[1] = chi2; a.sig[2] = flag;
        __threadfence_system();
        ((volatile double*)a.sig)[3] = a.sigSeq;
    }
}

// Independent outlier checks against the same (m, P): one launch of 8-CTA clusters. A small check runs on one CTA of a shared
// cluster (ek2_check_cta), any other on a cluster of its own (ek2_body); ekf_launch_check_batch2 decides and sets `compact`.
#define EKF_MAX_BATCH 24
#define EKF_RES_STRIDE 32
struct EkfCheckItem {
    const double* H; const double* f; const double* y;   // device
    int n, l;
    double Rdiag, chi2Thr, rmseThr;
    int skipChi2;
    int compact;          // 1: runs on one CTA
};
struct EkfCheckBatch { int count; int compact; EkfCheckItem it[EKF_MAX_BATCH]; };   // compact: number of items with it[i].compact

#define EKF_MAX_PREDICT 16
struct EkfPredictSample {
    double dt;
    double xg[3], xa[3];
    double baaDecay, bgaDecay;      // exp(-dt * rev) or 1 when the random walk is off (ekf.cpp:443-448)
    double qBaa, qBga;              // >= 0: value of the Q drift-block diagonal for this dt (ekf.cpp:397-412); < 0: keep
    int normAfter, pad;             // normalizeQuaternions(true) follows this sample (backend.cpp:734-735): folded into the chain
};
// `count` consecutive IMU samples in one launch (the 10 samples between two frames at 200 Hz / 20 fps)
struct EkfPredictArgs {
    EkfBufs b;
    double gravity;                 // gravity vector = (0, 0, -gravity)
    // meanOut != NULL: only the 20 inertial states the samples lead to are computed and written there (nothing else is read or written):
    // the part of predict() that consumers of the POSE need (the optical-flow predictor, backend.cpp:547-600), ~1/4 of the launch
    double* meanOut;
    int count;
    EkfPredictSample s[EKF_MAX_PREDICT];
};

// elementwise / structural operations on (m, P)
#define EKF_EW_SYMMETRIZE 1
#define EKF_EW_UNAUGMENT 2
#define EKF_EW_NORMALIZE 3          // ival0 = onlyCurrent
#define EKF_EW_TRANSLATE 4          // dval[0..2] = target position
#define EKF_EW_TRANSFORM 5          // dval[0..2] pos, dval[3..6] q, ival0 = pose index
#define EKF_EW_INSERT_MAP_POINT 6   // ival0 = state offset, dval[0..2] = point
#define EKF_EW_LOCK_BIASES 7
#define EKF_EW_CONDITION_LAST_POSE 8
#define EKF_EW_INIT_ORIENTATION 9   // dval[0..3] = q, dval[4] = variance (noiseInitialOri^2 * noiseScale)
struct EkfEwArgs {
    EkfBufs b;
    int op;
    int ival0;
    double dval[8];
};

cudaError_t ekf_launch_update(const EkfUpdateArgs& a, cudaStream_t s);
// ekf_launch_update picks the cluster kernel (the only one with specP / specM, Rdiag2 and the device-side gates) iff this holds or
// a.rowChunk > 0
bool ekf_cluster2_fits(int n, int l, int N, bool joseph);
// Rows per pass of the row-chunked form of a dense visual op of shape (n, l): the largest height whose working set fits beside the
// resident P blocks (n: one pass); 0 if not even min(n, EK2_MIN_CHUNK) rows fit
int ekf_cluster2_chunk_rows(int n, int l, int N);
// a.rowChunk > 0: the row-chunked form (whether or not the whole tableau would fit)
cudaError_t ekf_launch_update_cluster2(const EkfUpdateArgs& a, cudaStream_t s);
// aug != NULL: one more cluster of the same launch runs the augmentation *aug (results into aug->specP / aug->specM)
cudaError_t ekf_launch_check_batch2(const EkfUpdateArgs& a, const EkfCheckBatch& b, cudaStream_t s, const EkfUpdateArgs* aug = nullptr);
// The state mean of the augmentation a (EKF_OP_AUGMENT) into a.specM on one CTA, bitwise what the cluster kernel writes there; its
// covariance is left to a cluster launched elsewhere (flush_checks). Fits iff ekf_aug_mean_fits(a.b.N).
bool ekf_aug_mean_fits(int N);
cudaError_t ekf_launch_aug_mean(const EkfUpdateArgs& a, cudaStream_t s);
// Group launches (hv_ekf_group_run_device): instance i of the launch runs dArgs[i], a fully resolved argument block in device memory;
// hArgs is the host copy of the same blocks (launch shape: shared memory of the largest instance)
cudaError_t ekf_launch_group_cluster2(const EkfUpdateArgs* hArgs, const EkfUpdateArgs* dArgs, int count, cudaStream_t s);
cudaError_t ekf_launch_group_predict(const EkfPredictArgs* hArgs, const EkfPredictArgs* dArgs, int count, cudaStream_t s);
struct TmArgs;
cudaError_t ekf_launch_predict(const EkfPredictArgs& a, cudaStream_t s);
cudaError_t ekf_launch_elementwise(const EkfEwArgs& a, cudaStream_t s);
