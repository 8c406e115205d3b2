// hybvio_b200/csrc/ekf_capi.cu -- C ABI of the EKF (include/hybvio_b200.h). Host side of odometry::EKF:
// the scalar bookkeeping EKFImplementation keeps next to m and P (sample times, ZUPT rate limits, augment times;
// src/odometry/ekf.cpp:145-151) lives here; m, P and all arithmetic on them live on the device (ekf.cu).
#include "capi_internal.h"
#include "ekf.cuh"
#include "track_model.h"
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>
#include <chrono>

#define HV_RUN_MAX_OPS 256       // ops of one hv_ekf_run_host list that can report through the mapped result area

struct hv_ekf {
    hv_ctx* ctx = nullptr;
    hv_ekf_params prm;
    int N = 0, trail = 0, mapDim = 0;
    double noiseScale = 1.0;      // = odometry.noiseScale^2 (ekf.cpp:154)
    double* d_block = nullptr;    // one allocation: m | P | P2 | work | Hs | Q | dydx | res | in
    EkfBufs b;
    double* d_in = nullptr;       // staging for H, f, y uploads
    size_t inDoubles = 0;
    double* h_pin = nullptr;      // pinned host staging: [in (inDoubles) | out (N + 8)]
    cudaEvent_t evStaged = nullptr;   // recorded after the H2D copy out of h_pin: the staging block may be refilled once it has fired
    bool stagedPending = false;
    double* h_sig = nullptr;      // mapped pinned result words the kernels write for a polling host: 4 doubles per batch slot
    double* d_sig = nullptr;      // (device alias)
    double* h_run = nullptr;      // mapped pinned result words of hv_ekf_run_host: 4 doubles per op of the list (HV_RUN_MAX_OPS)
    double* d_run = nullptr;      // (device alias)
    // Speculative update behind an INLIER check (visual_host): results wait in P2 / m2 until hv_ekf_visual_update adopts them
    double* m2 = nullptr;                   // second state mean (device)
    unsigned long long epoch = 0;           // bumped by everything that changes the filter state on the device
    struct { bool valid = false; unsigned long long epoch = 0; int n = 0, l = 0; } spec;
    double specR = -1.0;                    // noise level of the last updateVisualTrack (what the next check speculates with); < 0: none yet
    bool specEnabled = false;               // the caller follows INLIER checks with updates (switched off by the first speculation nobody adopts)
    cudaStream_t copyStream = nullptr;            // hv_ekf_run_host: the measurement inputs travel on their own stream, ahead of the kernels
    std::vector<cudaEvent_t> copyEvents;          // one per measurement group of a list (created on demand)
    double sigSeq = 0.0;
    // hv_ekf_run_device in latency mode: a run of outlier checks that is followed by the pose augmentation goes to a SIDE stream together
    // with the augmentation's covariance (one launch: the checks read (m, P), the augmentation cluster writes P2); the augmentation's mean
    // is formed on the context's stream by one CTA (ekf_launch_aug_mean, into m2), so that the next frame's mean propagation and optical
    // flow do not wait for the covariance. While sideBusy, P is on the side stream: join_side() makes the context's stream wait for it,
    // and every consumer of P (or writer of the second buffers) calls it before it issues; readers of the mean alone do not.
    cudaEvent_t evFork = nullptr, evJoin = nullptr;       // (the stream itself belongs to the context: hv_ctx::sideStream)
    // After hv_ekf_predicted_mean_device the full launch of the IMU burst (covariance) goes to a stream of its own (hv_ctx::covStream):
    // whatever the caller issues next on the context's stream without touching the filter (the optical flow, when tracker and filter
    // share a stream) does not queue behind it; the next call that touches the filter joins it
    cudaEvent_t evCovFork = nullptr, evCov = nullptr;
    bool covBusy = false, meanIssued = false;
    bool sideBusy = false;
    double* cworkSide = nullptr;            // exchange areas and result words of the clusters on the side stream
    double* resSide = nullptr;
    double* mSide = nullptr;                // where the augmentation cluster on the side stream leaves its mean (N; read by nobody)
    double* d_opres = nullptr;              // hv_ekf_run_device: result words per op of the list (4 doubles each, HV_RUN_MAX_OPS)
    double* d_mean20 = nullptr;             // hv_ekf_predicted_mean: device scratch
    std::vector<unsigned char> lastVisual;  // per op of the last hv_ekf_run_device list: 1 = VISUAL (has result words)
    double hostTimes[4] = {0, 0, 0, 0};     // last hv_ekf_run_host list: {issue, wait, total} in us, number of ops (hv_ekf_debug_host_times)
    // host bookkeeping, exactly the members of EKFImplementation (ekf.cpp:145-151)
    int augmentCount = 0;
    std::vector<double> augmentTimes;
    double time = 0.0, ZUPTtime = -1.0, ZRUPTtime = -1.0, initZUPTtime = -1.0;
    bool wasStationary = false;
    double prevSampleT = -1.0, firstSampleT = -1.0;
    bool firstSample = true;
    std::vector<double> chi2inv95;
    // Deferred work (issued by the next call that needs the state, or hv_ekf_flush): the IMU samples of consecutive
    // predict() calls -- with the normalizeQuaternions(true) that follows each of them in the reference loop
    // (src/odometry/backend.cpp:734-735) -- become ONE launch; a maintainPositiveSemiDefinite() directly followed by the
    // pose augmentation (backend.cpp:1267 -> 805) is applied inside the augmentation kernel.
    EkfPredictArgs pend;
    bool pendSym = false;
    int imuBatch = EKF_MAX_PREDICT;
    struct TrackModels* tm = nullptr;    // per-track measurement model on the device (hv_ekf_track_models), created on first use
};

// Buffers of hv_ekf_track_models: inputs packed by the host into one pinned block, outputs in HBM (H, f, d pf) + a small
// status block that travels back.
struct TrackModels {
    hv_camera_model cam;
    bool camSet = false;
    int cap = 0, last = 0;
    std::vector<int> lastNpose;
    TmArgs lastArgs;
    char* d_in = nullptr;  char* h_in = nullptr;      // [npose int cap | idx int cap x MAXPOSE | ip | vel]
    char* d_out = nullptr; char* h_out = nullptr;     // [status int 4 cap | pf double 4 cap]
    double *d_dpf = nullptr, *d_H = nullptr, *d_f = nullptr;
    char* d_ctl = nullptr; char* h_ctl = nullptr; int ctlCap = 0;      // chains: [success counter int, pad to 16 B | 8 doubles per track]
    static size_t ctlBytes(int c) { return 16 + (size_t)c * 64; }
    static size_t inBytes(int c) { return (size_t)c * (sizeof(int) * (1 + TM_MAXPOSE + 1) + sizeof(double) * 4 * TM_MAXOBS); }   // +1 int: keeps the doubles 8-byte aligned
    static size_t outBytes(int c) { return (size_t)c * (sizeof(int) * 4 + sizeof(double) * 4); }
    static size_t hStride() { return (size_t)2 * TM_MAXOBS * TM_MAXN; }
    void release()
    {
        cudaFree(d_in); cudaFree(d_out); cudaFree(d_dpf); cudaFree(d_H); cudaFree(d_f); cudaFreeHost(h_in); cudaFreeHost(h_out);
        cudaFree(d_ctl); cudaFreeHost(h_ctl);
        d_in = d_out = h_in = h_out = d_ctl = h_ctl = nullptr; d_dpf = d_H = d_f = nullptr; cap = 0; ctlCap = 0;
    }
};

// ---- chi-square 95% quantiles (the reference hard-codes the table odometry/util.hpp:23; recomputed here by
// inverting the regularised incomplete gamma function to ~1e-14 relative)
static double gamma_p(double a, double x)
{
    if (x <= 0) return 0.0;
    const double gln = lgamma(a);
    if (x < a + 1.0) {
        double ap = a, sum = 1.0 / a, del = sum;
        for (int i = 0; i < 2000; i++) { ap += 1.0; del *= x / ap; sum += del; if (fabs(del) < fabs(sum) * 1e-17) break; }
        return sum * exp(-x + a * log(x) - gln);
    }
    double bq = x + 1.0 - a, c = 1e300, d = 1.0 / bq, h = d;
    for (int i = 1; i < 2000; i++) {
        const double an = -i * (i - a); bq += 2.0;
        d = an * d + bq; if (fabs(d) < 1e-300) d = 1e-300;
        c = bq + an / c; if (fabs(c) < 1e-300) c = 1e-300;
        d = 1.0 / d; const double del = d * c; h *= del;
        if (fabs(del - 1.0) < 1e-17) break;
    }
    return 1.0 - exp(-x + a * log(x) - gln) * h;
}
static double chi2inv(double p, int k)
{
    double lo = 0.0, hi = k + 10.0 * sqrt(2.0 * k) + 20.0;
    for (int it = 0; it < 200; it++) {
        const double mid = 0.5 * (lo + hi);
        if (gamma_p(0.5 * k, 0.5 * mid) < p) lo = mid; else hi = mid;
        if (hi - lo < 1e-15 * hi) break;
    }
    return 0.5 * (lo + hi);
}

static inline double pow2(double x) { return x * x; }

static int ekf_check(const hv_ekf* e, const char* who)
{
    if (!e) { hv_set_error("%s: NULL ekf", who); return HV_ERR_INVALID; }
    return HV_OK;
}

extern "C" { static int flush_pending(hv_ekf* e); }
static int join_side(hv_ekf* e);
extern "C" { static int staging_acquire(hv_ekf* e); }
// EKF_ENTER_LAZY: entry points that only extend the deferred queue; EKF_ENTER: everything else issues the queue first
#define EKF_ENTER_LAZY(e, who)                         \
    do { int rc_ = ekf_check(e, who); if (rc_ != HV_OK) return rc_; HV_CUDA(cudaSetDevice((e)->ctx->device)); } while (0)
#define EKF_ENTER(e, who)                              \
    do { EKF_ENTER_LAZY(e, who); int rc2_ = flush_pending(e); if (rc2_ != HV_OK) return rc2_; } while (0)

// The filter's side of an update's argument block, at the moment it is issued
static void update_settle(hv_ekf* e, EkfUpdateArgs& a)
{
    e->epoch++;
    a.b = e->b;
    a.noiseScale = e->noiseScale;
}
static int launch_update(hv_ekf* e, EkfUpdateArgs& a)
{
    int rcj = join_side(e);
    if (rcj != HV_OK) return rcj;
    update_settle(e, a);
    HV_CUDA(ekf_launch_update(a, e->ctx->stream));
    e->ctx->launches++;
    return HV_OK;
}

static void fill_small(EkfUpdateArgs& a, int op, int n, int l, double Rdiag, int mode = EKF_MODE_UPDATE)
{
    memset(&a, 0, sizeof(a));
    a.op = op; a.n = n; a.l = l; a.mode = mode; a.Rdiag = Rdiag; a.rmseThr = -1.0; a.chi2Thr = 0.0;
}

static int launch_ew(hv_ekf* e, int op, int ival0 = 0, const double* dv = nullptr, int ndv = 0)
{
    EkfEwArgs a; memset(&a, 0, sizeof(a));
    int rcj = join_side(e);                           // (UNAUGMENT / TRANSFORM: out of place into P2)
    if (rcj != HV_OK) return rcj;
    e->epoch++;
    a.b = e->b; a.op = op; a.ival0 = ival0;
    for (int i = 0; i < ndv; i++) a.dval[i] = dv[i];
    HV_CUDA(ekf_launch_elementwise(a, e->ctx->stream));
    e->ctx->launches++;
    return HV_OK;
}

static void swap_P(hv_ekf* e) { double* t = e->b.P; e->b.P = e->b.P2; e->b.P2 = t; }
// The launch on the side stream writes P (the augmentation's covariance) and reads what are now the SECOND buffers: every consumer of P and
// every writer of P2 / m2 on the context's stream waits for it first (the covariance launch of an IMU burst on its own stream waits for
// evJoin itself, predict_launch)
static int join_side(hv_ekf* e)
{
    if (!e->sideBusy) return HV_OK;
    HV_CUDA(cudaStreamWaitEvent(e->ctx->stream, e->evJoin, 0));
    e->sideBusy = false;
    return HV_OK;
}

extern "C" {

void hv_ekf_default_params(hv_ekf_params* p)
{
    if (!p) return;
    // codegen/parameter_definitions.c:68-160
    p->camera_trail_length = 20; p->hybrid_map_size = 0;
    p->noise_scale = 100; p->gravity = 9.819;
    p->noise_initial_pos = 1e-5; p->noise_initial_vel = 0.1; p->noise_initial_ori = 0.0316227766;
    p->noise_initial_bga = 1e-3; p->noise_initial_baa = 1e-6; p->noise_initial_bat = 1e-5; p->noise_initial_sft = 1e-5;
    p->noise_initial_pos_trail = 100; p->noise_initial_ori_trail = 3.16227766;
    p->noise_process_acc = 0.003; p->noise_process_gyro = 0.00017;
    p->noise_process_baa = 1e-4; p->noise_process_baa_rev = 0.1; p->noise_process_bga = 0; p->noise_process_bga_rev = 0.1;
    p->augment_r = 1e-9; p->init_zupt_r = 1e-4; p->rotation_zupt_r = 1e-6;
}

static int ekf_alloc(hv_ctx* c, const hv_ekf_params* prm, hv_ekf** out)
{
    hv_ekf* e = new hv_ekf;
    memset(&e->pend, 0, sizeof(e->pend));
    e->ctx = c; e->prm = *prm;
    e->trail = prm->camera_trail_length; e->mapDim = prm->hybrid_map_size * EKF_MAP_POINT;
    e->N = EKF_INER + e->trail * EKF_POSE + e->mapDim;
    e->noiseScale = prm->noise_scale * prm->noise_scale;
    const size_t N = e->N, NN = N * N;
    const size_t workD = N * (2 * N + 4);
    const size_t cworkD = (size_t)(EKF_MAX_BATCH + 1) * 10 * NN;       // one exchange area per cluster of a check batch (+ its augmentation)
    e->inDoubles = (size_t)EKF_MAX_BATCH * (NN + 2 * N);
    const size_t resD = (size_t)EKF_RES_STRIDE * (EKF_MAX_BATCH + 1);
    const size_t total = N + NN + NN + workD + 2 * cworkD + EKF_SMALL_MAXN * EKF_SMALL_MAXL + 144 + 400 + 2 * resD + e->inDoubles + N + 4 * HV_RUN_MAX_OPS + 32 + N;
    cudaError_t err = cudaMalloc(&e->d_block, total * sizeof(double));
    if (err != cudaSuccess) { delete e; hv_set_error("hv_ekf_create: cudaMalloc failed: %s", cudaGetErrorString(err)); return HV_ERR_OOM; }
    cudaMemsetAsync(e->d_block, 0, total * sizeof(double), c->stream);
    double* p = e->d_block;
    e->b.m = p; p += N; e->b.P = p; p += NN; e->b.P2 = p; p += NN; e->b.work = p; p += workD; e->b.cwork = p; p += cworkD;
    e->b.Hs = p; p += EKF_SMALL_MAXN * EKF_SMALL_MAXL; e->b.Q = p; p += 144; e->b.dydx = p; p += 400; e->b.res = p; p += EKF_RES_STRIDE * (EKF_MAX_BATCH + 1);
    e->d_in = p; p += e->inDoubles;
    e->m2 = p; p += N;
    e->cworkSide = p; p += cworkD; e->resSide = p; p += resD; e->d_opres = p; p += 4 * HV_RUN_MAX_OPS;
    e->d_mean20 = p; p += 32;
    e->mSide = p;
    e->b.N = e->N; e->b.trail = e->trail; e->b.mapDim = e->mapDim;
    err = cudaMallocHost(&e->h_pin, (e->inDoubles + N + 8) * sizeof(double));
    if (err != cudaSuccess) { cudaFree(e->d_block); delete e; hv_set_error("hv_ekf_create: cudaMallocHost failed"); return HV_ERR_OOM; }
    if (cudaEventCreateWithFlags(&e->evStaged, cudaEventDisableTiming) != cudaSuccess) { cudaFree(e->d_block); cudaFreeHost(e->h_pin); delete e; hv_set_error("hv_ekf_create: cudaEventCreate failed"); return HV_ERR_CUDA; }
    err = cudaHostAlloc(&e->h_sig, 4 * sizeof(double) * (EKF_MAX_BATCH + 1), cudaHostAllocMapped);
    if (err == cudaSuccess) err = cudaHostGetDevicePointer(&e->d_sig, e->h_sig, 0);
    if (err != cudaSuccess) { cudaFree(e->d_block); cudaFreeHost(e->h_pin); delete e; hv_set_error("hv_ekf_create: mapped result buffer: %s", cudaGetErrorString(err)); return HV_ERR_OOM; }
    memset(e->h_sig, 0, 4 * sizeof(double) * (EKF_MAX_BATCH + 1));
    err = cudaHostAlloc(&e->h_run, 4 * sizeof(double) * HV_RUN_MAX_OPS, cudaHostAllocMapped);
    if (err == cudaSuccess) err = cudaHostGetDevicePointer(&e->d_run, e->h_run, 0);
    if (err != cudaSuccess) { cudaFree(e->d_block); cudaFreeHost(e->h_pin); cudaFreeHost(e->h_sig); delete e; hv_set_error("hv_ekf_create: mapped result buffer: %s", cudaGetErrorString(err)); return HV_ERR_OOM; }
    memset(e->h_run, 0, 4 * sizeof(double) * HV_RUN_MAX_OPS);
    *out = e;
    return HV_OK;
}

int hv_ekf_create(hv_ctx* c, const hv_ekf_params* prm, hv_ekf** out)
{
    if (!c || !prm || !out || prm->camera_trail_length < 1 || prm->hybrid_map_size < 0) {
        hv_set_error("hv_ekf_create: invalid argument"); return HV_ERR_INVALID;
    }
    const int N = EKF_INER + prm->camera_trail_length * EKF_POSE + prm->hybrid_map_size * EKF_MAP_POINT;
    if (N > 768) { hv_set_error("hv_ekf_create: state dimension %d > 768 unsupported", N); return HV_ERR_UNSUPPORTED; }
    HV_CUDA(cudaSetDevice(c->device));
    hv_ekf* e = nullptr;
    int rc = ekf_alloc(c, prm, &e);
    if (rc != HV_OK) return rc;
    // initial state (ekf.cpp:174-225)
    std::vector<double> m(N, 0.0), P((size_t)N * N, 0.0), Q(144, 0.0);
    m[EKF_ORI] = 1.0;
    for (int i = 0; i < 3; i++) m[EKF_BAT + i] = 1.0;
    auto diag = [&](int i, double v) { P[(size_t)i * (N + 1)] = v; };
    for (int i = 0; i < 3; i++) { diag(EKF_POS + i, pow2(prm->noise_initial_pos)); diag(EKF_VEL + i, pow2(prm->noise_initial_vel)); }
    for (int i = 0; i < 4; i++) diag(EKF_ORI + i, 1.0);
    for (int i = 0; i < 3; i++) { diag(EKF_BGA + i, pow2(prm->noise_initial_bga)); diag(EKF_BAA + i, pow2(prm->noise_initial_baa)); diag(EKF_BAT + i, pow2(prm->noise_initial_bat)); }
    diag(EKF_SFT, pow2(prm->noise_initial_sft));
    for (int p = 0; p < e->trail; p++) {
        const int o = EKF_CAM + p * EKF_POSE;
        for (int i = 0; i < 3; i++) diag(o + i, pow2(prm->noise_initial_pos_trail));
        for (int i = 0; i < 4; i++) diag(o + 3 + i, pow2(prm->noise_initial_ori_trail));
    }
    for (int i = 0; i < 3; i++) { Q[(EKF_Q_ACC + i) * 13] = pow2(prm->noise_process_acc); Q[(EKF_Q_GYRO + i) * 13] = pow2(prm->noise_process_gyro); }
    for (auto& v : P) v *= e->noiseScale;
    for (auto& v : Q) v *= e->noiseScale;
    HV_CUDA(cudaMemcpyAsync(e->b.m, m.data(), sizeof(double) * N, cudaMemcpyHostToDevice, c->stream));
    HV_CUDA(cudaMemcpyAsync(e->b.P, P.data(), sizeof(double) * N * N, cudaMemcpyHostToDevice, c->stream));
    HV_CUDA(cudaMemcpyAsync(e->b.Q, Q.data(), sizeof(double) * 144, cudaMemcpyHostToDevice, c->stream));
    HV_CUDA(cudaStreamSynchronize(c->stream));
    e->chi2inv95.resize(201);
    e->chi2inv95[0] = 0.0;
    for (int k = 1; k <= 200; k++) e->chi2inv95[k] = chi2inv(0.95, k);
    *out = e;
    return HV_OK;
}

int hv_ekf_destroy(hv_ekf* e)
{
    if (!e) return HV_OK;
    cudaSetDevice(e->ctx->device);
    cudaStreamSynchronize(e->ctx->stream);
    cudaFree(e->d_block);
    cudaFreeHost(e->h_pin);
    cudaFreeHost(e->h_sig);
    cudaFreeHost(e->h_run);
    for (cudaEvent_t ev : e->copyEvents) cudaEventDestroy(ev);
    if (e->copyStream) cudaStreamDestroy(e->copyStream);
    if (e->ctx->sideStream) cudaStreamSynchronize(e->ctx->sideStream);
    if (e->ctx->covStream) cudaStreamSynchronize(e->ctx->covStream);
    if (e->evCovFork) cudaEventDestroy(e->evCovFork);
    if (e->evCov) cudaEventDestroy(e->evCov);
    if (e->evFork) cudaEventDestroy(e->evFork);
    if (e->evJoin) cudaEventDestroy(e->evJoin);
    if (e->evStaged) cudaEventDestroy(e->evStaged);
    if (e->tm) { e->tm->release(); delete e->tm; }
    delete e;
    return HV_OK;
}

int hv_ekf_clone(const hv_ekf* src, hv_ekf** out)
{
    if (!src || !out) { hv_set_error("hv_ekf_clone: NULL"); return HV_ERR_INVALID; }
    HV_CUDA(cudaSetDevice(src->ctx->device));
    hv_ekf* e = nullptr;
    int rc = flush_pending(const_cast<hv_ekf*>(src));     // deferred work belongs to the state being copied
    if (rc == HV_OK) rc = join_side(const_cast<hv_ekf*>(src));
    if (rc != HV_OK) return rc;
    rc = ekf_alloc(src->ctx, &src->prm, &e);
    if (rc != HV_OK) return rc;
    const size_t N = src->N;
    cudaStream_t s = src->ctx->stream;
    HV_CUDA(cudaMemcpyAsync(e->b.m, src->b.m, sizeof(double) * N, cudaMemcpyDeviceToDevice, s));
    HV_CUDA(cudaMemcpyAsync(e->b.P, src->b.P, sizeof(double) * N * N, cudaMemcpyDeviceToDevice, s));
    HV_CUDA(cudaMemcpyAsync(e->b.Q, src->b.Q, sizeof(double) * 144, cudaMemcpyDeviceToDevice, s));
    HV_CUDA(cudaMemcpyAsync(e->b.dydx, src->b.dydx, sizeof(double) * 400, cudaMemcpyDeviceToDevice, s));
    e->augmentCount = src->augmentCount; e->augmentTimes = src->augmentTimes;
    e->time = src->time; e->ZUPTtime = src->ZUPTtime; e->ZRUPTtime = src->ZRUPTtime; e->initZUPTtime = src->initZUPTtime;
    e->wasStationary = src->wasStationary; e->prevSampleT = src->prevSampleT; e->firstSampleT = src->firstSampleT;
    e->firstSample = src->firstSample; e->chi2inv95 = src->chi2inv95; e->imuBatch = src->imuBatch;
    if (src->tm && src->tm->camSet) { e->tm = new TrackModels(); e->tm->cam = src->tm->cam; e->tm->camSet = true; }
    *out = e;
    return HV_OK;
}

int hv_ekf_state_dim(const hv_ekf* e) { return e ? e->N : HV_ERR_INVALID; }
int hv_ekf_pose_count(const hv_ekf* e) { return e ? e->augmentCount + 1 : HV_ERR_INVALID; }
double hv_ekf_platform_time(const hv_ekf* e) { return e ? e->firstSampleT + e->time : 0.0; }
double hv_ekf_history_time(const hv_ekf* e, int i)
{
    if (!e) return 0.0;
    if (i == -1) return hv_ekf_platform_time(e);
    const int n = (int)e->augmentTimes.size();
    if (i < 0 || i >= n) return 0.0;
    return e->augmentTimes[n - i - 1];
}
int hv_ekf_was_stationary(const hv_ekf* e) { return e && e->wasStationary ? 1 : 0; }
int hv_ekf_set_first_sample_time(hv_ekf* e, double t)
{
    if (!e || !(t > 0.0)) { hv_set_error("hv_ekf_set_first_sample_time: invalid"); return HV_ERR_INVALID; }
    e->firstSample = false; e->firstSampleT = t; e->prevSampleT = t; e->time = t;   // ekf.cpp:1035-1041
    return HV_OK;
}

int hv_ekf_upload(hv_ekf* e, const double* m, const double* P)
{
    EKF_ENTER(e, "hv_ekf_upload");
    { int rcj = join_side(e); if (rcj != HV_OK) return rcj; }
    e->epoch++;
    const size_t N = e->N;
    if (m) HV_CUDA(cudaMemcpyAsync(e->b.m, m, sizeof(double) * N, cudaMemcpyHostToDevice, e->ctx->stream));
    if (P) HV_CUDA(cudaMemcpyAsync(e->b.P, P, sizeof(double) * N * N, cudaMemcpyHostToDevice, e->ctx->stream));
    HV_CUDA(cudaStreamSynchronize(e->ctx->stream));   // caller's buffers may be pageable / reused
    return HV_OK;
}

int hv_ekf_download(hv_ekf* e, double* m, double* P)
{
    EKF_ENTER(e, "hv_ekf_download");
    { int rcj = join_side(e); if (rcj != HV_OK) return rcj; }
    const size_t N = e->N;
    if (m) HV_CUDA(cudaMemcpyAsync(m, e->b.m, sizeof(double) * N, cudaMemcpyDeviceToHost, e->ctx->stream));
    if (P) HV_CUDA(cudaMemcpyAsync(P, e->b.P, sizeof(double) * N * N, cudaMemcpyDeviceToHost, e->ctx->stream));
    HV_CUDA(cudaStreamSynchronize(e->ctx->stream));
    return HV_OK;
}

int hv_ekf_download_inertial(hv_ekf* e, double* m20, double* P20)
{
    EKF_ENTER(e, "hv_ekf_download_inertial");
    { int rcj = join_side(e); if (rcj != HV_OK) return rcj; }
    if (m20) HV_CUDA(cudaMemcpyAsync(m20, e->b.m, sizeof(double) * 20, cudaMemcpyDeviceToHost, e->ctx->stream));
    if (P20) HV_CUDA(cudaMemcpy2DAsync(P20, 20 * sizeof(double), e->b.P, e->N * sizeof(double), 20 * sizeof(double), 20,
                                       cudaMemcpyDeviceToHost, e->ctx->stream));
    HV_CUDA(cudaStreamSynchronize(e->ctx->stream));
    return HV_OK;
}

int hv_ekf_set_inertial_state(hv_ekf* e, const double* m20, const double* P20)
{
    EKF_ENTER(e, "hv_ekf_set_inertial_state");
    { int rcj = join_side(e); if (rcj != HV_OK) return rcj; }
    if (!m20 || !P20) { hv_set_error("hv_ekf_set_inertial_state: NULL"); return HV_ERR_INVALID; }
    e->epoch++;
    HV_CUDA(cudaMemcpyAsync(e->b.m, m20, sizeof(double) * 20, cudaMemcpyHostToDevice, e->ctx->stream));
    HV_CUDA(cudaMemcpy2DAsync(e->b.P, e->N * sizeof(double), P20, 20 * sizeof(double), 20 * sizeof(double), 20,
                              cudaMemcpyHostToDevice, e->ctx->stream));
    HV_CUDA(cudaStreamSynchronize(e->ctx->stream));
    e->augmentCount = 0; e->augmentTimes.clear();   // pose trail invalid (ekf.cpp:687-689)
    return HV_OK;
}

int hv_ekf_set_process_noise(hv_ekf* e, const double* Q)
{
    EKF_ENTER(e, "hv_ekf_set_process_noise");
    if (!Q) { hv_set_error("hv_ekf_set_process_noise: NULL"); return HV_ERR_INVALID; }
    HV_CUDA(cudaMemcpyAsync(e->b.Q, Q, sizeof(double) * 144, cudaMemcpyHostToDevice, e->ctx->stream));
    HV_CUDA(cudaStreamSynchronize(e->ctx->stream));
    return HV_OK;
}

int hv_ekf_get_dydx(hv_ekf* e, double* d)
{
    EKF_ENTER(e, "hv_ekf_get_dydx");
    if (!d) { hv_set_error("hv_ekf_get_dydx: NULL output"); return HV_ERR_INVALID; }
    HV_CUDA(cudaMemcpyAsync(d, e->b.dydx, sizeof(double) * 400, cudaMemcpyDeviceToHost, e->ctx->stream));
    HV_CUDA(cudaStreamSynchronize(e->ctx->stream));
    return HV_OK;
}

int hv_ekf_initialize_orientation(hv_ekf* e, const double xa[3])
{
    EKF_ENTER(e, "hv_ekf_initialize_orientation");
    // Eigen::Quaterniond::FromTwoVectors(-gravity, xa), -gravity = (0, 0, +g)  (ekf.cpp:301)
    const double nb = std::sqrt(xa[0] * xa[0] + xa[1] * xa[1] + xa[2] * xa[2]);
    if (!(nb > 0)) { hv_set_error("hv_ekf_initialize_orientation: zero accelerometer sample"); return HV_ERR_INVALID; }
    const double v0[3] = {0, 0, e->prm.gravity >= 0 ? 1.0 : -1.0}, v1[3] = {xa[0] / nb, xa[1] / nb, xa[2] / nb};
    double c = v0[2] * v1[2];
    double dv[5];
    if (c < -1.0 + 1e-12) {
        // antiparallel: Eigen takes the rotation axis from an SVD null vector (any axis orthogonal to v0); we fix
        // the x axis, which keeps q[3] == 0 as ekf.cpp:310 asserts.
        c = c < -1.0 ? -1.0 : c;
        const double w2 = (1.0 + c) * 0.5;
        dv[0] = std::sqrt(w2); dv[1] = std::sqrt(1.0 - w2); dv[2] = 0.0; dv[3] = 0.0;
    } else {
        const double ax[3] = {v0[1] * v1[2] - v0[2] * v1[1], v0[2] * v1[0] - v0[0] * v1[2], v0[0] * v1[1] - v0[1] * v1[0]};
        const double s = std::sqrt((1.0 + c) * 2.0), invs = 1.0 / s;
        dv[0] = s * 0.5; dv[1] = ax[0] * invs; dv[2] = ax[1] * invs; dv[3] = ax[2] * invs;
    }
    dv[4] = pow2(e->prm.noise_initial_ori) * e->noiseScale;
    return launch_ew(e, EKF_EW_INIT_ORIENTATION, 0, dv, 5);
}

// Host bookkeeping of one predict() call (ekf.cpp:357-370); appends a device sample unless the call is a no-op.
static void predict_bookkeep(hv_ekf* e, double t, const double xg[3], const double xa[3], EkfPredictArgs& a)
{
    double dt = 0.0;
    if (!e->firstSample) { dt = t - e->prevSampleT; e->time = t - e->firstSampleT; }
    else { e->firstSampleT = t; e->firstSample = false; }
    e->prevSampleT = t;
    if (dt <= 0.0) return;
    EkfPredictSample& s = a.s[a.count++];
    s.dt = dt;
    for (int i = 0; i < 3; i++) { s.xg[i] = xg[i]; s.xa[i] = xa[i]; }
    s.qBaa = -1.0; s.qBga = -1.0; s.baaDecay = 1.0; s.bgaDecay = 1.0; s.normAfter = 0; s.pad = 0;
    if (e->prm.noise_process_baa > 0.0) {  // ekf.cpp:397-404, 443-445
        const double th = e->prm.noise_process_baa_rev;
        s.qBaa = e->noiseScale * pow2(e->prm.noise_process_baa);
        if (th > 0.0) s.qBaa *= (1 - std::exp(-2 * dt * th)) / (2 * th);
        s.baaDecay = std::exp(-dt * th);
    }
    if (e->prm.noise_process_bga > 0.0) {  // ekf.cpp:405-412, 446-448
        const double th = e->prm.noise_process_bga_rev;
        s.qBga = e->noiseScale * pow2(e->prm.noise_process_bga);
        if (th > 0.0) s.qBga *= (1 - std::exp(-2 * dt * th)) / (2 * th);
        s.bgaDecay = std::exp(-dt * th);
    }
}

static int join_cov(hv_ekf* e)
{
    if (!e->covBusy) return HV_OK;
    HV_CUDA(cudaStreamWaitEvent(e->ctx->stream, e->evCov, 0));
    e->covBusy = false;
    return HV_OK;
}
static void predict_settle(hv_ekf* e, EkfPredictArgs& a)
{
    a.b = e->b; a.gravity = e->prm.gravity;
    e->epoch++;
}
static int predict_launch(hv_ekf* e, EkfPredictArgs& a)
{
    if (a.count == 0) return HV_OK;
    predict_settle(e, a);
    static const bool latencyMode = getenv("HV_EKF_NO_PDL") == nullptr;
    if (e->meanIssued && latencyMode) {
        // the mean of this burst is out already (hv_ekf_predicted_mean_device): the full launch runs beside the context's stream
        hv_ctx* c = e->ctx;
        if (!c->covStream) HV_CUDA(cudaStreamCreateWithFlags(&c->covStream, cudaStreamNonBlocking));
        if (!e->evCov) {
            HV_CUDA(cudaEventCreateWithFlags(&e->evCovFork, cudaEventDisableTiming));
            HV_CUDA(cudaEventCreateWithFlags(&e->evCov, cudaEventDisableTiming));
        }
        HV_CUDA(cudaEventRecord(e->evCovFork, c->stream));        // behind everything issued so far (earlier filter work, the mean launch)
        HV_CUDA(cudaStreamWaitEvent(c->covStream, e->evCovFork, 0));
        if (e->sideBusy) HV_CUDA(cudaStreamWaitEvent(c->covStream, e->evJoin, 0));     // ... and behind the covariance on the side stream
        HV_CUDA(ekf_launch_predict(a, c->covStream));
        HV_CUDA(cudaEventRecord(e->evCov, c->covStream));
        e->covBusy = true;
    } else {
        int rc = join_cov(e);
        if (rc == HV_OK) rc = join_side(e);
        if (rc != HV_OK) return rc;
        HV_CUDA(ekf_launch_predict(a, e->ctx->stream));
    }
    e->meanIssued = false;
    e->ctx->launches++;
    a.count = 0;
    return HV_OK;
}

static int flush_predicts(hv_ekf* e) { return predict_launch(e, e->pend); }
static int flush_sym(hv_ekf* e)
{
    if (!e->pendSym) return HV_OK;
    e->pendSym = false;
    int rc = join_cov(e);
    if (rc != HV_OK) return rc;
    return launch_ew(e, EKF_EW_SYMMETRIZE);
}
// At most one kind of work is pending at a time (predict() issues a pending symmetrisation first, symmetrize() issues
// pending samples first), so the order of the reference's calls is preserved.
static int flush_pending(hv_ekf* e)
{
    int rc = flush_predicts(e);
    if (rc != HV_OK) return rc;
    rc = join_cov(e);                                  // the caller is about to touch the filter on the context's stream
    if (rc != HV_OK) return rc;
    return flush_sym(e);
}

int hv_ekf_predict(hv_ekf* e, double t, const double xg[3], const double xa[3])
{
    EKF_ENTER_LAZY(e, "hv_ekf_predict");
    int rc = flush_sym(e);
    if (rc != HV_OK) return rc;
    predict_bookkeep(e, t, xg, xa, e->pend);
    if (e->pend.count >= e->imuBatch) return flush_predicts(e);
    return HV_OK;
}

int hv_ekf_predicted_mean_device(hv_ekf* e, double* dMean20)
{
    EKF_ENTER_LAZY(e, "hv_ekf_predicted_mean_device");
    if (!dMean20) { hv_set_error("hv_ekf_predicted_mean_device: NULL output"); return HV_ERR_INVALID; }
    int rc = join_cov(e);                                         // (a covariance launch of an earlier burst writes the mean as well)
    if (rc != HV_OK) return rc;
    rc = flush_sym(e);
    if (rc != HV_OK) return rc;
    cudaStream_t s = e->ctx->stream;
    if (e->pend.count == 0) {                                     // nothing queued: the state as it is
        HV_CUDA(cudaMemcpyAsync(dMean20, e->b.m, sizeof(double) * EKF_INER, cudaMemcpyDeviceToDevice, s));
        return HV_OK;
    }
    EkfPredictArgs a = e->pend;                                   // the queue stays: the full launch follows with the next call that needs P
    a.b = e->b; a.gravity = e->prm.gravity; a.meanOut = dMean20;
    HV_CUDA(ekf_launch_predict(a, s));
    e->ctx->launches++;
    e->meanIssued = true;
    return HV_OK;
}

int hv_ekf_predicted_mean(hv_ekf* e, double* mean20)
{
    EKF_ENTER_LAZY(e, "hv_ekf_predicted_mean");
    if (!mean20) { hv_set_error("hv_ekf_predicted_mean: NULL output"); return HV_ERR_INVALID; }
    int rc = staging_acquire(e);
    if (rc != HV_OK) return rc;
    rc = hv_ekf_predicted_mean_device(e, e->d_mean20);
    if (rc != HV_OK) return rc;
    double* hout = e->h_pin;
    HV_CUDA(cudaMemcpyAsync(hout, e->d_mean20, sizeof(double) * EKF_INER, cudaMemcpyDeviceToHost, e->ctx->stream));
    HV_CUDA(cudaStreamSynchronize(e->ctx->stream));
    memcpy(mean20, hout, sizeof(double) * EKF_INER);
    return HV_OK;
}

int hv_ekf_flush(hv_ekf* e)
{
    EKF_ENTER_LAZY(e, "hv_ekf_flush");
    int rc = flush_predicts(e);                        // (may go to the covariance stream: not joined here, see join_cov)
    if (rc != HV_OK) return rc;
    if (e->pendSym) { rc = join_cov(e); if (rc != HV_OK) return rc; return flush_sym(e); }
    return HV_OK;
}

int hv_ekf_set_imu_batching(hv_ekf* e, int max_samples)
{
    EKF_ENTER(e, "hv_ekf_set_imu_batching");
    if (max_samples < 1 || max_samples > EKF_MAX_PREDICT) { hv_set_error("hv_ekf_set_imu_batching: 1..%d", EKF_MAX_PREDICT); return HV_ERR_INVALID; }
    e->imuBatch = max_samples;
    return HV_OK;
}

int hv_ekf_update_zupt(hv_ekf* e, double r)
{
    EKF_ENTER(e, "hv_ekf_update_zupt");
    if (e->time - e->ZUPTtime < 0.25) return HV_OK;          // ekf.cpp:574-578
    e->ZUPTtime = e->time; e->wasStationary = true;
    EkfUpdateArgs a; fill_small(a, EKF_OP_ZUPT, 3, EKF_VEL + 3, r * e->noiseScale);
    return launch_update(e, a);
}

int hv_ekf_update_zupt_initialization(hv_ekf* e)
{
    EKF_ENTER(e, "hv_ekf_update_zupt_initialization");
    if (e->wasStationary || e->time > 60 || e->time - e->initZUPTtime < 0.1) return HV_OK;   // ekf.cpp:598-601
    e->initZUPTtime = e->time;
    EkfUpdateArgs a; fill_small(a, EKF_OP_ZUPT, 3, EKF_VEL + 3, e->prm.init_zupt_r * e->noiseScale * std::exp(0.5 * e->time));
    return launch_update(e, a);
}

int hv_ekf_update_zrupt(hv_ekf* e, const double xg[3])
{
    EKF_ENTER(e, "hv_ekf_update_zrupt");
    if (e->time - e->ZRUPTtime < 0.25) return HV_OK;         // ekf.cpp:615-618
    e->ZRUPTtime = e->time;
    EkfUpdateArgs a; fill_small(a, EKF_OP_ZRUPT, 3, EKF_BGA + 3, e->prm.rotation_zupt_r * e->noiseScale);
    for (int i = 0; i < 3; i++) a.ysmall[i] = xg[i];
    return launch_update(e, a);
}

int hv_ekf_update_pseudo_velocity(hv_ekf* e, double defaultSpeed, double r)
{
    EKF_ENTER(e, "hv_ekf_update_pseudo_velocity");
    EkfUpdateArgs a; fill_small(a, EKF_OP_PSEUDO_VELOCITY, 1, EKF_VEL + 2, r * e->noiseScale);
    a.defaultSpeed = defaultSpeed;
    return launch_update(e, a);
}

int hv_ekf_update_position(hv_ekf* e, const double y[3], double r)
{
    EKF_ENTER(e, "hv_ekf_update_position");
    EkfUpdateArgs a; fill_small(a, EKF_OP_POSITION, 3, EKF_POS + 3, r * e->noiseScale);
    for (int i = 0; i < 3; i++) a.ysmall[i] = y[i];
    a.symmetrize = 1;
    return launch_update(e, a);
}

int hv_ekf_update_zero_height(hv_ekf* e, double r)
{
    EKF_ENTER(e, "hv_ekf_update_zero_height");
    EkfUpdateArgs a; fill_small(a, EKF_OP_ZERO_HEIGHT, 1, EKF_POS + 3, r * e->noiseScale);
    a.symmetrize = 1;
    return launch_update(e, a);
}

int hv_ekf_update_orientation(hv_ekf* e, const double q[4], double r)
{
    EKF_ENTER(e, "hv_ekf_update_orientation");
    EkfUpdateArgs a; fill_small(a, EKF_OP_ORIENTATION, 4, EKF_ORI + 4, r * e->noiseScale);
    for (int i = 0; i < 4; i++) a.ysmall[i] = q[i];
    a.normalizeAll = 1; a.symmetrize = 1;
    return launch_update(e, a);
}

static int visual_args(hv_ekf* e, const char* who, int n, int l, double r, double rmseThr, int mode, EkfUpdateArgs& a)
{
    if (n <= 0 || l <= 0 || l > e->N || n > e->N) {   // maxHRows = stateDim (ekf.cpp:177-180)
        hv_set_error("%s: bad shape n=%d l=%d (N=%d)", who, n, l, e->N); return HV_ERR_INVALID;
    }
    if (mode != EKF_MODE_UPDATE && n >= (int)e->chi2inv95.size()) { hv_set_error("%s: n=%d exceeds the chi2 table", who, n); return HV_ERR_INVALID; }
    memset(&a, 0, sizeof(a));
    a.op = EKF_OP_DENSE; a.n = n; a.l = l; a.mode = mode;
    a.Rdiag = (r * r) * e->noiseScale;                          // ekf.cpp:777
    a.rmseThr = mode == EKF_MODE_UPDATE ? -1.0 : rmseThr;
    a.chi2Thr = mode == EKF_MODE_UPDATE ? 0.0 : e->chi2inv95[n];
    a.skipChi2 = (mode != EKF_MODE_UPDATE && r < 0.0) ? 1 : 0;
    a.normalizeAll = 1;
    return HV_OK;
}

// The pinned staging block is shared by all calls; an asynchronous call (updateVisualTrack) returns while its H2D copy may
// still be queued, so the next call must not refill the block before that copy has read it.
static int staging_acquire(hv_ekf* e)
{
    if (e->stagedPending) { HV_CUDA(cudaEventSynchronize(e->evStaged)); e->stagedPending = false; }
    return HV_OK;
}
static int staging_release(hv_ekf* e)      // call right after the H2D copy has been enqueued
{
    HV_CUDA(cudaEventRecord(e->evStaged, e->ctx->stream));
    e->stagedPending = true;
    return HV_OK;
}

// Waits for `count` result slots of the mapped buffer to carry sequence number seq (written by ekf_report).
static int poll_results(hv_ekf* e, int count, double seq, const char* who)
{
    int ready = 0;
    return hv_poll(e->ctx->stream, who, [&] {
        while (ready < count && ((volatile double*)e->h_sig)[4 * ready + 3] == seq) ready++;
        return ready == count;
    });
}

static int visual_host(hv_ekf* e, const char* who, const double* H, int n, int l, const double* f, const double* y, double r,
                       double rmseThr, int mode, int* vuStatus, double* chi2, double* mOut)
{
    if (!H || !f || !y) { hv_set_error("%s: NULL input", who); return HV_ERR_INVALID; }
    EkfUpdateArgs a;
    int rc = visual_args(e, who, n, l, r, rmseThr, mode, a);
    if (rc != HV_OK) return rc;
    cudaStream_t s = e->ctx->stream;
    const size_t nl = (size_t)n * l, inD = nl + 2 * (size_t)n;
    double* hin = e->h_pin;
    if (mode == EKF_MODE_UPDATE && !mOut && e->spec.valid) {
        // updateVisualTrack right behind an INLIER visualTrackOutlierCheck of the SAME measurement (the reference's per-track loop,
        // backend.cpp:1158-1185): the check kernel has already produced the updated state with this noise level in P2 / m2 -- adopt it.
        const bool same = e->spec.epoch == e->epoch && e->spec.n == n && e->spec.l == l && r == e->specR &&
                          memcmp(hin, H, nl * sizeof(double)) == 0 && memcmp(hin + nl, f, n * sizeof(double)) == 0 && memcmp(hin + nl + n, y, n * sizeof(double)) == 0;
        e->spec.valid = false;
        if (same) {
            double* t = e->b.P; e->b.P = e->b.P2; e->b.P2 = t;
            t = e->b.m; e->b.m = e->m2; e->m2 = t;
            e->epoch++;
            return HV_OK;
        }
    }
    if (e->spec.valid) e->specEnabled = false;     // an INLIER check that was NOT followed by its update: stop speculating until an update call comes again
    e->spec.valid = false;
    if (mode == EKF_MODE_UPDATE) { e->specR = r; e->specEnabled = true; }
    rc = staging_acquire(e);
    if (rc != HV_OK) return rc;
    memcpy(hin, H, nl * sizeof(double)); memcpy(hin + nl, f, n * sizeof(double)); memcpy(hin + nl + n, y, n * sizeof(double));
    HV_CUDA(cudaMemcpyAsync(e->d_in, hin, inD * sizeof(double), cudaMemcpyHostToDevice, s));
    rc = staging_release(e);
    if (rc != HV_OK) return rc;
    a.H = e->d_in; a.f = e->d_in + nl; a.y = e->d_in + nl + n;
    const bool polled = mode != EKF_MODE_UPDATE && !mOut;
    if (polled) { a.sig = e->d_sig; a.sigSeq = (e->sigSeq += 1.0); }
    // A pure check speculates: the same kernel goes on to compute the update the reference issues for an INLIER (with the noise level of the
    // previous updateVisualTrack) into P2 / m2, while the host already has the decision; P and m stay as they are. Only the cluster kernel
    // has the second buffers (the single-CTA kernel would update P in place).
    const bool speculate = mode == EKF_MODE_CHECK && e->specEnabled && e->specR > 0.0 && !a.skipChi2 && a.rmseThr < 0.0 && r > 0.0 &&
                           ekf_cluster2_fits(n, l, e->N, false);
    if (speculate) {
        int rcj = join_side(e);
        if (rcj != HV_OK) return rcj;
        a.mode = EKF_MODE_CHECK_UPDATE; a.Rdiag2 = (e->specR * e->specR) * e->noiseScale;
        a.specP = e->b.P2; a.specM = e->m2;
    }
    rc = launch_update(e, a);
    if (rc != HV_OK) return rc;
    if (mode == EKF_MODE_UPDATE && !mOut) return HV_OK;          // asynchronous
    if (polled) {
        // the kernel writes (status, chi2, flag) into mapped pinned memory the moment the decision is known; a check+update
        // carries on with the update while the host already prepares its next call (which is stream-ordered behind it)
        rc = poll_results(e, 1, a.sigSeq, who);
        if (rc != HV_OK) return rc;
        if (vuStatus) *vuStatus = (int)e->h_sig[0];
        if (chi2) *chi2 = e->h_sig[1];
        if (e->h_sig[2] != 0.0) { hv_set_error("%s: innovation covariance not positive definite", who); return HV_ERR_STATE; }
        if (speculate && e->h_sig[0] == 0.0) { e->spec.valid = true; e->spec.epoch = e->epoch; e->spec.n = n; e->spec.l = l; }
        return HV_OK;
    }
    double* hout = e->h_pin + e->inDoubles;
    HV_CUDA(cudaMemcpyAsync(hout, e->b.res, 3 * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (mOut) HV_CUDA(cudaMemcpyAsync(hout + 8, e->b.m, e->N * sizeof(double), cudaMemcpyDeviceToHost, s));
    HV_CUDA(cudaStreamSynchronize(s));
    if (vuStatus) *vuStatus = (int)hout[0];
    if (chi2) *chi2 = hout[1];
    if (mOut) memcpy(mOut, hout + 8, e->N * sizeof(double));
    if (hout[2] != 0.0) { hv_set_error("%s: innovation covariance not positive definite", who); return HV_ERR_STATE; }
    return HV_OK;
}

int hv_ekf_visual_check(hv_ekf* e, const double* H, int n, int l, const double* f, const double* y, double r, double rmseThr,
                        int* vuStatus, double* chi2)
{
    EKF_ENTER(e, "hv_ekf_visual_check");
    return visual_host(e, "hv_ekf_visual_check", H, n, l, f, y, r, rmseThr, EKF_MODE_CHECK, vuStatus, chi2, nullptr);
}

int hv_ekf_visual_update(hv_ekf* e, const double* H, int n, int l, const double* f, const double* y, double r)
{
    EKF_ENTER(e, "hv_ekf_visual_update");
    return visual_host(e, "hv_ekf_visual_update", H, n, l, f, y, r, -1.0, EKF_MODE_UPDATE, nullptr, nullptr, nullptr);
}

int hv_ekf_visual_check_update(hv_ekf* e, const double* H, int n, int l, const double* f, const double* y, double r, double rmseThr,
                               int* vuStatus, double* chi2, double* mOut)
{
    EKF_ENTER(e, "hv_ekf_visual_check_update");
    return visual_host(e, "hv_ekf_visual_check_update", H, n, l, f, y, r, rmseThr, EKF_MODE_CHECK_UPDATE, vuStatus, chi2, mOut);
}

static int visual_device_args(hv_ekf* e, const double* dH, int n, int l, const double* df, const double* dy, double r, double rmseThr,
                              int mode, int lateH, double* slot, EkfUpdateArgs& a)
{
    if (!dH || !df || !dy || mode < 0 || mode > 2) { hv_set_error("hv_ekf_visual_device: invalid argument"); return HV_ERR_INVALID; }
    int rc = visual_args(e, "hv_ekf_visual_device", n, l, r, rmseThr, mode, a);
    if (rc != HV_OK) return rc;
    a.H = dH; a.f = df; a.y = dy;
    // caller-owned device pointers: H may have been produced by the caller's previous kernel on this stream (hv_ctx_create_on_stream),
    // so it is staged AFTER griddepcontrol.wait; early staging is kept for H that arrived through the library's own H2D copy
    a.lateH = lateH;
    a.slot = slot;                                                 // the kernel writes its result words into the slot itself
    return HV_OK;
}
static int visual_device(hv_ekf* e, const double* dH, int n, int l, const double* df, const double* dy, double r, double rmseThr,
                         int mode, double* dResult, int lateH, double* slot = nullptr)
{
    EkfUpdateArgs a;
    int rc = visual_device_args(e, dH, n, l, df, dy, r, rmseThr, mode, lateH, slot, a);
    if (rc != HV_OK) return rc;
    rc = launch_update(e, a);
    if (rc != HV_OK) return rc;
    if (dResult) HV_CUDA(cudaMemcpyAsync(dResult, e->b.res, 2 * sizeof(double), cudaMemcpyDeviceToDevice, e->ctx->stream));
    return HV_OK;
}

int hv_ekf_visual_device(hv_ekf* e, const double* dH, int n, int l, const double* df, const double* dy, double r, double rmseThr,
                         int mode, double* dResult)
{
    EKF_ENTER(e, "hv_ekf_visual_device");
    return visual_device(e, dH, n, l, df, dy, r, rmseThr, mode, dResult, 1);
}

// Argument block of the pose augmentation (ekf.cpp:848-885); symFirst: a deferred maintainPositiveSemiDefinite() rides along
static void augment_args(hv_ekf* e, int discarded, bool symFirst, EkfUpdateArgs& a)
{
    fill_small(a, EKF_OP_AUGMENT, EKF_POSE, EKF_CAM + EKF_POSE, e->prm.augment_r * e->noiseScale);
    a.b = e->b;
    a.symFirst = symFirst ? 1 : 0;
    a.dropIdx = discarded;
    a.augNoisePos = pow2(e->prm.noise_initial_pos_trail) * e->noiseScale;
    a.augNoiseOri = pow2(e->prm.noise_initial_ori_trail) * e->noiseScale;
    a.normalizeAll = 1; a.symmetrize = 1;
}
static void augment_done(hv_ekf* e)
{
    e->augmentTimes.push_back(hv_ekf_platform_time(e));          // ekf.cpp:876-884
    if (e->augmentCount < e->trail) e->augmentCount++;
    else e->augmentTimes.erase(e->augmentTimes.begin());
}

int hv_ekf_augment(hv_ekf* e, int discarded)
{
    EKF_ENTER_LAZY(e, "hv_ekf_augment");
    int rcf = flush_predicts(e);
    if (rcf == HV_OK) rcf = join_cov(e);
    if (rcf != HV_OK) return rcf;
    if (discarded == -1) discarded = e->trail - 1;               // ekf.cpp:849
    if (discarded < 0 || discarded >= e->trail) { hv_set_error("hv_ekf_augment: pose index %d out of range", discarded); return HV_ERR_INVALID; }
    EkfUpdateArgs a; augment_args(e, discarded, e->pendSym, a);  // a deferred symmetrisation rides along
    e->pendSym = false;
    int rc = launch_update(e, a);   // (single-CTA kernel: shift into P2, update there, Joseph product back into P: no swap)
    if (rc != HV_OK) return rc;
    augment_done(e);
    return HV_OK;
}

int hv_ekf_unaugment(hv_ekf* e)
{
    EKF_ENTER(e, "hv_ekf_unaugment");
    if (e->augmentCount <= 0) { hv_set_error("hv_ekf_unaugment: no augmented pose (ekf.cpp:899 asserts)"); return HV_ERR_STATE; }
    int rc = launch_ew(e, EKF_EW_UNAUGMENT);
    if (rc != HV_OK) return rc;
    swap_P(e);
    e->augmentTimes.pop_back(); e->augmentCount--;
    return HV_OK;
}

int hv_ekf_symmetrize(hv_ekf* e)
{
    EKF_ENTER(e, "hv_ekf_symmetrize");
    // deferred: rides along with a directly following augmentation (cluster kernel), otherwise issued by the next call
    e->pendSym = true;
    return HV_OK;
}
int hv_ekf_normalize_quaternions(hv_ekf* e, int onlyCurrent)
{
    EKF_ENTER_LAZY(e, "hv_ekf_normalize_quaternions");
    if (onlyCurrent && e->pend.count > 0 && !e->pend.s[e->pend.count - 1].normAfter) {
        e->pend.s[e->pend.count - 1].normAfter = 1;              // folded into the deferred predict launch
        return HV_OK;
    }
    int rc = flush_pending(e);
    if (rc != HV_OK) return rc;
    return launch_ew(e, EKF_EW_NORMALIZE, onlyCurrent ? 1 : 0);
}
int hv_ekf_translate_to(hv_ekf* e, const double pos[3]) { EKF_ENTER(e, "hv_ekf_translate_to"); return launch_ew(e, EKF_EW_TRANSLATE, 0, pos, 3); }

int hv_ekf_transform_to(hv_ekf* e, const double pos[3], const double q[4], int poseIndex)
{
    EKF_ENTER(e, "hv_ekf_transform_to");
    if (poseIndex < -1 || poseIndex >= e->trail) { hv_set_error("hv_ekf_transform_to: pose index out of range"); return HV_ERR_INVALID; }
    const double dv[7] = {pos[0], pos[1], pos[2], q[0], q[1], q[2], q[3]};
    int rc = launch_ew(e, EKF_EW_TRANSFORM, poseIndex, dv, 7);
    if (rc != HV_OK) return rc;
    swap_P(e);
    return HV_OK;
}

int hv_ekf_insert_map_point(hv_ekf* e, int idx, const double pf[3])
{
    EKF_ENTER(e, "hv_ekf_insert_map_point");
    const int off = e->N - e->mapDim + idx * EKF_MAP_POINT;      // getMapPointStateIndex (ekf.cpp:923-926)
    if (idx < 0 || off + EKF_MAP_POINT > e->N) { hv_set_error("hv_ekf_insert_map_point: index out of range"); return HV_ERR_INVALID; }
    return launch_ew(e, EKF_EW_INSERT_MAP_POINT, off, pf, 3);
}

int hv_ekf_condition_on_last_pose(hv_ekf* e)
{
    EKF_ENTER(e, "hv_ekf_condition_on_last_pose");
    if (e->mapDim != 0 || e->augmentCount <= 0) { hv_set_error("hv_ekf_condition_on_last_pose: needs no hybrid map and >= 1 augmented pose"); return HV_ERR_STATE; }
    return launch_ew(e, EKF_EW_CONDITION_LAST_POSE);
}

// An op list that continues "[SYMMETRIZE,] AUGMENT" behind a run of outlier checks (the end of a frame, backend.cpp): the augmentation does
// not depend on the checks and the checks only read (m, P), so it is issued as one more cluster of the same launch, writing into the
// second buffers (P2 / m2), which are swapped in afterwards. Returns the number of ops consumed behind the checks (0: no fusion).
static int augment_follows(const hv_ekf* e, const hv_ekf_op* ops, int nops, int k, int* discarded, bool* symFirst)
{
    int used = 0;
    *symFirst = false;
    if (k < nops && ops[k].kind == HV_EKF_OP_SYMMETRIZE) { *symFirst = true; used = 1; }
    if (k + used >= nops || ops[k + used].kind != HV_EKF_OP_AUGMENT) return 0;
    int d = ops[k + used].index;
    if (d == -1) d = e->trail - 1;
    if (d < 0 || d >= e->trail) return 0;                        // the plain path reports the error
    if (!ekf_cluster2_fits(EKF_POSE, EKF_CAM + EKF_POSE, e->N, true)) return 0;
    *discarded = d;
    return used + 1;
}
static void adopt_second_buffers(hv_ekf* e)
{
    swap_P(e);
    double* t = e->b.m; e->b.m = e->m2; e->m2 = t;
    e->epoch++;
    e->spec.valid = false;
}

// Argument block of the first of `count` consecutive outlier checks and one batch item per check, with the list's measurement pointers
static int check_items(hv_ekf* e, const hv_ekf_op* ops, int first, int count, EkfUpdateArgs& a, EkfCheckBatch& b)
{
    memset(&b, 0, sizeof(b));
    b.count = count;
    for (int i = 0; i < count; i++) {
        const hv_ekf_op& o = ops[first + i];
        EkfUpdateArgs tmp;
        int rc = visual_args(e, "hv_ekf_run", o.n, o.l, o.r, o.rmse_thr, EKF_MODE_CHECK, tmp);
        if (rc != HV_OK) return rc;
        if (i == 0) a = tmp;
        if (!o.H || !o.f || !o.y) { hv_set_error("hv_ekf_run: op %d: NULL input", first + i); return HV_ERR_INVALID; }
        EkfCheckItem& it = b.it[i];
        it.n = o.n; it.l = o.l; it.Rdiag = tmp.Rdiag; it.chi2Thr = tmp.chi2Thr; it.rmseThr = tmp.rmseThr; it.skipChi2 = tmp.skipChi2;
        it.H = o.H; it.f = o.f; it.y = o.y;
    }
    return HV_OK;
}
// The augmentation that shares the launch of the checks before it: results into the second buffers
static void fused_augment_args(hv_ekf* e, int discarded, bool symFirst, EkfUpdateArgs& aug)
{
    augment_args(e, discarded, symFirst, aug);
    aug.noiseScale = e->noiseScale; aug.specP = e->b.P2; aug.specM = e->m2;
}

// A run of consecutive check-only VISUAL ops (mode 0) reads the same (m, P) and is therefore issued as ONE launch
// (one cluster per measurement); with host buffers it is also one H2D copy, one D2H copy and one synchronisation.
static int flush_checks(hv_ekf* e, const hv_ekf_op* ops, int first, int count, bool host, int* vuStatus, double* chi2, int augDiscarded = -1, bool augSym = false)
{
    if (count == 0) return HV_OK;
    cudaStream_t s = e->ctx->stream;
    EkfUpdateArgs a; EkfCheckBatch b;
    int rci = check_items(e, ops, first, count, a, b);
    if (rci == HV_OK) rci = join_side(e);             // (the checks read P; an augmentation writes the buffers earlier checks read)
    if (rci != HV_OK) return rci;
    if (host) {
        int rc = staging_acquire(e);
        if (rc != HV_OK) return rc;
        size_t off = 0;
        for (int i = 0; i < count; i++) {
            const hv_ekf_op& o = ops[first + i];
            EkfCheckItem& it = b.it[i];
            const size_t nl = (size_t)o.n * o.l;
            double* hin = e->h_pin + off;
            memcpy(hin, o.H, nl * sizeof(double)); memcpy(hin + nl, o.f, o.n * sizeof(double)); memcpy(hin + nl + o.n, o.y, o.n * sizeof(double));
            it.H = e->d_in + off; it.f = e->d_in + off + nl; it.y = e->d_in + off + nl + o.n;
            off += nl + 2 * (size_t)o.n;
        }
        HV_CUDA(cudaMemcpyAsync(e->d_in, e->h_pin, off * sizeof(double), cudaMemcpyHostToDevice, s));
        rc = staging_release(e);
        if (rc != HV_OK) return rc;
    }
    a.b = e->b; a.noiseScale = e->noiseScale;
    if (host) { a.sig = e->d_sig; a.sigSeq = (e->sigSeq += 1.0); }       // every item fits the cluster kernel (batchable_check)
    if (!host && first + count <= HV_RUN_MAX_OPS) a.slot = e->d_opres + 4 * first;      // hv_ekf_run_device_results
    if (augDiscarded >= 0) {
        EkfUpdateArgs aug; fused_augment_args(e, augDiscarded, augSym, aug);
        // HV_EKF_NO_PDL=1 (throughput mode, many sessions per GPU): nothing is launched early or beside the main stream
        static const bool latencyMode = getenv("HV_EKF_NO_PDL") == nullptr;
        if (host || !latencyMode || !ekf_aug_mean_fits(e->N)) {
            // results are wanted now (or: one stream per session): the augmentation is one more cluster of the checks' launch
            HV_CUDA(ekf_launch_check_batch2(a, b, s, &aug));
        } else {
            // nothing goes back to the host: the checks and the augmentation's covariance leave the main stream (fork -> side stream, one
            // launch, P2 written there), and the augmentation's mean is formed on the main stream by one CTA (m2): the next frame's mean
            // propagation and optical flow, which read the mean only, run beside the covariance; its consumers of P join the side stream
            if (!e->ctx->sideStream) HV_CUDA(cudaStreamCreateWithFlags(&e->ctx->sideStream, cudaStreamNonBlocking));
            if (!e->evFork) {
                HV_CUDA(cudaEventCreateWithFlags(&e->evFork, cudaEventDisableTiming));
                HV_CUDA(cudaEventCreateWithFlags(&e->evJoin, cudaEventDisableTiming));
            }
            cudaStream_t side = e->ctx->sideStream;
            HV_CUDA(cudaEventRecord(e->evFork, s));
            HV_CUDA(cudaStreamWaitEvent(side, e->evFork, 0));
            a.b.cwork = e->cworkSide; a.b.res = e->resSide;
            EkfUpdateArgs augCov = aug;                   // the cluster's mean goes to a scratch buffer: m2 has one writer, the kernel below
            augCov.b.cwork = e->cworkSide; augCov.b.res = e->resSide; augCov.specM = e->mSide;
            HV_CUDA(ekf_launch_check_batch2(a, b, side, &augCov));
            HV_CUDA(cudaEventRecord(e->evJoin, side));
            e->sideBusy = true;
            e->ctx->launches++;
            HV_CUDA(ekf_launch_aug_mean(aug, s));
        }
        adopt_second_buffers(e);
        augment_done(e);
    } else HV_CUDA(ekf_launch_check_batch2(a, b, s));
    e->ctx->launches++;
    if (host) {
        int rc = poll_results(e, count, a.sigSeq, "hv_ekf_run");
        if (rc != HV_OK) return rc;
        for (int i = 0; i < count; i++) {
            if (vuStatus) vuStatus[first + i] = (int)e->h_sig[4 * i];
            if (chi2) chi2[first + i] = e->h_sig[4 * i + 1];
            if (e->h_sig[4 * i + 2] != 0.0) { hv_set_error("hv_ekf_run: op %d: innovation covariance not positive definite", first + i); return HV_ERR_STATE; }
        }
    }
    return HV_OK;
}

static bool batchable_check(const hv_ekf* e, const hv_ekf_op& o)
{
    return o.kind == HV_EKF_OP_VISUAL && o.mode == 0 && o.n > 0 && o.l > 0 && o.l <= e->N && o.n <= e->N &&
           ekf_cluster2_fits(o.n, o.l, e->N, false);
}

static void note_visual_ops(hv_ekf* e, const hv_ekf_op* ops, int nops)       // which slots of d_opres a list fills (hv_ekf_run_device_results)
{
    e->lastVisual.assign(nops, 0);
    for (int i = 0; i < nops && i < HV_RUN_MAX_OPS; i++) if (ops[i].kind == HV_EKF_OP_VISUAL) e->lastVisual[i] = 1;
}

static int run_ops(hv_ekf* e, const hv_ekf_op* ops, int nops, bool host, int* vuStatus, double* chi2, double* mOut)
{
    if (!ops || nops < 0) { hv_set_error("hv_ekf_run: invalid argument"); return HV_ERR_INVALID; }
    if (!host) note_visual_ops(e, ops, nops);
    for (int i = 0; i < nops; i++) {
        const hv_ekf_op& o = ops[i];
        int rc = HV_OK;
        if (o.kind == HV_EKF_OP_VISUAL) { rc = flush_pending(e); if (rc != HV_OK) return rc; }   // the other kinds enter through their own entry points
        if (batchable_check(e, o)) {
            int cnt = 1;
            while (i + cnt < nops && cnt < EKF_MAX_BATCH && batchable_check(e, ops[i + cnt])) cnt++;
            int disc = -1; bool sym = false;
            const int extra = augment_follows(e, ops, nops, i + cnt, &disc, &sym);
            rc = flush_checks(e, ops, i, cnt, host, vuStatus, chi2, extra ? disc : -1, sym);
            if (rc != HV_OK) return rc;
            i += cnt - 1 + extra;
            continue;
        }
        switch (o.kind) {
            case HV_EKF_OP_PREDICT: rc = hv_ekf_predict(e, o.t, o.gyro, o.acc); break;
            case HV_EKF_OP_VISUAL:
                if (o.mode < 0 || o.mode > 2) { hv_set_error("hv_ekf_run: op %d: bad mode", i); return HV_ERR_INVALID; }
                if (host) rc = visual_host(e, "hv_ekf_run_host", o.H, o.n, o.l, o.f, o.y, o.r, o.rmse_thr, o.mode,
                                           vuStatus ? vuStatus + i : nullptr, chi2 ? chi2 + i : nullptr, nullptr);
                else rc = visual_device(e, o.H, o.n, o.l, o.f, o.y, o.r, o.rmse_thr, o.mode, nullptr, 0,       // prepared inputs (see the header): staged early
                                        i < HV_RUN_MAX_OPS ? e->d_opres + 4 * i : nullptr);
                break;
            case HV_EKF_OP_SYMMETRIZE: rc = hv_ekf_symmetrize(e); break;
            case HV_EKF_OP_AUGMENT: rc = hv_ekf_augment(e, o.index); break;
            case HV_EKF_OP_UNAUGMENT: rc = hv_ekf_unaugment(e); break;
            case HV_EKF_OP_NORMALIZE: rc = hv_ekf_normalize_quaternions(e, o.index); break;
            default: hv_set_error("hv_ekf_run: op %d: unknown kind %d", i, o.kind); return HV_ERR_INVALID;
        }
        if (rc != HV_OK) return rc;
    }
    if (host && mOut) return hv_ekf_download(e, mOut, nullptr);
    return HV_OK;
}

// hv_ekf_run_host without a round trip per measurement: the list is known up front and a check+update decides on the device whether
// its update is applied, so nothing the host would do depends on an intermediate result. Every measurement gets its own slice of the
// pinned staging block (the host stages and issues op i+1 while the GPU works on op i), the kernels write their result words into a
// mapped pinned area (one 4-double slot per op), and the ONE synchronisation at the end also covers the state read-back.
// Leaves *handled = 0 if the list cannot be handled here (too long, staging too small, an invalid visual op: run_ops reports it).
static int run_ops_host_async(hv_ekf* e, const hv_ekf_op* ops, int nops, int* vuStatus, double* chi2, double* mOut, int* handled)
{
    *handled = 0;
    if (nops > HV_RUN_MAX_OPS) return HV_OK;
    size_t need = 0;
    for (int i = 0; i < nops; i++) {
        const hv_ekf_op& o = ops[i];
        if (o.kind != HV_EKF_OP_VISUAL) continue;
        if (o.mode < 0 || o.mode > 2 || !o.H || !o.f || !o.y || o.n <= 0 || o.l <= 0 || o.l > e->N || o.n > e->N) return HV_OK;
        need += (size_t)o.n * o.l + 2 * (size_t)o.n;
    }
    if (need > e->inDoubles) return HV_OK;
    *handled = 1;
    const auto tHost0 = std::chrono::steady_clock::now();
    cudaStream_t s = e->ctx->stream;
    if (!e->copyStream) HV_CUDA(cudaStreamCreateWithFlags(&e->copyStream, cudaStreamNonBlocking));
    cudaStream_t cs = e->copyStream;
    int rc = staging_acquire(e);
    if (rc != HV_OK) return rc;
    // kernels queued by earlier asynchronous calls (updateVisualTrack) may still read the device input block: the copies start behind them
    HV_CUDA(cudaEventRecord(e->evStaged, s));
    HV_CUDA(cudaStreamWaitEvent(cs, e->evStaged, 0));
    const double seq = (e->sigSeq += 1.0);
    size_t off = 0;
    bool staged = false;
    int group = 0;
    for (int i = 0; i < nops; i++) {
        const hv_ekf_op& o = ops[i];
        rc = HV_OK;
        if (o.kind == HV_EKF_OP_VISUAL) {
            rc = flush_pending(e);
            if (rc != HV_OK) return rc;
            // consecutive pure checks that fit the cluster kernel: one launch (one cluster per track)
            const bool batch = batchable_check(e, o);
            int cnt = 1;
            if (batch) while (i + cnt < nops && cnt < EKF_MAX_BATCH && batchable_check(e, ops[i + cnt])) cnt++;
            EkfUpdateArgs a; EkfCheckBatch b;
            memset(&b, 0, sizeof(b));
            b.count = cnt;
            for (int j = 0; j < cnt; j++) {
                const hv_ekf_op& q = ops[i + j];
                EkfUpdateArgs t;
                rc = visual_args(e, "hv_ekf_run_host", q.n, q.l, q.r, q.rmse_thr, q.mode, t);
                if (rc != HV_OK) return rc;
                const size_t nl = (size_t)q.n * q.l, tot = nl + 2 * (size_t)q.n;
                // The inputs go to the device on the COPY stream (they depend on nothing the kernels produce), so that they run ahead of
                // the kernels instead of sitting between them. A packed measurement (f = H + n l, y = f + n) in page-locked memory is
                // copied straight from the caller's buffer; anything else is packed into the pinned staging block first.
                bool direct = false;
                if (q.f == q.H + nl && q.y == q.f + q.n) {
                    cudaPointerAttributes at;
                    if (cudaPointerGetAttributes(&at, q.H) == cudaSuccess && at.type == cudaMemoryTypeHost) direct = true;
                    else cudaGetLastError();
                }
                if (direct) HV_CUDA(cudaMemcpyAsync(e->d_in + off, q.H, tot * sizeof(double), cudaMemcpyHostToDevice, cs));
                else {
                    double* hin = e->h_pin + off;
                    memcpy(hin, q.H, nl * sizeof(double)); memcpy(hin + nl, q.f, q.n * sizeof(double)); memcpy(hin + nl + q.n, q.y, q.n * sizeof(double));
                    HV_CUDA(cudaMemcpyAsync(e->d_in + off, hin, tot * sizeof(double), cudaMemcpyHostToDevice, cs));
                    staged = true;
                }
                t.H = e->d_in + off; t.f = e->d_in + off + nl; t.y = e->d_in + off + nl + q.n;
                off += tot;
                if (j == 0) a = t;
                EkfCheckItem& it = b.it[j];
                it.n = q.n; it.l = q.l; it.Rdiag = t.Rdiag; it.chi2Thr = t.chi2Thr; it.rmseThr = t.rmseThr; it.skipChi2 = t.skipChi2;
                it.H = t.H; it.f = t.f; it.y = t.y;
            }
            if ((int)e->copyEvents.size() <= group) { cudaEvent_t ev; HV_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming)); e->copyEvents.push_back(ev); }
            HV_CUDA(cudaEventRecord(e->copyEvents[group], cs));
            HV_CUDA(cudaStreamWaitEvent(s, e->copyEvents[group], 0));
            group++;
            a.sig = e->d_run + 4 * i; a.sigSeq = seq;
            int disc = -1; bool sym = false;
            const int extra = batch ? augment_follows(e, ops, nops, i + cnt, &disc, &sym) : 0;
            if (cnt > 1 || extra) {
                rc = join_side(e);
                if (rc != HV_OK) return rc;
                a.b = e->b; a.noiseScale = e->noiseScale;
                if (extra) {
                    EkfUpdateArgs aug; augment_args(e, disc, sym, aug);
                    aug.noiseScale = e->noiseScale; aug.specP = e->b.P2; aug.specM = e->m2;
                    HV_CUDA(ekf_launch_check_batch2(a, b, s, &aug));
                    adopt_second_buffers(e);
                    augment_done(e);
                } else HV_CUDA(ekf_launch_check_batch2(a, b, s));
                e->ctx->launches++;
            } else {
                rc = launch_update(e, a);
                if (rc != HV_OK) return rc;
            }
            i += cnt - 1 + extra;
            continue;
        }
        switch (o.kind) {
            case HV_EKF_OP_PREDICT: rc = hv_ekf_predict(e, o.t, o.gyro, o.acc); break;
            case HV_EKF_OP_SYMMETRIZE: rc = hv_ekf_symmetrize(e); break;
            case HV_EKF_OP_AUGMENT: rc = hv_ekf_augment(e, o.index); break;
            case HV_EKF_OP_UNAUGMENT: rc = hv_ekf_unaugment(e); break;
            case HV_EKF_OP_NORMALIZE: rc = hv_ekf_normalize_quaternions(e, o.index); break;
            default: hv_set_error("hv_ekf_run: op %d: unknown kind %d", i, o.kind); return HV_ERR_INVALID;
        }
        if (rc != HV_OK) return rc;
    }
    (void)staged;            // the staging block is free again after the synchronisation below (the copies precede the kernels that wait for them)
    rc = flush_pending(e);
    if (rc != HV_OK) return rc;
    double* hout = e->h_pin + e->inDoubles;
    if (!mOut && need == 0) return HV_OK;                        // nothing to hand back (e.g. the IMU burst of a frame): fully asynchronous
    if (mOut) HV_CUDA(cudaMemcpyAsync(hout + 8, e->b.m, e->N * sizeof(double), cudaMemcpyDeviceToHost, s));
    const auto tHost1 = std::chrono::steady_clock::now();
    HV_CUDA(cudaStreamSynchronize(s));                           // the only synchronisation of the list
    {
        const auto tHost2 = std::chrono::steady_clock::now();
        auto us = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) { return std::chrono::duration<double, std::micro>(b - a).count(); };
        e->hostTimes[0] = us(tHost0, tHost1); e->hostTimes[1] = us(tHost1, tHost2); e->hostTimes[2] = us(tHost0, tHost2); e->hostTimes[3] = nops;
    }
    __atomic_thread_fence(__ATOMIC_ACQUIRE);
    if (mOut) memcpy(mOut, hout + 8, e->N * sizeof(double));
    for (int i = 0; i < nops; i++) {
        if (ops[i].kind != HV_EKF_OP_VISUAL) continue;
        const volatile double* w = e->h_run + 4 * i;
        if (w[3] != seq) { hv_set_error("hv_ekf_run_host: op %d did not report its result", i); return HV_ERR_STATE; }
        if (vuStatus) vuStatus[i] = (int)w[0];
        if (chi2) chi2[i] = w[1];
        if (w[2] != 0.0) { hv_set_error("hv_ekf_run: op %d: innovation covariance not positive definite", i); return HV_ERR_STATE; }
    }
    return HV_OK;
}

int hv_ekf_run_device(hv_ekf* e, const hv_ekf_op* ops, int nops)
{
    EKF_ENTER(e, "hv_ekf_run_device");
    return run_ops(e, ops, nops, false, nullptr, nullptr, nullptr);
}

int hv_ekf_run_device_results(hv_ekf* e, int nops, int* vuStatus, double* chi2)
{
    EKF_ENTER(e, "hv_ekf_run_device_results");
    if (nops < 0 || nops > (int)e->lastVisual.size() || nops > HV_RUN_MAX_OPS) { hv_set_error("hv_ekf_run_device_results: the last list had %d ops (at most %d report)", (int)e->lastVisual.size(), HV_RUN_MAX_OPS); return HV_ERR_INVALID; }
    int rc = join_side(e);
    if (rc != HV_OK) return rc;
    int rca = staging_acquire(e);
    if (rca != HV_OK) return rca;
    double* hout = e->h_pin;                                      // (inDoubles >= 4 HV_RUN_MAX_OPS for every state size)
    HV_CUDA(cudaMemcpyAsync(hout, e->d_opres, sizeof(double) * 4 * nops, cudaMemcpyDeviceToHost, e->ctx->stream));
    HV_CUDA(cudaStreamSynchronize(e->ctx->stream));
    for (int i = 0; i < nops; i++) {
        if (!e->lastVisual[i]) continue;
        if (vuStatus) vuStatus[i] = (int)hout[4 * i];
        if (chi2) chi2[i] = hout[4 * i + 1];
        if (hout[4 * i + 2] != 0.0) { hv_set_error("hv_ekf_run_device_results: op %d: innovation covariance not positive definite", i); return HV_ERR_STATE; }
    }
    return HV_OK;
}

// ---------------------------------------------------------------------------------------------------- a group of filters
// hv_ekf_group_run_device: every list is cut into the steps run_ops issues for it -- an IMU burst, one visual update, a run of outlier
// checks with the augmentation that follows them as one more cluster, an augmentation -- and step k of every filter goes into one launch
// per kernel, so that a group of filters takes the launches of one. The instances of a step belong to different filters, and step k of
// a filter is stream-ordered behind its step k - 1.
struct GroupStep {
    bool predict = false;
    EkfPredictArgs p;                       // predict: the burst
    std::vector<EkfUpdateArgs> u;           // otherwise: one argument block per cluster
};

static int group_refuse(int rc, int f, int i, const char* what)
{
    hv_set_error("hv_ekf_group_run_device: filter %d, op %d: %s", f, i, what);
    return rc;
}

// Checks a list against the group's vocabulary (see the header) without changing anything: a dry run of the IMU bookkeeping
// (predict_bookkeep, the burst length) tells whether each NORMALIZE folds into the sample before it.
static int group_check_list(hv_ekf* e, const hv_ekf_op* ops, int nops, int f)
{
    if (!ops || nops < 0) return group_refuse(HV_ERR_INVALID, f, -1, "NULL list or negative length");
    bool firstSample = e->firstSample, normed = false;
    double prevT = e->prevSampleT;
    int pend = 0;                                        // (the queue is issued before the list: flush_pending)
    for (int i = 0; i < nops; i++) {
        const hv_ekf_op& o = ops[i];
        switch (o.kind) {
        case HV_EKF_OP_PREDICT: {
            double dt = 0.0;
            if (!firstSample) dt = o.t - prevT; else firstSample = false;
            prevT = o.t;
            if (dt <= 0.0) break;
            pend++; normed = false;
            if (pend >= e->imuBatch) pend = 0;
        } break;
        case HV_EKF_OP_NORMALIZE:
            if (!o.index || pend == 0 || normed) return group_refuse(HV_ERR_UNSUPPORTED, f, i, "NORMALIZE that does not fold into the IMU sample before it");
            normed = true;
            break;
        case HV_EKF_OP_VISUAL: {
            if (o.mode < 0 || o.mode > 2) return group_refuse(HV_ERR_INVALID, f, i, "bad mode");
            if (!o.H || !o.f || !o.y) return group_refuse(HV_ERR_INVALID, f, i, "NULL measurement");
            EkfUpdateArgs a;
            const int rc = visual_args(e, "hv_ekf_group_run_device", o.n, o.l, o.r, o.rmse_thr, o.mode, a);
            if (rc != HV_OK) return rc;
            if (!ekf_cluster2_fits(o.n, o.l, e->N, false)) return group_refuse(HV_ERR_UNSUPPORTED, f, i, "measurement does not fit the cluster kernel whole");
            pend = 0;
        } break;
        case HV_EKF_OP_SYMMETRIZE:
            if (i + 1 >= nops || ops[i + 1].kind != HV_EKF_OP_AUGMENT) return group_refuse(HV_ERR_UNSUPPORTED, f, i, "SYMMETRIZE not followed by AUGMENT");
            pend = 0;
            break;
        case HV_EKF_OP_AUGMENT: {
            const int d = o.index == -1 ? e->trail - 1 : o.index;
            if (d < 0 || d >= e->trail) return group_refuse(HV_ERR_INVALID, f, i, "discarded pose index out of range");
            if (!ekf_cluster2_fits(EKF_POSE, EKF_CAM + EKF_POSE, e->N, true)) return group_refuse(HV_ERR_UNSUPPORTED, f, i, "augmentation does not fit the cluster kernel");
            pend = 0;
        } break;
        case HV_EKF_OP_UNAUGMENT: return group_refuse(HV_ERR_UNSUPPORTED, f, i, "UNAUGMENT");
        default: return group_refuse(HV_ERR_INVALID, f, i, "unknown kind");
        }
    }
    return HV_OK;
}

// What ekf_check_batch_cluster2_kernel makes of (a, b, aug) for its cluster inst
static EkfUpdateArgs check_instance(const EkfUpdateArgs& a, const EkfCheckBatch& b, const EkfUpdateArgs& aug, int inst)
{
    EkfUpdateArgs r = a;
    if (inst >= b.count) r = aug;
    else {
        const EkfCheckItem& it = b.it[inst];
        r.H = it.H; r.f = it.f; r.y = it.y; r.n = it.n; r.l = it.l;
        r.Rdiag = it.Rdiag; r.chi2Thr = it.chi2Thr; r.rmseThr = it.rmseThr; r.skipChi2 = it.skipChi2;
        if (r.sig) r.sig += 4 * inst;
        if (r.slot) r.slot += 4 * inst;
    }
    r.b.res += (size_t)EKF_RES_STRIDE * inst;
    r.b.cwork += (size_t)inst * 10 * r.b.N * r.b.N;
    return r;
}

// The steps of one filter's (checked) list, with the host bookkeeping of every op done as run_ops does it
static int group_steps(hv_ekf* e, const hv_ekf_op* ops, int nops, std::vector<GroupStep>& st)
{
    int rc = flush_pending(e);                           // work queued by earlier calls goes first
    if (rc == HV_OK) rc = join_side(e);
    if (rc != HV_OK) return rc;
    note_visual_ops(e, ops, nops);
    auto burst = [&]() {
        if (e->pend.count == 0) return;
        st.emplace_back();
        st.back().predict = true;
        st.back().p = e->pend;
        predict_settle(e, st.back().p);
        e->meanIssued = false;
        e->pend.count = 0;
    };
    for (int i = 0; i < nops; i++) {
        const hv_ekf_op& o = ops[i];
        if (o.kind == HV_EKF_OP_PREDICT) {
            predict_bookkeep(e, o.t, o.gyro, o.acc, e->pend);
            if (e->pend.count >= e->imuBatch) burst();
            continue;
        }
        if (o.kind == HV_EKF_OP_NORMALIZE) { e->pend.s[e->pend.count - 1].normAfter = 1; continue; }
        burst();
        st.emplace_back();
        std::vector<EkfUpdateArgs>& u = st.back().u;
        if (batchable_check(e, o)) {
            int cnt = 1;
            while (i + cnt < nops && cnt < EKF_MAX_BATCH && batchable_check(e, ops[i + cnt])) cnt++;
            int disc = -1; bool sym = false;
            const int extra = augment_follows(e, ops, nops, i + cnt, &disc, &sym);
            EkfUpdateArgs a, aug; EkfCheckBatch b;
            rc = check_items(e, ops, i, cnt, a, b);
            if (rc != HV_OK) return rc;
            a.b = e->b; a.noiseScale = e->noiseScale;
            if (i + cnt <= HV_RUN_MAX_OPS) a.slot = e->d_opres + 4 * i;
            if (extra) fused_augment_args(e, disc, sym, aug);
            else aug = a;
            for (int j = 0; j < cnt + (extra ? 1 : 0); j++) u.push_back(check_instance(a, b, aug, j));
            if (extra) { adopt_second_buffers(e); augment_done(e); }
            i += cnt - 1 + extra;
        } else if (o.kind == HV_EKF_OP_VISUAL) {
            EkfUpdateArgs a;
            rc = visual_device_args(e, o.H, o.n, o.l, o.f, o.y, o.r, o.rmse_thr, o.mode, 0, i < HV_RUN_MAX_OPS ? e->d_opres + 4 * i : nullptr, a);
            if (rc != HV_OK) return rc;
            update_settle(e, a);
            u.push_back(a);
        } else {                                                  // [SYMMETRIZE,] AUGMENT
            const bool sym = o.kind == HV_EKF_OP_SYMMETRIZE;
            const int d = ops[i + sym].index;
            EkfUpdateArgs a;
            augment_args(e, d == -1 ? e->trail - 1 : d, sym, a);
            update_settle(e, a);
            u.push_back(a);
            augment_done(e);
            i += sym;
        }
    }
    return HV_OK;
}

// Staging of a group call's argument blocks: pinned block `ekfStageNext` of the context's ring (refilled once the copy out of it has
// completed) and the device block (reused in stream order: the copy into it follows the kernels that read it before)
static int group_stage(hv_ctx* c, size_t bytes, char** h, char** d, cudaEvent_t* ev)
{
    const int i = c->ekfStageNext;
    if (!c->evEkfStage[i]) HV_CUDA(cudaEventCreateWithFlags(&c->evEkfStage[i], cudaEventDisableTiming));
    else HV_CUDA(cudaEventSynchronize(c->evEkfStage[i]));
    size_t cap = 4096;
    while (cap < bytes) cap *= 2;
    if (bytes > c->h_ekfStageBytes[i]) {
        if (c->h_ekfStage[i]) cudaFreeHost(c->h_ekfStage[i]);
        c->h_ekfStage[i] = nullptr; c->h_ekfStageBytes[i] = 0;
        HV_CUDA(cudaMallocHost(&c->h_ekfStage[i], cap));
        c->h_ekfStageBytes[i] = cap;
    }
    if (bytes > c->ekfStageBytes) {
        if (c->d_ekfStage) HV_CUDA(cudaFreeAsync(c->d_ekfStage, c->stream));
        c->d_ekfStage = nullptr; c->ekfStageBytes = 0;
        HV_CUDA(cudaMallocAsync(&c->d_ekfStage, cap, c->stream));
        c->ekfStageBytes = cap;
    }
    c->ekfStageNext = (i + 1) % HV_EKF_STAGES;
    *h = (char*)c->h_ekfStage[i]; *d = (char*)c->d_ekfStage; *ev = c->evEkfStage[i];
    return HV_OK;
}

int hv_ekf_group_run_device(hv_ekf* const* ekfs, int count, const hv_ekf_op* const* ops, const int* nops)
{
    if (!ekfs || !ops || !nops || count < 1 || count > HV_EKF_GROUP_MAX) {
        hv_set_error("hv_ekf_group_run_device: NULL array or count %d outside 1..%d", count, HV_EKF_GROUP_MAX); return HV_ERR_INVALID;
    }
    for (int f = 0; f < count; f++) {
        hv_ekf* e = ekfs[f];
        if (!e) return group_refuse(HV_ERR_INVALID, f, -1, "NULL filter");
        if (e->ctx != ekfs[0]->ctx) return group_refuse(HV_ERR_INVALID, f, -1, "filter of another context");
        if (e->N != ekfs[0]->N) return group_refuse(HV_ERR_INVALID, f, -1, "state dimension differs from filter 0");
        for (int g = 0; g < f; g++) if (ekfs[g] == e) return group_refuse(HV_ERR_INVALID, f, -1, "filter appears twice");
        const int rc = group_check_list(e, ops[f], nops[f], f);
        if (rc != HV_OK) return rc;
    }
    hv_ctx* c = ekfs[0]->ctx;
    HV_CUDA(cudaSetDevice(c->device));
    std::vector<std::vector<GroupStep>> steps(count);
    size_t nsteps = 0;
    for (int f = 0; f < count; f++) {
        const int rc = group_steps(ekfs[f], ops[f], nops[f], steps[f]);
        if (rc != HV_OK) return rc;
        nsteps = std::max(nsteps, steps[f].size());
    }
    // one predict and one cluster launch per step: their argument arrays one after the other in the staging block
    struct Launch { size_t off; int count; bool predict; };
    std::vector<Launch> launches;
    std::vector<size_t> predOff(nsteps), updOff(nsteps);
    size_t bytes = 0;
    auto align16 = [](size_t v) { return (v + 15) & ~(size_t)15; };
    for (size_t k = 0; k < nsteps; k++) {
        int np = 0, nu = 0;
        for (int f = 0; f < count; f++) if (k < steps[f].size()) { if (steps[f][k].predict) np++; else nu += (int)steps[f][k].u.size(); }
        predOff[k] = bytes;
        if (np) { launches.push_back({bytes, np, true}); bytes = align16(bytes + np * sizeof(EkfPredictArgs)); }
        updOff[k] = bytes;
        if (nu) { launches.push_back({bytes, nu, false}); bytes = align16(bytes + nu * sizeof(EkfUpdateArgs)); }
    }
    if (launches.empty()) return HV_OK;
    char *h = nullptr, *d = nullptr; cudaEvent_t ev = nullptr;
    int rc = group_stage(c, bytes, &h, &d, &ev);
    if (rc != HV_OK) return rc;
    for (size_t k = 0; k < nsteps; k++) {
        EkfPredictArgs* hp = (EkfPredictArgs*)(h + predOff[k]);
        EkfUpdateArgs* hu = (EkfUpdateArgs*)(h + updOff[k]);
        for (int f = 0; f < count; f++) {
            if (k >= steps[f].size()) continue;
            const GroupStep& s = steps[f][k];
            if (s.predict) *hp++ = s.p;
            else for (const EkfUpdateArgs& a : s.u) *hu++ = a;
        }
    }
    HV_CUDA(cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, c->stream));
    HV_CUDA(cudaEventRecord(ev, c->stream));
    for (const Launch& L : launches) {
        if (L.predict) HV_CUDA(ekf_launch_group_predict((const EkfPredictArgs*)(h + L.off), (const EkfPredictArgs*)(d + L.off), L.count, c->stream));
        else HV_CUDA(ekf_launch_group_cluster2((const EkfUpdateArgs*)(h + L.off), (const EkfUpdateArgs*)(d + L.off), L.count, c->stream));
        c->launches++;
    }
    return HV_OK;
}

int hv_ekf_run_host(hv_ekf* e, const hv_ekf_op* ops, int nops, int* vuStatus, double* chi2, double* mOut)
{
    EKF_ENTER(e, "hv_ekf_run_host");
    if (!ops || nops < 0) { hv_set_error("hv_ekf_run: invalid argument"); return HV_ERR_INVALID; }
    int handled = 0;
    const int rc = run_ops_host_async(e, ops, nops, vuStatus, chi2, mOut, &handled);
    if (handled || rc != HV_OK) return rc;
    return run_ops(e, ops, nops, true, vuStatus, chi2, mOut);
}

int hv_ekf_debug_host_times(hv_ekf* e, double* out4)
{
    if (!e || !out4) { hv_set_error("hv_ekf_debug_host_times: NULL"); return HV_ERR_INVALID; }
    for (int i = 0; i < 4; i++) out4[i] = e->hostTimes[i];
    return HV_OK;
}

int hv_ekf_debug_result_words(hv_ekf* e, double* out32)
{
    EKF_ENTER(e, "hv_ekf_debug_result_words");
    if (!out32) { hv_set_error("hv_ekf_debug_result_words: NULL output"); return HV_ERR_INVALID; }
    HV_CUDA(cudaMemcpyAsync(out32, e->b.res, 32 * sizeof(double), cudaMemcpyDeviceToHost, e->ctx->stream));
    HV_CUDA(cudaStreamSynchronize(e->ctx->stream));
    return HV_OK;
}

// ---------------------------------------------------------------------------------------------------- per-track measurement model
void hv_camera_model_defaults(hv_camera_model* c)
{
    if (!c) return;
    memset(c, 0, sizeof(*c));
    c->estimate_imu_camera_time_shift = 1;
    c->gauss_newton_iterations = 10; c->convergence_threshold = 1e-2; c->convergence_r = 11.0; c->rcond_threshold = 1e-8;
    c->min_dist = 0.0; c->max_dist = 1e300;
}

int hv_ekf_set_camera_model(hv_ekf* e, const hv_camera_model* c)
{
    EKF_ENTER_LAZY(e, "hv_ekf_set_camera_model");
    if (!c || c->gauss_newton_iterations < 1) { hv_set_error("hv_ekf_set_camera_model: invalid argument"); return HV_ERR_INVALID; }
    bool zero = true;
    for (int i = 0; i < 16; i++) zero = zero && c->imu_to_camera[i] == 0.0;
    if (zero) { hv_set_error("hv_ekf_set_camera_model: imu_to_camera is the zero sentinel (triangulation.cpp:78-79)"); return HV_ERR_INVALID; }
    if (!e->tm) e->tm = new TrackModels();
    e->tm->cam = *c; e->tm->camSet = true;
    return HV_OK;
}

static int tm_reserve(TrackModels* t, int n)
{
    if (n <= t->cap) return HV_OK;
    int cap = t->cap ? t->cap : 64;
    while (cap < n) cap *= 2;
    t->release();
    HV_CUDA(cudaMalloc(&t->d_in, TrackModels::inBytes(cap)));
    HV_CUDA(cudaMalloc(&t->d_out, TrackModels::outBytes(cap)));
    HV_CUDA(cudaMalloc(&t->d_dpf, sizeof(double) * cap * 3 * (7 * TM_MAXPOSE + 1)));
    HV_CUDA(cudaMalloc(&t->d_H, sizeof(double) * cap * TrackModels::hStride()));
    HV_CUDA(cudaMalloc(&t->d_f, sizeof(double) * cap * 2 * TM_MAXOBS));
    HV_CUDA(cudaHostAlloc(&t->h_in, TrackModels::inBytes(cap), cudaHostAllocDefault));
    HV_CUDA(cudaHostAlloc(&t->h_out, TrackModels::outBytes(cap), cudaHostAllocDefault));
    t->cap = cap;
    return HV_OK;
}

// The checks of tm_submit: a camera model, and well-formed tracks
static int tm_validate(const hv_ekf* e, const char* who, const hv_track_obs* tracks, int ntracks)
{
    const TrackModels* t = e->tm;
    if (!t || !t->camSet) { hv_set_error("%s: hv_ekf_set_camera_model has not been called", who); return HV_ERR_STATE; }
    if (!tracks || ntracks < 1) { hv_set_error("%s: invalid argument", who); return HV_ERR_INVALID; }
    const int maxIndex = e->trail < TM_MAXPOSE - 1 ? e->trail : TM_MAXPOSE - 1;
    for (int k = 0; k < ntracks; k++) {
        const hv_track_obs& o = tracks[k];
        if (o.npose < 2 || o.npose > TM_MAXPOSE || !o.pose_trail_index || !o.ip || !o.velocities) {
            hv_set_error("%s: track %d: npose %d outside 2..%d or NULL arrays", who, k, o.npose, TM_MAXPOSE); return HV_ERR_INVALID;
        }
        for (int i = 0; i < o.npose; i++)
            if (o.pose_trail_index[i] < 0 || o.pose_trail_index[i] > maxIndex) {
                hv_set_error("%s: track %d: pose index %d outside 0..%d", who, k, o.pose_trail_index[i], maxIndex); return HV_ERR_INVALID;
            }
    }
    return HV_OK;
}

// Validates a batch of tracks, packs it into the pinned block, enqueues the H2D copies and fills the kernel arguments
// (everything except ntracks / trackOffset / counter).
static int tm_submit(hv_ekf* e, const char* who, const hv_track_obs* tracks, int ntracks, TmArgs& a)
{
    int rc = tm_validate(e, who, tracks, ntracks);
    if (rc != HV_OK) return rc;
    TrackModels* t = e->tm;
    const int ncam = t->cam.use_stereo ? 2 : 1;
    rc = tm_reserve(t, ntracks);
    if (rc != HV_OK) return rc;
    cudaStream_t s = e->ctx->stream;
    // pack: the block layout is fixed by the capacity, so that the live ranges are three contiguous copies
    const int cap = t->cap;
    int* h_np = (int*)t->h_in;
    int* h_idx = h_np + cap;
    double* h_ip = (double*)(t->h_in + sizeof(int) * (size_t)cap * (TM_MAXPOSE + 2));
    double* h_vel = h_ip + (size_t)cap * 2 * TM_MAXOBS;
    for (int k = 0; k < ntracks; k++) {
        const hv_track_obs& o = tracks[k];
        h_np[k] = o.npose;
        memcpy(h_idx + (size_t)k * TM_MAXPOSE, o.pose_trail_index, sizeof(int) * o.npose);
        memcpy(h_ip + (size_t)k * 2 * TM_MAXOBS, o.ip, sizeof(double) * 2 * o.npose * ncam);
        memcpy(h_vel + (size_t)k * 2 * TM_MAXOBS, o.velocities, sizeof(double) * 2 * o.npose * ncam);
    }
    HV_CUDA(cudaMemcpyAsync(t->d_in, t->h_in, sizeof(int) * ((size_t)cap + (size_t)ntracks * TM_MAXPOSE), cudaMemcpyHostToDevice, s));
    const size_t ipOff = sizeof(int) * (size_t)cap * (TM_MAXPOSE + 2), velOff = ipOff + sizeof(double) * (size_t)cap * 2 * TM_MAXOBS;
    HV_CUDA(cudaMemcpyAsync(t->d_in + ipOff, t->h_in + ipOff, sizeof(double) * (size_t)ntracks * 2 * TM_MAXOBS, cudaMemcpyHostToDevice, s));
    HV_CUDA(cudaMemcpyAsync(t->d_in + velOff, t->h_in + velOff, sizeof(double) * (size_t)ntracks * 2 * TM_MAXOBS, cudaMemcpyHostToDevice, s));
    memset(&a, 0, sizeof(a));
    a.m = e->b.m; a.N = e->N; a.stereo = t->cam.use_stereo ? 1 : 0; a.timeShift = t->cam.estimate_imu_camera_time_shift ? 1 : 0; a.ntracks = ntracks;
    for (int c = 0; c < 2; c++) {
        const double* T = c ? t->cam.second_imu_to_camera : t->cam.imu_to_camera;
        for (int r = 0; r < 3; r++) { for (int k = 0; k < 3; k++) a.Rc[c][3 * r + k] = T[4 * k + r]; a.base[c][r] = T[12 + r]; }
    }
    a.gnIterations = t->cam.gauss_newton_iterations; a.convThreshold = t->cam.convergence_threshold; a.convR = t->cam.convergence_r;
    a.rcondThreshold = t->cam.rcond_threshold; a.minDist = t->cam.min_dist; a.maxDist = t->cam.max_dist;
    a.npose = (const int*)t->d_in; a.idx = a.npose + cap;
    a.ip = (const double*)(t->d_in + ipOff); a.vel = (const double*)(t->d_in + velOff);
    a.status = (int*)t->d_out; a.pf = (double*)(t->d_out + sizeof(int) * 4 * (size_t)cap);
    a.dpf = t->d_dpf; a.H = t->d_H; a.f = t->d_f; a.Hstride = TrackModels::hStride();
    t->last = ntracks; t->lastNpose.resize(ntracks);
    for (int k = 0; k < ntracks; k++) t->lastNpose[k] = tracks[k].npose;
    return HV_OK;
}

// D2H of the status / point words of tracks [first, first + count) (asynchronous)
static int tm_fetch(hv_ekf* e, int first, int count)
{
    TrackModels* t = e->tm;
    cudaStream_t s = e->ctx->stream;
    const size_t pfOff = sizeof(int) * 4 * (size_t)t->cap;
    HV_CUDA(cudaMemcpyAsync(t->h_out + sizeof(int) * 4 * (size_t)first, t->d_out + sizeof(int) * 4 * (size_t)first, sizeof(int) * 4 * (size_t)count, cudaMemcpyDeviceToHost, s));
    HV_CUDA(cudaMemcpyAsync(t->h_out + pfOff + sizeof(double) * 4 * (size_t)first, t->d_out + pfOff + sizeof(double) * 4 * (size_t)first,
                            sizeof(double) * 4 * (size_t)count, cudaMemcpyDeviceToHost, s));
    return HV_OK;
}

static void tm_result(const hv_ekf* e, const TmArgs& a, int k, hv_track_model& o)
{
    const TrackModels* t = e->tm;
    const int* st = (const int*)t->h_out;
    const double* pf = (const double*)(t->h_out + sizeof(int) * 4 * (size_t)t->cap);
    o.triangulator_status = st[4 * k]; o.prepare_vu_status = st[4 * k + 1]; o.rows = st[4 * k + 2]; o.cols = st[4 * k + 3];
    for (int r = 0; r < 3; r++) o.pf[r] = pf[4 * k + r];
    o.depth = pf[4 * k + 3];
    o.d_H = t->d_H + (size_t)k * TrackModels::hStride();
    o.d_f = t->d_f + (size_t)k * 2 * TM_MAXOBS;
    o.d_y = a.ip + (size_t)k * 2 * TM_MAXOBS;
}

int hv_ekf_track_models(hv_ekf* e, const hv_track_obs* tracks, int ntracks, hv_track_model* out)
{
    EKF_ENTER(e, "hv_ekf_track_models");
    if (!out) { hv_set_error("hv_ekf_track_models: invalid argument"); return HV_ERR_INVALID; }
    TmArgs a;
    int rc = tm_submit(e, "hv_ekf_track_models", tracks, ntracks, a);
    if (rc != HV_OK) return rc;
    cudaStream_t s = e->ctx->stream;
    HV_CUDA(tm_launch(a, s));
    e->ctx->launches++;
    e->tm->lastArgs = a;
    rc = tm_fetch(e, 0, ntracks);
    if (rc != HV_OK) return rc;
    HV_CUDA(cudaStreamSynchronize(s));
    for (int k = 0; k < ntracks; k++) tm_result(e, a, k, out[k]);
    return HV_OK;
}

// Columns of H of a track: the truncation of prepareVisualUpdate (triangulation.cpp:909-921)
static int track_cols(const hv_track_obs& o)
{
    int l = 0;
    for (int i = 0; i < o.npose; i++) { const int x = o.pose_trail_index[i]; const int end = x == 0 ? 10 : 20 + 7 * (x - 1) + 7; if (end > l) l = end; }
    return l;
}

// The per-track loop of Session::trackerVisualUpdate (src/odometry/backend.cpp:1012-1252, per-track mode) as ONE stream-ordered
// chain with the control flow on the device: for every track  model(state) -> outlier check -> update if inlier,  each kernel
// gated by words the previous ones wrote (model valid, fewer than max_successful_updates so far, check said INLIER). The host
// synchronises once per `lookahead` tracks instead of twice per track. A chain belongs to one filter: hv_ekf_visual_tracks issues it
// alone, hv_ekf_group_visual_tracks track by track beside the chains of other filters; both through the chain_* functions below.
struct VisualChain {
    const hv_track_obs* tracks = nullptr;
    int ntracks = 0;
    hv_visual_update_params p;
    TmArgs base;                            // the model arguments of the whole batch (tm_submit)
    std::vector<int> chunkRows;             // per track: 0 = the cluster kernel on the whole measurement, else its row-chunked form
    int* d_counter = nullptr;               // control block (TrackModels::d_ctl): success counter, then per track the result slots of
    double* d_slots = nullptr;              // check (4 doubles) and update (4 doubles)
    int maxSucc = 0, step = 0;              // step: tracks per host synchronisation
    bool fused = false;                     // check and update of a track in ONE kernel
    int issued = 0, succ = 0;               // tracks issued and successful updates, as of the last synchronisation
};

// Every track's kernel form up front: the cluster kernel on the whole measurement, or its row-chunked form beside the resident P
// blocks; a chain that contains a track neither fits is refused before anything is issued (tm_submit reports malformed tracks)
static int chain_forms(const hv_ekf* e, const char* who, const hv_track_obs* tracks, int ntracks, std::vector<int>& chunkRows)
{
    chunkRows.assign(ntracks > 0 ? ntracks : 0, 0);
    if (!e->tm || !e->tm->camSet || !tracks) return HV_OK;
    const int ncam = e->tm->cam.use_stereo ? 2 : 1;
    for (int k = 0; k < ntracks; k++) {
        const hv_track_obs& o = tracks[k];
        if (o.npose < 2 || o.npose > TM_MAXPOSE || !o.pose_trail_index) continue;
        const int n = 2 * o.npose * ncam, l = track_cols(o);
        if (ekf_cluster2_fits(n, l, e->N, false)) continue;
        chunkRows[k] = ekf_cluster2_chunk_rows(n, l, e->N);
        if (chunkRows[k] == 0) {
            hv_set_error("%s: track %d (n=%d, l=%d): state dimension %d too large for the cluster kernel, even in row chunks", who, k, n, l, e->N);
            return HV_ERR_UNSUPPORTED;
        }
    }
    return HV_OK;
}

// What precedes the chain's first kernel: the tracks' inputs on the device (tm_submit) and the success counter reset
static int chain_begin(hv_ekf* e, const char* who, const hv_track_obs* tracks, int ntracks, const hv_visual_update_params* p, VisualChain& ch)
{
    int rc = chain_forms(e, who, tracks, ntracks, ch.chunkRows);
    if (rc != HV_OK) return rc;
    rc = tm_submit(e, who, tracks, ntracks, ch.base);
    if (rc != HV_OK) return rc;
    TrackModels* t = e->tm;
    if (t->ctlCap < t->cap) {
        cudaFree(t->d_ctl); cudaFreeHost(t->h_ctl); t->d_ctl = t->h_ctl = nullptr; t->ctlCap = 0;
        HV_CUDA(cudaMalloc(&t->d_ctl, TrackModels::ctlBytes(t->cap)));
        HV_CUDA(cudaHostAlloc(&t->h_ctl, TrackModels::ctlBytes(t->cap), cudaHostAllocDefault));
        t->ctlCap = t->cap;
    }
    ch.d_counter = (int*)t->d_ctl;
    ch.d_slots = (double*)(t->d_ctl + 16);
    HV_CUDA(cudaMemsetAsync(t->d_ctl, 0, 16, e->ctx->stream));
    ch.tracks = tracks; ch.ntracks = ntracks; ch.p = *p;
    ch.maxSucc = p->max_successful_updates > 0 ? p->max_successful_updates : 0x7fffffff;
    ch.step = p->lookahead > 0 ? p->lookahead : ntracks;
    // check and update of a track in ONE kernel (S0 = H P H' formed once, factorised with each of the two R): one launch
    // fewer per track than separate gated check / update launches.
    ch.fused = p->chi_outlier_r >= 0.0 && p->visual_r > 0.0;
    ch.issued = ch.succ = 0;
    return HV_OK;
}

static bool chain_open(const VisualChain& ch) { return ch.issued < ch.ntracks && ch.succ < ch.maxSucc; }      // another window to issue
static int chain_window(const VisualChain& ch) { return std::min(ch.step, ch.ntracks - ch.issued); }         // its length

// The argument blocks of track k, settled for issue in this order: the model m, the check (fused: check + update) c and, unless the
// chain is fused, the update u. pdl: m follows a kernel of the chain on the stream.
static int chain_track(hv_ekf* e, const char* who, const VisualChain& ch, int k, int pdl, TmArgs& m, EkfUpdateArgs& c, EkfUpdateArgs& u)
{
    m = ch.base;
    m.ntracks = 1; m.trackOffset = k; m.counter = ch.d_counter; m.counterMax = ch.maxSucc; m.pdl = pdl;
    const TrackModels* t = e->tm;
    const hv_track_obs& o = ch.tracks[k];
    const int n = 2 * o.npose * (t->cam.use_stereo ? 2 : 1), l = track_cols(o);
    double* slotC = ch.d_slots + 8 * (size_t)k;
    int rc = visual_args(e, who, n, l, ch.p.chi_outlier_r, ch.p.track_rmse_threshold, ch.fused ? EKF_MODE_CHECK_UPDATE : EKF_MODE_CHECK, c);
    if (rc != HV_OK) return rc;
    c.H = t->d_H + (size_t)k * TrackModels::hStride(); c.f = t->d_f + (size_t)k * 2 * TM_MAXOBS; c.y = ch.base.ip + (size_t)k * 2 * TM_MAXOBS;
    c.gateI = ch.base.status + 4 * (size_t)k + 1; c.gateIExpect = 0; c.counter = ch.d_counter; c.counterMax = ch.maxSucc; c.slot = slotC; c.lateH = 1;
    if (ch.fused) { c.Rdiag2 = (ch.p.visual_r * ch.p.visual_r) * e->noiseScale; c.bump = ch.d_counter; }      // check with chi_outlier_r, update with visual_r, one kernel
    c.rowChunk = ch.chunkRows[k];
    update_settle(e, c);
    if (ch.fused) return HV_OK;
    rc = visual_args(e, who, n, l, ch.p.visual_r, -1.0, EKF_MODE_UPDATE, u);
    if (rc != HV_OK) return rc;
    u.H = c.H; u.f = c.f; u.y = c.y;
    u.gateD = slotC; u.gateDExpect = 0.0;                     // VuOutlierStatus::INLIER
    u.bump = ch.d_counter; u.slot = slotC + 4; u.lateH = 1; u.rowChunk = ch.chunkRows[k];
    update_settle(e, u);
    return HV_OK;
}

// D2H copies (asynchronous) of what the window [ch.issued, ch.issued + count) wrote: model words, success counter, result slots
static int chain_fetch(hv_ekf* e, const VisualChain& ch, int count)
{
    const int first = ch.issued;
    int rc = tm_fetch(e, first, count);
    if (rc != HV_OK) return rc;
    TrackModels* t = e->tm;
    cudaStream_t s = e->ctx->stream;
    HV_CUDA(cudaMemcpyAsync(t->h_ctl, t->d_ctl, 16, cudaMemcpyDeviceToHost, s));
    HV_CUDA(cudaMemcpyAsync(t->h_ctl + 16 + 64 * (size_t)first, t->d_ctl + 16 + 64 * (size_t)first, 64 * (size_t)count, cudaMemcpyDeviceToHost, s));
    return HV_OK;
}
// after the synchronisation behind chain_fetch(ch, count)
static void chain_synced(const hv_ekf* e, VisualChain& ch, int count)
{
    ch.succ = *(const int*)e->tm->h_ctl;
    ch.issued += count;
}

// Every track's record (tracks the chain never issued: not attempted) and the number of successful updates
static int chain_results(const hv_ekf* e, const char* who, const VisualChain& ch, hv_track_result* out, int* successfulUpdates)
{
    const double* slots = (const double*)(e->tm->h_ctl + 16);
    bool numeric = false;
    for (int k = 0; k < ch.ntracks; k++) {
        hv_track_result& o = out[k];
        memset(&o, 0, sizeof(o));
        if (k >= ch.issued) { o.triangulator_status = TM_SKIPPED; o.prepare_vu_status = TM_VU_NOT_RUN; o.outlier_status = 1; continue; }
        hv_track_model mdl;
        tm_result(e, ch.base, k, mdl);
        o.triangulator_status = mdl.triangulator_status; o.prepare_vu_status = mdl.prepare_vu_status;
        for (int r = 0; r < 3; r++) o.pf[r] = mdl.pf[r];
        o.depth = mdl.depth;
        const double* sc = slots + 8 * (size_t)k;
        o.outlier_status = (int)sc[0]; o.chi2 = sc[1];
        o.updated = ch.fused ? ((sc[0] == 0.0 && sc[2] == 0.0) ? 1 : 0) : ((sc[0] == 0.0 && sc[4] == 0.0 && sc[6] == 0.0) ? 1 : 0);
        numeric = numeric || sc[2] != 0.0 || (!ch.fused && sc[6] != 0.0);
    }
    if (successfulUpdates) *successfulUpdates = ch.succ;
    if (numeric) { hv_set_error("%s: innovation covariance not positive definite", who); return HV_ERR_STATE; }
    return HV_OK;
}

int hv_ekf_visual_tracks(hv_ekf* e, const hv_track_obs* tracks, int ntracks, const hv_visual_update_params* p, hv_track_result* out,
                         int* successfulUpdates)
{
    EKF_ENTER(e, "hv_ekf_visual_tracks");
    { int rcj = join_side(e); if (rcj != HV_OK) return rcj; }
    const char* who = "hv_ekf_visual_tracks";
    if (!p || !out) { hv_set_error("%s: invalid argument", who); return HV_ERR_INVALID; }
    VisualChain ch;
    int rc = chain_begin(e, who, tracks, ntracks, p, ch);
    if (rc != HV_OK) return rc;
    cudaStream_t s = e->ctx->stream;
    while (chain_open(ch)) {
        const int first = ch.issued, count = chain_window(ch);
        for (int k = first; k < first + count; k++) {
            TmArgs m; EkfUpdateArgs c, u;
            rc = chain_track(e, who, ch, k, k > first ? 1 : 0, m, c, u);     // pdl: behind a cluster kernel of this chain, overlap the launch with its tail
            if (rc != HV_OK) return rc;
            HV_CUDA(tm_launch(m, s));
            e->ctx->launches++;
            HV_CUDA(ekf_launch_update(c, s));
            e->ctx->launches++;
            if (ch.fused) continue;
            HV_CUDA(ekf_launch_update(u, s));
            e->ctx->launches++;
        }
        rc = chain_fetch(e, ch, count);
        if (rc != HV_OK) return rc;
        HV_CUDA(cudaStreamSynchronize(s));
        chain_synced(e, ch, count);
    }
    return chain_results(e, who, ch, out, successfulUpdates);
}

// ---------------------------------------------------------------------------------------------------- visual-update chains of a group
// hv_ekf_group_visual_tracks: step j issues the next track of every chain that has one left in its current window -- one launch of
// hv_track_model_group_kernel (a CTA per filter), one of ekf_group_cluster2_kernel (a cluster per filter: the check + update, or the check
// of a chain in the separate form) and, if a chain of the step uses the separate form, one more for the updates of those chains. Each
// chain keeps its own windows of `lookahead` tracks; the host synchronises, once for all, when a chain has reached the end of a window
// after which it may have to stop (a window that ends the list needs no decision).
int hv_ekf_group_visual_tracks(hv_ekf* const* ekfs, int count, const hv_track_obs* const* tracks, const int* ntracks,
                               const hv_visual_update_params* params, hv_track_result* const* out, int* successfulUpdates)
{
    const char* who = "hv_ekf_group_visual_tracks";
    if (!ekfs || !tracks || !ntracks || !params || !out || count < 1 || count > HV_EKF_GROUP_MAX) {
        hv_set_error("%s: NULL array or count %d outside 1..%d", who, count, HV_EKF_GROUP_MAX); return HV_ERR_INVALID;
    }
    // everything that can be refused, before anything is issued
    std::vector<std::string> whoF(count);               // "hv_ekf_group_visual_tracks: filter f" (error messages name the filter)
    for (int f = 0; f < count; f++) {
        char buf[64];
        snprintf(buf, sizeof(buf), "%s: filter %d", who, f);
        whoF[f] = buf;
        const char* wf = whoF[f].c_str();
        hv_ekf* e = ekfs[f];
        if (!e) { hv_set_error("%s: NULL filter", wf); return HV_ERR_INVALID; }
        if (e->ctx != ekfs[0]->ctx) { hv_set_error("%s: filter of another context", wf); return HV_ERR_INVALID; }
        if (e->N != ekfs[0]->N) { hv_set_error("%s: state dimension differs from filter 0", wf); return HV_ERR_INVALID; }
        for (int g = 0; g < f; g++) if (ekfs[g] == e) { hv_set_error("%s: filter appears twice", wf); return HV_ERR_INVALID; }
        if (ntracks[f] < 0 || (ntracks[f] > 0 && (!tracks[f] || !out[f]))) { hv_set_error("%s: negative track count, or NULL tracks or results", wf); return HV_ERR_INVALID; }
        if (!e->tm || !e->tm->camSet) { hv_set_error("%s: hv_ekf_set_camera_model has not been called", wf); return HV_ERR_STATE; }
        if (ntracks[f] == 0) continue;
        int rc = tm_validate(e, wf, tracks[f], ntracks[f]);
        if (rc != HV_OK) return rc;
        const int ncam = e->tm->cam.use_stereo ? 2 : 1;
        for (int k = 0; k < ntracks[f]; k++) {
            const hv_track_obs& o = tracks[f][k];
            const int n = 2 * o.npose * ncam, l = track_cols(o);
            EkfUpdateArgs a;
            rc = visual_args(e, wf, n, l, params[f].chi_outlier_r, params[f].track_rmse_threshold, EKF_MODE_CHECK, a);
            if (rc != HV_OK) return rc;
            if (!ekf_cluster2_fits(n, l, e->N, false)) {
                hv_set_error("%s, track %d (n=%d, l=%d): the measurement does not fit the cluster kernel whole at N = %d (the group has no row-chunked form)",
                             wf, k, n, l, e->N);
                return HV_ERR_UNSUPPORTED;
            }
        }
    }
    hv_ctx* c = ekfs[0]->ctx;
    HV_CUDA(cudaSetDevice(c->device));
    std::vector<VisualChain> ch(count);
    std::vector<int> next(count, 0), winEnd(count, 0);  // per chain: the next track to issue, the end of its current window
    for (int f = 0; f < count; f++) {
        if (ntracks[f] == 0) continue;
        int rc = flush_pending(ekfs[f]);                 // (EKF_ENTER: work queued by earlier calls goes first)
        if (rc == HV_OK) rc = join_side(ekfs[f]);
        if (rc == HV_OK) rc = chain_begin(ekfs[f], whoF[f].c_str(), tracks[f], ntracks[f], &params[f], ch[f]);
        if (rc != HV_OK) return rc;
        winEnd[f] = chain_window(ch[f]);
    }
    auto align16 = [](size_t v) { return (v + 15) & ~(size_t)15; };
    for (;;) {
        // steps up to the first window end that needs a decision; if none does, up to the end of the longest chain
        int D = 0x7fffffff, longest = 0;
        for (int f = 0; f < count; f++) {
            const int left = winEnd[f] - next[f];
            if (left <= 0) continue;
            longest = std::max(longest, left);
            if (winEnd[f] < ntracks[f]) D = std::min(D, left);
        }
        if (longest == 0) break;
        if (D == 0x7fffffff) D = longest;
        // the argument blocks of these D steps: per step the model blocks, the cluster blocks, the update blocks, in one staging block
        std::vector<std::vector<TmArgs>> M(D);
        std::vector<std::vector<EkfUpdateArgs>> C(D), U(D);
        for (int j = 0; j < D; j++)
            for (int f = 0; f < count; f++) {
                if (next[f] + j >= winEnd[f]) continue;
                TmArgs m; EkfUpdateArgs cu, u;
                const int rc = chain_track(ekfs[f], whoF[f].c_str(), ch[f], next[f] + j, j > 0 ? 1 : 0, m, cu, u);
                if (rc != HV_OK) return rc;
                M[j].push_back(m); C[j].push_back(cu);
                if (!ch[f].fused) U[j].push_back(u);
            }
        std::vector<size_t> offM(D), offC(D), offU(D);
        size_t bytes = 0;
        for (int j = 0; j < D; j++) {
            offM[j] = bytes; bytes = align16(bytes + M[j].size() * sizeof(TmArgs));
            offC[j] = bytes; bytes = align16(bytes + C[j].size() * sizeof(EkfUpdateArgs));
            offU[j] = bytes; bytes = align16(bytes + U[j].size() * sizeof(EkfUpdateArgs));
        }
        char *h = nullptr, *d = nullptr; cudaEvent_t ev = nullptr;
        int rc = group_stage(c, bytes, &h, &d, &ev);
        if (rc != HV_OK) return rc;
        for (int j = 0; j < D; j++) {
            memcpy(h + offM[j], M[j].data(), M[j].size() * sizeof(TmArgs));
            memcpy(h + offC[j], C[j].data(), C[j].size() * sizeof(EkfUpdateArgs));
            if (!U[j].empty()) memcpy(h + offU[j], U[j].data(), U[j].size() * sizeof(EkfUpdateArgs));
        }
        HV_CUDA(cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, c->stream));
        HV_CUDA(cudaEventRecord(ev, c->stream));
        for (int j = 0; j < D; j++) {
            HV_CUDA(tm_launch_group((const TmArgs*)(h + offM[j]), (const TmArgs*)(d + offM[j]), (int)M[j].size(), c->stream));
            HV_CUDA(ekf_launch_group_cluster2((const EkfUpdateArgs*)(h + offC[j]), (const EkfUpdateArgs*)(d + offC[j]), (int)C[j].size(), c->stream));
            c->launches += 2;
            if (U[j].empty()) continue;
            HV_CUDA(ekf_launch_group_cluster2((const EkfUpdateArgs*)(h + offU[j]), (const EkfUpdateArgs*)(d + offU[j]), (int)U[j].size(), c->stream));
            c->launches++;
        }
        // the chains that have reached the end of a window hand their results back: one synchronisation for all of them
        std::vector<int> ended;
        for (int f = 0; f < count; f++) {
            if (next[f] >= winEnd[f]) continue;
            next[f] = std::min(next[f] + D, winEnd[f]);
            if (next[f] < winEnd[f]) continue;
            ended.push_back(f);
            rc = chain_fetch(ekfs[f], ch[f], winEnd[f] - ch[f].issued);
            if (rc != HV_OK) return rc;
        }
        HV_CUDA(cudaStreamSynchronize(c->stream));
        for (int f : ended) {
            chain_synced(ekfs[f], ch[f], winEnd[f] - ch[f].issued);
            if (chain_open(ch[f])) winEnd[f] = ch[f].issued + chain_window(ch[f]);
        }
    }
    int rc = HV_OK;
    for (int f = count - 1; f >= 0; f--) {               // (in reverse: the error message names the first filter whose update failed)
        if (ntracks[f] == 0) { if (successfulUpdates) successfulUpdates[f] = 0; continue; }
        const int rcf = chain_results(ekfs[f], whoF[f].c_str(), ch[f], out[f], successfulUpdates ? successfulUpdates + f : nullptr);
        if (rcf != HV_OK) rc = rcf;
    }
    return rc;
}

// Outlier check / update on a measurement model that is already on the device (hv_ekf_track_models): same launch and result
// protocol as visual_host, without the staging copy.
int hv_ekf_visual_track(hv_ekf* e, const hv_track_model* t, double r, double rmseThr, int mode, int* vuStatus, double* chi2)
{
    EKF_ENTER(e, "hv_ekf_visual_track");
    const char* who = "hv_ekf_visual_track";
    if (!t || !t->d_H || !t->d_f || !t->d_y || mode < 0 || mode > 2) { hv_set_error("%s: invalid argument", who); return HV_ERR_INVALID; }
    if (t->triangulator_status != 0 || t->prepare_vu_status != 0) { hv_set_error("%s: the track has no valid measurement model", who); return HV_ERR_INVALID; }
    EkfUpdateArgs a;
    int rc = visual_args(e, who, t->rows, t->cols, r, rmseThr, mode, a);
    if (rc != HV_OK) return rc;
    a.H = t->d_H; a.f = t->d_f; a.y = t->d_y;
    if (mode != EKF_MODE_UPDATE) { a.sig = e->d_sig; a.sigSeq = (e->sigSeq += 1.0); }
    rc = launch_update(e, a);
    if (rc != HV_OK) return rc;
    if (mode == EKF_MODE_UPDATE) return HV_OK;                   // asynchronous
    rc = poll_results(e, 1, a.sigSeq, who);
    if (rc != HV_OK) return rc;
    if (vuStatus) *vuStatus = (int)e->h_sig[0];
    if (chi2) *chi2 = e->h_sig[1];
    if (e->h_sig[2] != 0.0) { hv_set_error("%s: innovation covariance not positive definite", who); return HV_ERR_STATE; }
    return HV_OK;
}

// Measurement aid: re-issues the kernel of the last hv_ekf_track_models call `reps` times between two CUDA events on the
// context's stream (same inputs, same outputs) and returns the average device time per launch.
int hv_ekf_track_models_time(hv_ekf* e, int reps, float* msPerLaunch)
{
    EKF_ENTER(e, "hv_ekf_track_models_time");
    TrackModels* t = e->tm;
    if (!t || t->last < 1 || reps < 1 || !msPerLaunch) { hv_set_error("hv_ekf_track_models_time: nothing to repeat"); return HV_ERR_INVALID; }
    cudaStream_t s = e->ctx->stream;
    cudaEvent_t a, b;
    HV_CUDA(cudaEventCreate(&a)); HV_CUDA(cudaEventCreate(&b));
    for (int i = 0; i < 3; i++) HV_CUDA(tm_launch(t->lastArgs, s));
    HV_CUDA(cudaEventRecord(a, s));
    for (int i = 0; i < reps; i++) HV_CUDA(tm_launch(t->lastArgs, s));
    HV_CUDA(cudaEventRecord(b, s));
    HV_CUDA(cudaEventSynchronize(b));
    float ms = 0;
    HV_CUDA(cudaEventElapsedTime(&ms, a, b));
    cudaEventDestroy(a); cudaEventDestroy(b);
    e->ctx->launches += reps + 3;
    *msPerLaunch = ms / reps;
    return HV_OK;
}

int hv_ekf_track_model_download(hv_ekf* e, int track, double* H, double* f, double* dpf)
{
    EKF_ENTER_LAZY(e, "hv_ekf_track_model_download");
    TrackModels* t = e->tm;
    if (!t || track < 0 || track >= t->last) { hv_set_error("hv_ekf_track_model_download: no such track"); return HV_ERR_INVALID; }
    cudaStream_t s = e->ctx->stream;
    const int* st = (const int*)t->h_out + 4 * track;
    const size_t rows = st[2], cols = st[3];
    if (H && rows * cols) HV_CUDA(cudaMemcpyAsync(H, t->d_H + (size_t)track * TrackModels::hStride(), sizeof(double) * rows * cols, cudaMemcpyDeviceToHost, s));
    if (f && rows) HV_CUDA(cudaMemcpyAsync(f, t->d_f + (size_t)track * 2 * TM_MAXOBS, sizeof(double) * rows, cudaMemcpyDeviceToHost, s));
    if (dpf) HV_CUDA(cudaMemcpyAsync(dpf, t->d_dpf + (size_t)track * 3 * (7 * TM_MAXPOSE + 1), sizeof(double) * 3 * (7 * t->lastNpose[track] + 1), cudaMemcpyDeviceToHost, s));
    HV_CUDA(cudaStreamSynchronize(s));
    return HV_OK;
}

int hv_ekf_lock_biases(hv_ekf* e) { EKF_ENTER(e, "hv_ekf_lock_biases"); return launch_ew(e, EKF_EW_LOCK_BIASES); }

} // extern "C"
