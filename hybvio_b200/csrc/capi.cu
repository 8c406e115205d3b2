// hybvio_b200/csrc/capi.cu -- C ABI (include/hybvio_b200.h): context, image pyramid, Lucas-Kanade.
// The EKF entry points live in ekf_capi.cu.
#include "capi_internal.h"
#include <climits>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>

static thread_local char g_err[512] = "";

void hv_set_error(const char* fmt, ...)
{
    va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof(g_err), fmt, ap); va_end(ap);
}

extern "C" {

const char* hv_version(void) { return "hybvio_b200 0.1 (sm_90a)"; }
const char* hv_last_error(void) { return g_err; }

int hv_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

static int ctx_create(int device, cudaStream_t stream, bool own, hv_ctx** out)
{
    if (!out) { hv_set_error("hv_ctx_create: out is NULL"); return HV_ERR_INVALID; }
    *out = nullptr;
    int n = hv_device_count();
    if (n <= 0 || device < 0 || device >= n) {
        hv_set_error("hv_ctx_create: no CUDA device %d (found %d). hybvio_b200 has no CPU fallback.", device, n);
        return HV_ERR_NO_DEVICE;
    }
    cudaDeviceProp prop;
    HV_CUDA(cudaGetDeviceProperties(&prop, device));
    // arch-specific sm_90a code loads on compute capability 9.0 only
    if (prop.major != 9 || prop.minor != 0) {
        hv_set_error("hv_ctx_create: device %d is sm_%d%d; this library is built for sm_90a (H100) only", device, prop.major, prop.minor);
        return HV_ERR_NO_DEVICE;
    }
    HV_CUDA(cudaSetDevice(device));
    hv_ctx* c = new hv_ctx;
    c->device = device;
    // every failure below releases what has been created so far (hv_ctx_destroy tolerates a partly initialised context)
    auto fail = [&](cudaError_t e, const char* what) {
        hv_set_error("hv_ctx_create: %s failed: %s", what, cudaGetErrorString(e));
        hv_ctx_destroy(c);
        return e == cudaErrorMemoryAllocation ? HV_ERR_OOM : HV_ERR_CUDA;
    };
    cudaError_t e = cudaSuccess;
    if (own) { e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking); if (e != cudaSuccess) { c->stream = nullptr; return fail(e, "cudaStreamCreate"); } c->ownStream = true; }
    else c->stream = stream;
    if ((e = cudaMalloc(&c->d_table, sizeof(HvPyrDesc) * HV_TABLE_CAPACITY)) != cudaSuccess) { c->d_table = nullptr; return fail(e, "cudaMalloc"); }
    if ((e = cudaMemsetAsync(c->d_table, 0, sizeof(HvPyrDesc) * HV_TABLE_CAPACITY, c->stream)) != cudaSuccess) return fail(e, "cudaMemsetAsync");
    if ((e = cudaStreamSynchronize(c->stream)) != cudaSuccess) return fail(e, "cudaStreamSynchronize");
    for (int i = HV_TABLE_CAPACITY - 1; i >= 0; --i) c->freeSlots.push_back(i);
    *out = c;
    return HV_OK;
}

int hv_ctx_create(int device, hv_ctx** out) { return ctx_create(device, nullptr, true, out); }
int hv_ctx_create_on_stream(int device, void* s, hv_ctx** out) { return ctx_create(device, (cudaStream_t)s, false, out); }

int hv_ctx_destroy(hv_ctx* c)
{
    if (!c) return HV_OK;
    cudaSetDevice(c->device);
    if (c->stream || !c->ownStream) cudaStreamSynchronize(c->stream);
    if (c->sideStream) { cudaStreamSynchronize(c->sideStream); cudaStreamDestroy(c->sideStream); }
    if (c->covStream) { cudaStreamSynchronize(c->covStream); cudaStreamDestroy(c->covStream); }
    if (c->d_table) cudaFree(c->d_table);
    if (c->d_stage) cudaFree(c->d_stage);
    if (c->h_stage) cudaFreeHost(c->h_stage);
    if (c->d_done) cudaFree(c->d_done);
    if (c->d_selectScratch) cudaFree(c->d_selectScratch);
    if (c->d_fastScratch) cudaFree(c->d_fastScratch);
    if (c->d_gfScratch) cudaFree(c->d_gfScratch);
    if (c->d_essScratch) cudaFree(c->d_essScratch);
    if (c->d_ekfStage) cudaFree(c->d_ekfStage);
    for (int i = 0; i < HV_EKF_STAGES; i++) {
        if (c->h_ekfStage[i]) cudaFreeHost(c->h_ekfStage[i]);
        if (c->evEkfStage[i]) cudaEventDestroy(c->evEkfStage[i]);
    }
    if (c->ownStream && c->stream) cudaStreamDestroy(c->stream);
    delete c;
    return HV_OK;
}

int hv_ctx_sync(hv_ctx* c)
{
    if (!c) { hv_set_error("hv_ctx_sync: NULL ctx"); return HV_ERR_INVALID; }
    HV_CUDA(cudaStreamSynchronize(c->stream));
    if (c->sideStream) HV_CUDA(cudaStreamSynchronize(c->sideStream));
    if (c->covStream) HV_CUDA(cudaStreamSynchronize(c->covStream));
    return HV_OK;
}
void* hv_ctx_stream(hv_ctx* c) { return c ? (void*)c->stream : nullptr; }
long long hv_ctx_launch_count(hv_ctx* c) { return c ? c->launches : 0; }

} // extern "C"

int hv_ctx_reserve_stage(hv_ctx* c, size_t bytes)
{
    if (bytes <= c->stageBytes) return HV_OK;
    HV_CUDA(cudaStreamSynchronize(c->stream));
    if (c->d_stage) cudaFree(c->d_stage);
    if (c->h_stage) cudaFreeHost(c->h_stage);
    c->d_stage = nullptr; c->h_stage = nullptr; c->stageBytes = 0;
    size_t cap = 4096; while (cap < bytes) cap *= 2;
    HV_CUDA(cudaMalloc(&c->d_stage, cap));
    HV_CUDA(cudaHostAlloc(&c->h_stage, cap + 64, cudaHostAllocMapped));          // + 64: the completion flag
    HV_CUDA(cudaHostGetDevicePointer(&c->hd_stage, c->h_stage, 0));
    memset(c->h_stage, 0, cap + 64);
    // (stream-ordered: the context's stream is non-blocking, a cudaMemset on the legacy stream could land after the first kernel's counts)
    if (!c->d_done) { HV_CUDA(cudaMalloc(&c->d_done, sizeof(unsigned))); HV_CUDA(cudaMemsetAsync(c->d_done, 0, sizeof(unsigned), c->stream)); c->doneCount = 0; }
    c->stageBytes = cap;
    return HV_OK;
}

// Arms the completion signal of a host-buffer launch of `units` CTAs on the context's stage; the flag sits right behind the stage.
static HvDoneSignal done_arm(hv_ctx* c, unsigned units)
{
    c->doneCount += units;
    return HvDoneSignal{c->d_done, c->doneCount, ++c->seq, (volatile unsigned*)((uint8_t*)c->hd_stage + c->stageBytes)};
}

// Waits for the flag of a signal from done_arm; on failure resynchronises the counter before anybody polls again.
static int done_wait(hv_ctx* c, const HvDoneSignal& d, const char* who)
{
    volatile unsigned* flag = (volatile unsigned*)((uint8_t*)c->h_stage + c->stageBytes);
    const int rc = hv_poll(c->stream, who, [&] { return *flag == d.seq; });
    if (rc != HV_OK) {
        cudaStreamSynchronize(c->stream); cudaMemsetAsync(c->d_done, 0, sizeof(unsigned), c->stream); cudaStreamSynchronize(c->stream); c->doneCount = 0;
    }
    return rc;
}

// ------------------------------------------------------------------------------------------------ pyramid
static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

extern "C" {

int hv_pyr_create(hv_ctx* c, int w, int h, int win, int maxLevel, hv_pyr** out)
{
    if (!c || !out || w <= 0 || h <= 0 || win <= 2 || maxLevel < 0) {
        hv_set_error("hv_pyr_create: invalid argument (w=%d h=%d win=%d maxLevel=%d)", w, h, win, maxLevel);
        return HV_ERR_INVALID;
    }
    if (maxLevel > HV_MAX_LEVELS - 1) {
        hv_set_error("hv_pyr_create: maxLevel %d > %d unsupported", maxLevel, HV_MAX_LEVELS - 1);
        return HV_ERR_UNSUPPORTED;
    }
    if (c->freeSlots.empty()) { hv_set_error("hv_pyr_create: more than %d live pyramids", HV_TABLE_CAPACITY); return HV_ERR_OOM; }
    HV_CUDA(cudaSetDevice(c->device));
    hv_pyr* p = new hv_pyr;
    p->ctx = c; p->w = w; p->h = h; p->win = win;
    // level geometry (OCV/video/src/lkpyramid.cpp:776-816)
    int lw = w, lh = h, nl = 0;
    size_t off = 0, goff[HV_MAX_LEVELS], doff[HV_MAX_LEVELS];
    memset(&p->desc, 0, sizeof(p->desc));
    for (int level = 0; level <= maxLevel; ++level) {
        HvLevel& L = p->desc.lv[level];
        L.w = lw; L.h = lh;
        // Level 0 IS the input image: with a dense pitch (w % 4 == 0 keeps the kernels' 32-bit loads aligned) a contiguous
        // host frame is ONE 1-D H2D copy; a padded pitch would make it a 2-D copy of h rows, measured at ~5x the time of
        // the 1-D copy of the same 361 KB. Coarser levels are only ever written by the kernel.
        L.gpitch = (level == 0 && lw % 4 == 0) ? lw : (int)align_up((size_t)lw, 128);
        L.dpitch = (int)align_up((size_t)lw, 32);
        goff[level] = off; off = align_up(off + (size_t)L.gpitch * lh, 256);
        doff[level] = off; off = align_up(off + (size_t)L.dpitch * lh * sizeof(short2), 256);
        nl = level + 1;
        lw = (lw + 1) / 2; lh = (lh + 1) / 2;
        if (lw <= win || lh <= win) break;
    }
    p->nlevels = nl; p->desc.nlevels = nl; p->desc.win = win;
    p->bytes = off;
    cudaError_t e = cudaMalloc(&p->d_mem, off);
    if (e != cudaSuccess) { delete p; hv_set_error("hv_pyr_create: cudaMalloc(%zu) failed: %s", off, cudaGetErrorString(e)); return HV_ERR_OOM; }
    HV_CUDA(cudaMemsetAsync(p->d_mem, 0, off, c->stream));
    for (int level = 0; level < nl; ++level) {
        p->desc.lv[level].gray = (uint8_t*)p->d_mem + goff[level];
        p->desc.lv[level].deriv = (short2*)((uint8_t*)p->d_mem + doff[level]);
    }
    p->slot = c->freeSlots.back(); c->freeSlots.pop_back();
    HV_CUDA(cudaMemcpyAsync(c->d_table + p->slot, &p->desc, sizeof(HvPyrDesc), cudaMemcpyHostToDevice, c->stream));
    HV_CUDA(cudaStreamSynchronize(c->stream));   // desc is on the stack-owned object; creation is rare
    *out = p;
    return HV_OK;
}

int hv_pyr_release(hv_pyr* p)
{
    if (!p) return HV_OK;
    hv_ctx* c = p->ctx;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    if (p->d_mem) cudaFree(p->d_mem);
    c->freeSlots.push_back(p->slot);
    delete p;
    return HV_OK;
}

int hv_pyr_levels(const hv_pyr* p) { return p ? p->nlevels : HV_ERR_INVALID; }

int hv_pyr_level_size(const hv_pyr* p, int level, int* w, int* h)
{
    if (!p || level < 0 || level >= p->nlevels) { hv_set_error("hv_pyr_level_size: bad level"); return HV_ERR_INVALID; }
    if (w) *w = p->desc.lv[level].w;
    if (h) *h = p->desc.lv[level].h;
    return HV_OK;
}

int hv_pyr_build_batch(hv_pyr* const* pyrs, const uint8_t* const* gray, const size_t* strides, int n, int srcIsDevice)
{
    if (!pyrs || !gray || !strides || n <= 0) { hv_set_error("hv_pyr_build_batch: invalid argument"); return HV_ERR_INVALID; }
    hv_ctx* c = pyrs[0] ? pyrs[0]->ctx : nullptr;
    if (!c) { hv_set_error("hv_pyr_build_batch: NULL pyramid"); return HV_ERR_INVALID; }
    HV_CUDA(cudaSetDevice(c->device));
    std::vector<unsigned short> idx(n);
    std::vector<const uint8_t*> src(n);
    std::vector<int> srcPitch(n), l0Pitch(n), nls(n);
    std::vector<const uint8_t*> l0(n);
    int maxNl = 0;
    for (int i = 0; i < n; i++) {
        hv_pyr* p = pyrs[i];
        if (!p || p->ctx != c || p->w != pyrs[0]->w || p->h != pyrs[0]->h || !gray[i] || strides[i] < (size_t)p->w) {
            hv_set_error("hv_pyr_build_batch: pyramid %d invalid / different context or size", i);
            return HV_ERR_INVALID;
        }
        const HvLevel& L0 = p->desc.lv[0];
        if (srcIsDevice) {      // frame already in HBM: the kernel reads it in place and fills level 0 itself
            src[i] = gray[i]; srcPitch[i] = (int)strides[i];
        } else {                // the frame lands directly in the level-0 buffer: level 0 of the pyramid IS the input image
            if (strides[i] == (size_t)L0.gpitch)     // one 1-D copy up to the last pixel (the caller's buffer may end there)
                HV_CUDA(cudaMemcpyAsync(L0.gray, gray[i], (size_t)L0.gpitch * (p->h - 1) + p->w, cudaMemcpyHostToDevice, c->stream));
            else
                HV_CUDA(cudaMemcpy2DAsync(L0.gray, L0.gpitch, gray[i], strides[i], (size_t)p->w, (size_t)p->h, cudaMemcpyHostToDevice, c->stream));
            src[i] = nullptr; srcPitch[i] = 0;
        }
        idx[i] = (unsigned short)p->slot;
        l0[i] = L0.gray; l0Pitch[i] = L0.gpitch; nls[i] = p->nlevels;
        if (p->nlevels > maxNl) maxNl = p->nlevels;
    }
    HV_CUDA(hv_launch_pyr_fused(c->d_table, idx.data(), src.data(), srcPitch.data(), l0.data(), l0Pitch.data(), nls.data(), n, pyrs[0]->w, pyrs[0]->h,
                                maxNl, c->stream));
    c->launches += (n + 31) / 32;
    return HV_OK;
}

int hv_pyr_build(hv_pyr* p, const uint8_t* gray, size_t stride)
{
    return hv_pyr_build_batch(&p, &gray, &stride, 1, 0);
}

int hv_pyr_download_level(hv_pyr* p, int level, uint8_t* gray, int16_t* deriv)
{
    if (!p || level < 0 || level >= p->nlevels) { hv_set_error("hv_pyr_download_level: bad level"); return HV_ERR_INVALID; }
    hv_ctx* c = p->ctx;
    HV_CUDA(cudaSetDevice(c->device));
    const HvLevel& L = p->desc.lv[level];
    if (gray) HV_CUDA(cudaMemcpy2DAsync(gray, L.w, L.gray, L.gpitch, L.w, L.h, cudaMemcpyDeviceToHost, c->stream));
    if (deriv) HV_CUDA(cudaMemcpy2DAsync(deriv, (size_t)L.w * 4, L.deriv, (size_t)L.dpitch * 4, (size_t)L.w * 4, L.h,
                                         cudaMemcpyDeviceToHost, c->stream));
    HV_CUDA(cudaStreamSynchronize(c->stream));
    return HV_OK;
}

int hv_pyr_download_level_padded(hv_pyr* p, int level, uint8_t* gray, int16_t* deriv)
{
    if (!p || level < 0 || level >= p->nlevels) { hv_set_error("hv_pyr_download_level_padded: bad level"); return HV_ERR_INVALID; }
    const HvLevel& L = p->desc.lv[level];
    const int win = p->win, W = L.w + 2 * win, H = L.h + 2 * win;
    std::vector<uint8_t> g((size_t)L.w * L.h);
    std::vector<int16_t> d((size_t)L.w * L.h * 2);
    int rc = hv_pyr_download_level(p, level, gray ? g.data() : nullptr, deriv ? d.data() : nullptr);
    if (rc != HV_OK) return rc;
    // border exactly as the reference materialises it: gray REFLECT_101, gradient CONSTANT 0 (lkpyramid.cpp:761-808)
    for (int y = 0; y < H; y++) {
        const int sy = hv_reflect101(y - win, L.h);
        const bool rowIn = (unsigned)(y - win) < (unsigned)L.h;
        for (int x = 0; x < W; x++) {
            const int sx = hv_reflect101(x - win, L.w);
            const bool in = rowIn && (unsigned)(x - win) < (unsigned)L.w;
            if (gray) gray[(size_t)y * W + x] = g[(size_t)sy * L.w + sx];
            if (deriv) {
                deriv[((size_t)y * W + x) * 2] = in ? d[((size_t)sy * L.w + sx) * 2] : 0;
                deriv[((size_t)y * W + x) * 2 + 1] = in ? d[((size_t)sy * L.w + sx) * 2 + 1] : 0;
            }
        }
    }
    return HV_OK;
}

// ------------------------------------------------------------------------------------------------ LK
static int lk_fill(LkLaunch& L, hv_ctx* c, int maxLevel, int maxIter, double eps, double minEig)
{
    // criteria clamp of SparsePyrLKOpticalFlowImpl::calc (lkpyramid.cpp:1361-1369)
    L.table = c->d_table;
    L.prefetch = 1;
    L.maxLevel = maxLevel;
    L.maxIter = maxIter < 0 ? 0 : (maxIter > 100 ? 100 : maxIter);
    double e = eps < 0. ? 0. : (eps > 10. ? 10. : eps);
    L.eps2 = e * e;
    L.minEig = (float)minEig;
    L.done = HvDoneSignal{};
    return HV_OK;
}

static int lk_check_pair(const char* who, hv_ctx* c, hv_pyr* a, hv_pyr* b)
{
    if (!a || !b || a->ctx != c || b->ctx != c) { hv_set_error("%s: pyramid NULL or from another context", who); return HV_ERR_INVALID; }
    if (a->w != b->w || a->h != b->h || a->win != b->win) { hv_set_error("%s: pyramids differ in size/window", who); return HV_ERR_INVALID; }
    return HV_OK;
}

static int lk_track_batch_device_on(hv_ctx* c, cudaStream_t stream, const hv_lk_job* jobs, int njobs, int maxIter, double eps, double minEig, const float* initXY = nullptr)
{
    if (!c || !jobs || njobs < 0) { hv_set_error("hv_lk_track_batch_device: invalid argument"); return HV_ERR_INVALID; }
    HV_CUDA(cudaSetDevice(c->device));
    for (int base = 0; base < njobs; base += LK_MAX_JOBS) {
        LkLaunch L;
        int cnt = njobs - base < LK_MAX_JOBS ? njobs - base : LK_MAX_JOBS;
        int win = 0, maxLevel = HV_MAX_LEVELS;
        for (int i = 0; i < cnt; i++) {
            const hv_lk_job& j = jobs[base + i];
            int rc = lk_check_pair("hv_lk_track_batch_device", c, j.prev, j.next);
            if (rc != HV_OK) return rc;
            if (j.n < 0 || (j.n > 0 && (!j.d_prev_xy || !j.d_next_xy || !j.d_status))) {
                hv_set_error("hv_lk_track_batch_device: job %d has NULL buffers", base + i); return HV_ERR_INVALID;
            }
            if (win && win != j.prev->win) { hv_set_error("hv_lk_track_batch_device: mixed window sizes"); return HV_ERR_INVALID; }
            win = j.prev->win;
            LkJob& d = L.jobs[i];
            d.prevIdx = j.prev->slot; d.nextIdx = j.next->slot; d.n = j.n; d.useInitial = j.use_initial;
            d.prevPts = (const float2*)j.d_prev_xy; d.nextPts = (float2*)j.d_next_xy;
            d.status = j.d_status; d.trackStatus = j.d_track_status; d.initPts = initXY && cnt == 1 ? (const float2*)initXY : nullptr;
        }
        L.njobs = cnt;
        lk_fill(L, c, maxLevel, maxIter, eps, minEig);
        cudaError_t e = hv_launch_lk(L, win, stream);
        if (e == cudaErrorInvalidValue) { hv_set_error("hv_lk_track: window size %d unsupported (supported: 11, 15, 21, 31)", win); return HV_ERR_UNSUPPORTED; }
        HV_CUDA(e);
        c->launches += 1;
    }
    return HV_OK;
}
int hv_lk_track_batch_device(hv_ctx* c, const hv_lk_job* jobs, int njobs, int maxIter, double eps, double minEig)
{
    return lk_track_batch_device_on(c, c ? c->stream : nullptr, jobs, njobs, maxIter, eps, minEig);
}

static int lk_track_device_on(hv_ctx* c, cudaStream_t stream, hv_pyr* prev, hv_pyr* next, const float* dPrev, float* dNext, uint8_t* dStatus,
                              int32_t* dTs, int n, int useInitial, int maxIter, double eps, double minEig, const float* dInit = nullptr)
{
    if (!c || n < 0) { hv_set_error("hv_lk_track_device: invalid argument"); return HV_ERR_INVALID; }
    if (n == 0) {                 // optical_flow.cpp:41-44: empty input, empty output (the pyramids are still validated)
        int rc = lk_check_pair("hv_lk_track_device", c, prev, next);
        return rc;
    }
    hv_lk_job j; j.prev = prev; j.next = next; j.d_prev_xy = dPrev; j.d_next_xy = dNext; j.d_status = dStatus;
    j.d_track_status = dTs; j.n = n; j.use_initial = useInitial;
    return lk_track_batch_device_on(c, stream, &j, 1, maxIter, eps, minEig, dInit);
}
int hv_lk_track_device(hv_ctx* c, hv_pyr* prev, hv_pyr* next, const float* dPrev, float* dNext, uint8_t* dStatus,
                       int32_t* dTs, int n, int useInitial, int maxIter, double eps, double minEig)
{
    return lk_track_device_on(c, c ? c->stream : nullptr, prev, next, dPrev, dNext, dStatus, dTs, n, useInitial, maxIter, eps, minEig);
}
int hv_lk_track_device_on_stream(hv_ctx* c, void* cudaStream, hv_pyr* prev, hv_pyr* next, const float* dPrev, const float* dInit, float* dNext,
                                 uint8_t* dStatus, int32_t* dTs, int n, int maxIter, double eps, double minEig)
{
    return lk_track_device_on(c, (cudaStream_t)cudaStream, prev, next, dPrev, dNext, dStatus, dTs, n, dInit ? 1 : 0, maxIter, eps, minEig, dInit);
}

int hv_lk_track(hv_ctx* c, hv_pyr* prev, hv_pyr* next, const float* prevXY, float* nextXY, uint8_t* status,
                int32_t* trackStatus, int n, int useInitial, int maxIter, double eps, double minEig)
{
    if (!c || n < 0 || (n > 0 && (!prevXY || !nextXY))) { hv_set_error("hv_lk_track: invalid argument"); return HV_ERR_INVALID; }
    int rc = lk_check_pair("hv_lk_track", c, prev, next);
    if (rc != HV_OK) return rc;
    if (n == 0) return HV_OK;   // optical_flow.cpp:41-44: empty input, empty output
    HV_CUDA(cudaSetDevice(c->device));
    // staging block: [prev 8n | next 8n | trackStatus 4n | status n]
    const size_t oPrev = 0, oNext = 8 * (size_t)n, oTs = 16 * (size_t)n, oSt = 20 * (size_t)n, total = 21 * (size_t)n;
    rc = hv_ctx_reserve_stage(c, total);
    if (rc != HV_OK) return rc;
    uint8_t* hs = (uint8_t*)c->h_stage; uint8_t* ds = (uint8_t*)c->d_stage;
    memcpy(hs + oPrev, prevXY, 8 * (size_t)n);
    if (useInitial) memcpy(hs + oNext, nextXY, 8 * (size_t)n);
    if (hv_lk_uses_cta_kernel(n)) {     // only the CTA-per-feature kernel raises the host flag
        // The kernel reads the points from and writes the results to the mapped pinned block itself (a few KB over PCIe) and
        // raises a flag there when the last feature is done: no H2D / D2H copy calls, no stream synchronisation.
        uint8_t* hd = (uint8_t*)c->hd_stage;
        LkLaunch L;
        LkJob& d = L.jobs[0];
        d.prevIdx = prev->slot; d.nextIdx = next->slot; d.n = n; d.useInitial = useInitial;
        d.prevPts = (const float2*)(hd + oPrev); d.nextPts = (float2*)(hd + oNext);
        d.status = hd + oSt; d.trackStatus = (int32_t*)(hd + oTs); d.initPts = nullptr;
        L.njobs = 1;
        lk_fill(L, c, HV_MAX_LEVELS, maxIter, eps, minEig);
        L.done = done_arm(c, (unsigned)n);
        cudaError_t e = hv_launch_lk(L, prev->win, c->stream);
        if (e == cudaErrorInvalidValue) { hv_set_error("hv_lk_track: window size %d unsupported (supported: 11, 15, 21, 31)", prev->win); return HV_ERR_UNSUPPORTED; }
        HV_CUDA(e);
        c->launches += 1;
        rc = done_wait(c, L.done, "hv_lk_track");
        if (rc != HV_OK) return rc;
    } else {
        HV_CUDA(cudaMemcpyAsync(ds, hs, useInitial ? 16 * (size_t)n : 8 * (size_t)n, cudaMemcpyHostToDevice, c->stream));
        rc = hv_lk_track_device(c, prev, next, (const float*)(ds + oPrev), (float*)(ds + oNext), ds + oSt, (int32_t*)(ds + oTs),
                                n, useInitial, maxIter, eps, minEig);
        if (rc != HV_OK) return rc;
        HV_CUDA(cudaMemcpyAsync(hs + oNext, ds + oNext, total - oNext, cudaMemcpyDeviceToHost, c->stream));
        HV_CUDA(cudaStreamSynchronize(c->stream));
    }
    memcpy(nextXY, hs + oNext, 8 * (size_t)n);
    if (trackStatus) memcpy(trackStatus, hs + oTs, 4 * (size_t)n);
    if (status) memcpy(status, hs + oSt, (size_t)n);
    return HV_OK;
}

// ------------------------------------------------------------------------------------------------ corner detection (N2)
static int gftt_args(const char* who, hv_ctx* c, hv_pyr* pyr, int blockSize, int cell, float minResponse, GfttArgs& a)
{
    if (!c || !pyr || pyr->ctx != c) { hv_set_error("%s: invalid context / pyramid", who); return HV_ERR_INVALID; }
    if (blockSize != 3) { hv_set_error("%s: gfttBlockSize %d unsupported (3 only)", who, blockSize); return HV_ERR_UNSUPPORTED; }
    if (cell < 2 || cell > 32) { hv_set_error("%s: cell size %d unsupported (2..32)", who, cell); return HV_ERR_UNSUPPORTED; }
    const HvLevel& L = pyr->desc.lv[0];
    memset(&a, 0, sizeof(a));
    a.gray = L.gray; a.pitch = L.gpitch; a.w = L.w; a.h = L.h; a.cell = cell; a.minResponse = minResponse;
    const double scale = 1.0 / ((double)(1 << 2) * blockSize * 255.0);          // OCV/imgproc/src/corner.cpp:246-251
    a.k1 = (float)(1.0 * scale); a.k0 = (float)(2.0 * scale);
    return HV_OK;
}

int hv_gftt_cells(const hv_pyr* pyr, int cell, int* cellsX, int* cellsY)
{
    if (!pyr || cell <= 0) { hv_set_error("hv_gftt_cells: invalid argument"); return HV_ERR_INVALID; }
    if (cellsX) *cellsX = pyr->w / cell;
    if (cellsY) *cellsY = pyr->h / cell;
    return HV_OK;
}

int hv_gftt_detect_device(hv_ctx* c, hv_pyr* pyr, int blockSize, int cell, float minResponse, float* dKp)
{
    GfttArgs a;
    int rc = gftt_args("hv_gftt_detect_device", c, pyr, blockSize, cell, minResponse, a);
    if (rc != HV_OK) return rc;
    if (!dKp) { hv_set_error("hv_gftt_detect_device: NULL output"); return HV_ERR_INVALID; }
    HV_CUDA(cudaSetDevice(c->device));
    a.kp = dKp;
    HV_CUDA(hv_launch_gftt(a, c->stream));
    c->launches += 1;
    return HV_OK;
}

int hv_gftt_detect(hv_ctx* c, hv_pyr* pyr, int blockSize, int cell, float minResponse, float* kp)
{
    GfttArgs a;
    int rc = gftt_args("hv_gftt_detect", c, pyr, blockSize, cell, minResponse, a);
    if (rc != HV_OK) return rc;
    if (!kp) { hv_set_error("hv_gftt_detect: NULL output"); return HV_ERR_INVALID; }
    const int cells = (a.w / cell) * (a.h / cell);
    if (cells == 0) return HV_OK;
    HV_CUDA(cudaSetDevice(c->device));
    const size_t bytes = (size_t)cells * 3 * sizeof(float);
    rc = hv_ctx_reserve_stage(c, bytes);
    if (rc != HV_OK) return rc;
    // the kernel writes the key points straight into the mapped pinned block and the last cell raises the flag (as the LK kernel does)
    a.kp = (float*)c->hd_stage;
    a.done = done_arm(c, (unsigned)cells);
    HV_CUDA(hv_launch_gftt(a, c->stream));
    c->launches += 1;
    rc = done_wait(c, a.done, "hv_gftt_detect");
    if (rc != HV_OK) return rc;
    memcpy(kp, c->h_stage, bytes);
    return HV_OK;
}

// ------------------------------------------------------------------------------------------------ corner selection (N2)
static_assert(HV_CORNER_NONE == HV_CORNER_NONE_F, "padding value of the header and of the kernel");

// Checks the counts shared by both entry points (their pointers are checked by the callers first) and fills everything but the buffers;
// *need = the slots the call can fill.
static int select_args(const char* who, int nkp, int nprev, int maskRadius, int maxTracks, int capacity, GfttSelectArgs& a, int* need)
{
    if (nkp < 0 || nprev < 0 || maxTracks < 1) {
        hv_set_error("%s: invalid count (nkp %d, nprev %d, max_tracks %d)", who, nkp, nprev, maxTracks);
        return HV_ERR_INVALID;
    }
    if (nkp > HV_GFTT_SELECT_MAX_KP) { hv_set_error("%s: %d key points unsupported (at most %d)", who, nkp, HV_GFTT_SELECT_MAX_KP); return HV_ERR_UNSUPPORTED; }
    if (maskRadius > HV_GFTT_SELECT_MAX_RADIUS) {
        hv_set_error("%s: mask_radius %d unsupported (at most %d)", who, maskRadius, HV_GFTT_SELECT_MAX_RADIUS);
        return HV_ERR_UNSUPPORTED;
    }
    const int all = 2 * nkp;
    *need = maskRadius > 0 ? (maxTracks < all ? maxTracks : all) : all;
    if (capacity < *need) { hv_set_error("%s: capacity %d below the %d corners the call can return", who, capacity, *need); return HV_ERR_INVALID; }
    memset(&a, 0, sizeof(a));
    a.nkp = nkp; a.nprev = nprev; a.maskRadius = maskRadius; a.maxTracks = maxTracks; a.capacity = capacity;
    a.r2 = maskRadius > 0 ? (float)(maskRadius * maskRadius) : 0.f;             // applyMinDistance: float(maskRadius * maskRadius)
    a.pow2 = 2;
    while (a.pow2 < nkp) a.pow2 *= 2;
    return HV_OK;
}

int hv_gftt_select_device(hv_ctx* c, const float* dKp, int nkp, const float* dPrev, int nprev, int maskRadius, int maxTracks, float* dCorners,
                          int capacity, int* dCount)
{
    if (!c || !dCorners || !dCount || (nkp > 0 && !dKp) || (nprev > 0 && !dPrev)) {
        hv_set_error("hv_gftt_select_device: NULL context or buffer");
        return HV_ERR_INVALID;
    }
    GfttSelectArgs a;
    int need = 0;
    int rc = select_args("hv_gftt_select_device", nkp, nprev, maskRadius, maxTracks, capacity, a, &need);
    if (rc != HV_OK) return rc;
    HV_CUDA(cudaSetDevice(c->device));
    a.kp = dKp; a.prev = dPrev; a.out = dCorners; a.count = dCount;
    HV_CUDA(hv_launch_gftt_select(a, c->stream));      // nkp = 0: writes the count and the padding only
    c->launches += 1;
    return HV_OK;
}

int hv_gftt_corners(hv_ctx* c, hv_pyr* pyr, int blockSize, int cell, float minResponse, const float* prevXY, int nprev, int maskRadius,
                    int maxTracks, float* corners, int capacity, int* count)
{
    GfttArgs g;
    int rc = gftt_args("hv_gftt_corners", c, pyr, blockSize, cell, minResponse, g);
    if (rc != HV_OK) return rc;
    if (!corners || !count || (nprev > 0 && !prevXY)) { hv_set_error("hv_gftt_corners: NULL buffer"); return HV_ERR_INVALID; }
    const int nkp = (g.w / cell) * (g.h / cell);
    GfttSelectArgs a;
    int need = 0;
    rc = select_args("hv_gftt_corners", nkp, nprev, maskRadius, maxTracks, capacity, a, &need);
    if (rc != HV_OK) return rc;
    int got = 0;
    if (nkp > 0) {
        HV_CUDA(cudaSetDevice(c->device));
        // device scratch: [key points 3 nkp | previous corners 2 nprev] floats; the key points never leave the device
        const size_t scratch = sizeof(float) * (3 * (size_t)nkp + 2 * (size_t)nprev);
        if (scratch > c->selectScratchBytes) {
            if (c->d_selectScratch) { HV_CUDA(cudaStreamSynchronize(c->stream)); cudaFree(c->d_selectScratch); }
            c->d_selectScratch = nullptr; c->selectScratchBytes = 0;
            size_t cap = 4096; while (cap < scratch) cap *= 2;
            HV_CUDA(cudaMalloc(&c->d_selectScratch, cap));
            c->selectScratchBytes = cap;
        }
        // staging block: [previous corners 8 nprev | count (16 bytes) | corners 8 need]
        const size_t oCount = (8 * (size_t)nprev + 15) / 16 * 16, oCorners = oCount + 16, total = oCorners + 8 * (size_t)need;
        rc = hv_ctx_reserve_stage(c, total);
        if (rc != HV_OK) return rc;
        uint8_t* hs = (uint8_t*)c->h_stage; uint8_t* hd = (uint8_t*)c->hd_stage;
        float* dKp = c->d_selectScratch;
        if (nprev > 0) {
            memcpy(hs, prevXY, 8 * (size_t)nprev);
            HV_CUDA(cudaMemcpyAsync(dKp + 3 * (size_t)nkp, hs, 8 * (size_t)nprev, cudaMemcpyHostToDevice, c->stream));
        }
        g.kp = dKp;
        HV_CUDA(hv_launch_gftt(g, c->stream));
        c->launches += 1;
        a.kp = dKp; a.prev = dKp + 3 * (size_t)nkp; a.capacity = need;
        // the select kernel writes the corners and the count straight into the mapped pinned block and raises the flag
        a.out = (float*)(hd + oCorners); a.count = (int*)(hd + oCount);
        a.done = done_arm(c, 1u);
        HV_CUDA(hv_launch_gftt_select(a, c->stream));
        c->launches += 1;
        rc = done_wait(c, a.done, "hv_gftt_corners");
        if (rc != HV_OK) return rc;
        memcpy(&got, hs + oCount, sizeof(int));
        memcpy(corners, hs + oCorners, 8 * (size_t)got);
    }
    for (size_t i = 2 * (size_t)got; i < 2 * (size_t)capacity; i++) corners[i] = HV_CORNER_NONE;
    *count = got;
    return HV_OK;
}

// ------------------------------------------------------------------------------------------------ sub-pixel refinement (cornerSubPix)
// the checks of one point list on pyr's level 0
static int subpix_check(const char* who, hv_ctx* c, hv_pyr* pyr, int n, int hw, int hh)
{
    if (!c || !pyr || pyr->ctx != c || n < 0) { hv_set_error("%s: invalid context / pyramid / count", who); return HV_ERR_INVALID; }
    if (hw < 1 || hh < 1 || hw > HV_SUBPIX_MAX_HALF || hh > HV_SUBPIX_MAX_HALF) {
        hv_set_error("%s: half-window %d x %d unsupported (1..%d per axis)", who, hw, hh, HV_SUBPIX_MAX_HALF);
        return HV_ERR_UNSUPPORTED;
    }
    const HvLevel& L = pyr->desc.lv[0];
    if (L.w < 2 * hw + 5 || L.h < 2 * hh + 5) {          // cv::cornerSubPix asserts it
        hv_set_error("%s: image %d x %d smaller than the window needs (%d x %d)", who, L.w, L.h, 2 * hw + 5, 2 * hh + 5);
        return HV_ERR_INVALID;
    }
    return HV_OK;
}

static int subpix_args(const char* who, hv_ctx* c, hv_pyr* pyr, int n, int hw, int hh, int zw, int zh, int criteriaType, int maxCount,
                       double epsilon, SubpixArgs& a)
{
    int rc = subpix_check(who, c, pyr, n, hw, hh);
    if (rc != HV_OK) return rc;
    const HvLevel& L = pyr->desc.lv[0];
    memset(&a, 0, sizeof(a));
    a.gray = L.gray; a.pitch = L.gpitch; a.w = L.w; a.h = L.h; a.n = n; a.hw = hw; a.hh = hh;
    // criteria and mask exactly as cv::cornerSubPix forms them (OpenCV's MIN / MAX macros; std::exp(float))
    a.maxIters = 100;
    if (criteriaType & 1) { a.maxIters = maxCount < 1 ? 1 : maxCount; a.maxIters = a.maxIters > 100 ? 100 : a.maxIters; }
    double eps = (criteriaType & 2) ? (epsilon < 0. ? 0. : epsilon) : 0.;
    a.eps2 = eps * eps;
    const int ww = 2 * hw + 1, wh = 2 * hh + 1;
    for (int i = 0; i < wh; i++) {
        const float y = (float)(i - hh) / hh, vy = std::exp(-y * y);
        for (int j = 0; j < ww; j++) {
            const float x = (float)(j - hw) / hw;
            a.mask[i * ww + j] = (float)(vy * std::exp(-x * x));
        }
    }
    if (zw >= 0 && zh >= 0 && zw * 2 + 1 < ww && zh * 2 + 1 < wh)
        for (int i = hh - zh; i <= hh + zh; i++)
            for (int j = hw - zw; j <= hw + zw; j++) a.mask[i * ww + j] = 0.f;
    return HV_OK;
}

int hv_subpix_refine_device(hv_ctx* c, hv_pyr* pyr, float* dXY, int n, int hw, int hh, int zw, int zh, int criteriaType, int maxCount,
                            double epsilon)
{
    SubpixArgs a;
    int rc = subpix_args("hv_subpix_refine_device", c, pyr, n, hw, hh, zw, zh, criteriaType, maxCount, epsilon, a);
    if (rc != HV_OK) return rc;
    if (n == 0) return HV_OK;
    if (!dXY) { hv_set_error("hv_subpix_refine_device: NULL points"); return HV_ERR_INVALID; }
    HV_CUDA(cudaSetDevice(c->device));
    a.xy = (float2*)dXY;
    HV_CUDA(hv_launch_subpix(a, c->stream));
    c->launches += 1;
    return HV_OK;
}

int hv_subpix_refine(hv_ctx* c, hv_pyr* pyr, float* xy, int n, int hw, int hh, int zw, int zh, int criteriaType, int maxCount, double epsilon)
{
    SubpixArgs a;
    int rc = subpix_args("hv_subpix_refine", c, pyr, n, hw, hh, zw, zh, criteriaType, maxCount, epsilon, a);
    if (rc != HV_OK) return rc;
    if (n == 0) return HV_OK;
    if (!xy) { hv_set_error("hv_subpix_refine: NULL points"); return HV_ERR_INVALID; }
    for (int i = 0; i < n; i++) {
        const float x = xy[2 * i], y = xy[2 * i + 1];
        if (!(x >= 0.f && x < (float)a.w && y >= 0.f && y < (float)a.h)) {      // cv::cornerSubPix asserts it
            hv_set_error("hv_subpix_refine: corner %d (%g, %g) outside the %d x %d image", i, x, y, a.w, a.h);
            return HV_ERR_INVALID;
        }
    }
    HV_CUDA(cudaSetDevice(c->device));
    const size_t bytes = (size_t)n * 2 * sizeof(float);
    rc = hv_ctx_reserve_stage(c, bytes);
    if (rc != HV_OK) return rc;
    memcpy(c->h_stage, xy, bytes);
    // the kernel refines the points in the mapped pinned block itself and the last corner raises the flag (as the LK kernel does)
    a.xy = (float2*)c->hd_stage;
    a.done = done_arm(c, (unsigned)n);
    HV_CUDA(hv_launch_subpix(a, c->stream));
    c->launches += 1;
    rc = done_wait(c, a.done, "hv_subpix_refine");
    if (rc != HV_OK) return rc;
    memcpy(xy, c->h_stage, bytes);
    return HV_OK;
}

// ------------------------------------------------------------------------------------------------ the corner step of many sessions (N2)
// Each call checks every job with the checks of the per-session call and refuses before anything is launched; then one launch on the
// context's stream does what the per-session calls would do for every job, bit for bit. The argument blocks travel as kernel parameters.
static_assert(HV_CORNER_BATCH_MAX == 64, "batch size of the header and of the kernels");

static int corner_batch_check(const char* who, hv_ctx* c, const void* jobs, int njobs)
{
    if (!c || !jobs) { hv_set_error("%s: NULL context or jobs", who); return HV_ERR_INVALID; }
    if (njobs < 1 || njobs > HV_CORNER_BATCH_MAX) { hv_set_error("%s: %d jobs (1..%d per call)", who, njobs, HV_CORNER_BATCH_MAX); return HV_ERR_INVALID; }
    return HV_OK;
}

int hv_gftt_detect_batch_device(hv_ctx* c, const hv_corner_job* jobs, int njobs, int blockSize, int cell, float minResponse)
{
    int rc = corner_batch_check("hv_gftt_detect_batch_device", c, jobs, njobs);
    if (rc != HV_OK) return rc;
    GfttBatchArgs b;
    memset(&b, 0, sizeof(b));
    int ctas = 0;
    for (int j = 0; j < njobs; j++) {
        char who[64];
        snprintf(who, sizeof(who), "hv_gftt_detect_batch_device job %d", j);
        rc = gftt_args(who, c, jobs[j].pyr, blockSize, cell, minResponse, b.job[j]);
        if (rc != HV_OK) return rc;
        if (!jobs[j].d_kp) { hv_set_error("%s: NULL key points", who); return HV_ERR_INVALID; }
        b.job[j].kp = jobs[j].d_kp;
        const int cx = b.job[j].w / cell, cy = b.job[j].h / cell;       // as hv_launch_gftt: an image smaller than a cell adds no CTA
        b.first[j] = ctas;
        b.cellsX[j] = cx;
        if (cx > 0 && cy > 0) ctas += cx * cy;                          // at most 64 x (32767 / 2)^2: no overflow
    }
    for (int j = njobs; j <= HV_CORNER_BATCH_MAX; j++) b.first[j] = ctas;
    if (ctas == 0) return HV_OK;
    HV_CUDA(cudaSetDevice(c->device));
    HV_CUDA(hv_launch_gftt_batch(b, njobs, c->stream));
    c->launches += 1;
    return HV_OK;
}

int hv_gftt_select_batch_device(hv_ctx* c, const hv_corner_job* jobs, int njobs)
{
    int rc = corner_batch_check("hv_gftt_select_batch_device", c, jobs, njobs);
    if (rc != HV_OK) return rc;
    GfttSelectBatchArgs b;
    memset(&b, 0, sizeof(b));
    int maxPow2 = 2;
    for (int j = 0; j < njobs; j++) {
        const hv_corner_job& J = jobs[j];
        char who[64];
        snprintf(who, sizeof(who), "hv_gftt_select_batch_device job %d", j);
        if (!J.d_corners || !J.d_count || (J.nkp > 0 && !J.d_kp) || (J.nprev > 0 && !J.d_prev_xy)) {
            hv_set_error("%s: NULL buffer", who);
            return HV_ERR_INVALID;
        }
        GfttSelectArgs& a = b.job[j];
        int need = 0;
        rc = select_args(who, J.nkp, J.nprev, J.mask_radius, J.max_tracks, J.capacity, a, &need);
        if (rc != HV_OK) return rc;
        a.kp = J.d_kp; a.prev = J.d_prev_xy; a.out = J.d_corners; a.count = J.d_count;
        if (a.pow2 > maxPow2) maxPow2 = a.pow2;
    }
    HV_CUDA(cudaSetDevice(c->device));
    HV_CUDA(hv_launch_gftt_select_batch(b, njobs, maxPow2, c->stream));   // a job with nkp = 0 writes count 0 and its padding only
    c->launches += 1;
    return HV_OK;
}

int hv_subpix_refine_batch_device(hv_ctx* c, const hv_subpix_job* jobs, int njobs, int hw, int hh, int zw, int zh, int criteriaType,
                                  int maxCount, double epsilon)
{
    int rc = corner_batch_check("hv_subpix_refine_batch_device", c, jobs, njobs);
    if (rc != HV_OK) return rc;
    SubpixBatchArgs b;
    memset(&b, 0, sizeof(b));
    long long points = 0;
    for (int j = 0; j < njobs; j++) {
        const hv_subpix_job& J = jobs[j];
        char who[64];
        snprintf(who, sizeof(who), "hv_subpix_refine_batch_device job %d", j);
        // the window, criteria and mask are the batch's: formed once, with the checks of job 0
        rc = j == 0 ? subpix_args(who, c, J.pyr, J.n, hw, hh, zw, zh, criteriaType, maxCount, epsilon, b.s) : subpix_check(who, c, J.pyr, J.n, hw, hh);
        if (rc != HV_OK) return rc;
        if (J.n > 0 && !J.d_xy) { hv_set_error("%s: NULL points", who); return HV_ERR_INVALID; }
        const HvLevel& L = J.pyr->desc.lv[0];
        b.job[j] = SubpixJob{L.gray, L.gpitch, L.w, L.h, (float2*)J.d_xy, J.n};
        b.first[j] = (int)points;
        points += J.n;
        if (points > INT_MAX) { hv_set_error("%s: more than %d points in one batch", who, INT_MAX); return HV_ERR_INVALID; }
    }
    for (int j = njobs; j <= HV_CORNER_BATCH_MAX; j++) b.first[j] = (int)points;
    if (points == 0) return HV_OK;
    HV_CUDA(cudaSetDevice(c->device));
    HV_CUDA(hv_launch_subpix_batch(b, njobs, c->stream));
    c->launches += 1;
    return HV_OK;
}

// ------------------------------------------------------------------------------------------------ FAST corner detection (N2)
// Checks one job (its pointers and counts) and fills everything but the scratch; *scratch = the bytes of masks and tile counts it needs.
static int fast_args(const char* who, hv_ctx* c, hv_pyr* pyr, int threshold, int nonmax, float* xy, float* response, int capacity, int* count,
                     FastArgs& a, size_t* scratch)
{
    if (!c || !pyr || pyr->ctx != c) { hv_set_error("%s: invalid context / pyramid", who); return HV_ERR_INVALID; }
    if (capacity < 0 || !count || (capacity > 0 && !xy)) { hv_set_error("%s: NULL buffer or negative capacity (%d)", who, capacity); return HV_ERR_INVALID; }
    const HvLevel& L = pyr->desc.lv[0];
    memset(&a, 0, sizeof(a));
    a.gray = L.gray; a.pitch = L.gpitch; a.w = L.w; a.h = L.h;
    a.threshold = threshold < 0 ? 0 : (threshold > 255 ? 255 : threshold);       // FAST_t: std::min(std::max(threshold, 0), 255)
    a.nonmax = nonmax ? 1 : 0;
    a.tilesX = (L.w + 31) / 32; a.tilesY = (L.h + 7) / 8;
    a.xy = (float2*)xy; a.response = response; a.capacity = capacity; a.count = count;
    *scratch = align_up(sizeof(unsigned) * 8 * (size_t)a.tilesX * a.tilesY + sizeof(int) * (size_t)a.tilesX * a.tilesY, 256);
    return HV_OK;
}

// points the jobs' masks and tile counts into the context's FAST scratch, grown (after the work that may still read it) as needed
static int fast_scratch(hv_ctx* c, FastArgs* jobs, const size_t* bytes, int njobs)
{
    size_t total = 0;
    for (int j = 0; j < njobs; j++) total += bytes[j];
    if (total > c->fastScratchBytes) {
        if (c->d_fastScratch) { HV_CUDA(cudaStreamSynchronize(c->stream)); cudaFree(c->d_fastScratch); }
        c->d_fastScratch = nullptr; c->fastScratchBytes = 0;
        size_t cap = 65536; while (cap < total) cap *= 2;
        HV_CUDA(cudaMalloc(&c->d_fastScratch, cap));
        c->fastScratchBytes = cap;
    }
    uint8_t* p = (uint8_t*)c->d_fastScratch;
    for (int j = 0; j < njobs; j++) {
        FastArgs& a = jobs[j];
        a.mask = (unsigned*)p;
        a.tileCount = (int*)(p + sizeof(unsigned) * 8 * (size_t)a.tilesX * a.tilesY);
        p += bytes[j];
    }
    return HV_OK;
}

int hv_fast_detect_device(hv_ctx* c, hv_pyr* pyr, int threshold, int nonmax, float* dXY, float* dResponse, int capacity, int* dCount)
{
    FastArgs a;
    size_t bytes = 0;
    int rc = fast_args("hv_fast_detect_device", c, pyr, threshold, nonmax, dXY, dResponse, capacity, dCount, a, &bytes);
    if (rc != HV_OK) return rc;
    HV_CUDA(cudaSetDevice(c->device));
    rc = fast_scratch(c, &a, &bytes, 1);
    if (rc != HV_OK) return rc;
    HV_CUDA(hv_launch_fast(a, c->stream));
    c->launches += 2;
    return HV_OK;
}

int hv_fast_detect(hv_ctx* c, hv_pyr* pyr, int threshold, int nonmax, float* xy, float* response, int capacity, int* count)
{
    FastArgs a;
    size_t bytes = 0;
    int rc = fast_args("hv_fast_detect", c, pyr, threshold, nonmax, xy, response, capacity, count, a, &bytes);
    if (rc != HV_OK) return rc;
    HV_CUDA(cudaSetDevice(c->device));
    rc = fast_scratch(c, &a, &bytes, 1);
    if (rc != HV_OK) return rc;
    // staging block: [count (16 bytes) | xy 8 capacity | response 4 capacity]
    const size_t oXY = 16, oResp = oXY + 8 * (size_t)capacity, total = oResp + (response ? 4 * (size_t)capacity : 0);
    rc = hv_ctx_reserve_stage(c, total);
    if (rc != HV_OK) return rc;
    uint8_t* hs = (uint8_t*)c->h_stage; uint8_t* ds = (uint8_t*)c->d_stage;
    a.count = (int*)ds; a.xy = (float2*)(ds + oXY); a.response = response ? (float*)(ds + oResp) : nullptr;
    HV_CUDA(hv_launch_fast(a, c->stream));
    c->launches += 2;
    HV_CUDA(cudaMemcpyAsync(hs, ds, total, cudaMemcpyDeviceToHost, c->stream));
    HV_CUDA(cudaStreamSynchronize(c->stream));
    memcpy(count, hs, sizeof(int));
    if (capacity > 0) memcpy(xy, hs + oXY, 8 * (size_t)capacity);
    if (response && capacity > 0) memcpy(response, hs + oResp, 4 * (size_t)capacity);
    return HV_OK;
}

int hv_fast_detect_batch_device(hv_ctx* c, const hv_fast_job* jobs, int njobs, int threshold, int nonmax)
{
    int rc = corner_batch_check("hv_fast_detect_batch_device", c, jobs, njobs);
    if (rc != HV_OK) return rc;
    FastBatchArgs b;
    memset(&b, 0, sizeof(b));
    size_t bytes[HV_CORNER_BATCH_MAX];
    long long tiles = 0, bands = 0;
    for (int j = 0; j < njobs; j++) {
        const hv_fast_job& J = jobs[j];
        char who[64];
        snprintf(who, sizeof(who), "hv_fast_detect_batch_device job %d", j);
        rc = fast_args(who, c, J.pyr, threshold, nonmax, J.d_xy, J.d_response, J.capacity, J.d_count, b.job[j], &bytes[j]);
        if (rc != HV_OK) return rc;
        b.firstTile[j] = (int)tiles; b.firstBand[j] = (int)bands;
        tiles += (long long)b.job[j].tilesX * b.job[j].tilesY;
        bands += b.job[j].tilesY;
        if (tiles > INT_MAX) { hv_set_error("%s: more than %d tiles in one batch", who, INT_MAX); return HV_ERR_INVALID; }
    }
    for (int j = njobs; j <= HV_CORNER_BATCH_MAX; j++) { b.firstTile[j] = (int)tiles; b.firstBand[j] = (int)bands; }
    HV_CUDA(cudaSetDevice(c->device));
    rc = fast_scratch(c, b.job, bytes, njobs);
    if (rc != HV_OK) return rc;
    HV_CUDA(hv_launch_fast_batch(b, njobs, c->stream));
    c->launches += 2;
    return HV_OK;
}

// ------------------------------------------------------------------------------------------------ Shi-Tomasi corner detection (N2)
// Scratch: HV_CORNER_BATCH_MAX (max word, candidate count) pairs at the front (job j of a call uses pair j; the call zeroes the pairs it
// uses on the stream before its first launch), then per job its response map, candidate keys and min-distance grid.
static const size_t GF_WORDS = align_up(HV_CORNER_BATCH_MAX * 2 * sizeof(unsigned), 256);

// Checks one job and fills everything but the scratch; *scratch = the bytes of map, keys and grid it needs.
static int gf_args(const char* who, hv_ctx* c, hv_pyr* pyr, int blockSize, int maxCorners, double quality, double minDistance,
                   const uint8_t* mask, size_t maskStride, float* xy, float* response, int capacity, int* count, GoodFeaturesArgs& a,
                   size_t* scratch)
{
    if (!c || !pyr || pyr->ctx != c) { hv_set_error("%s: invalid context / pyramid", who); return HV_ERR_INVALID; }
    if (!xy || !count) { hv_set_error("%s: NULL xy or count", who); return HV_ERR_INVALID; }
    if (blockSize != 3) { hv_set_error("%s: block size %d unsupported (3 only)", who, blockSize); return HV_ERR_UNSUPPORTED; }
    if (maxCorners < 1) { hv_set_error("%s: max_corners %d unsupported (1 or more)", who, maxCorners); return HV_ERR_UNSUPPORTED; }
    if (capacity < maxCorners) { hv_set_error("%s: capacity %d below max_corners %d", who, capacity, maxCorners); return HV_ERR_INVALID; }
    if (!(quality > 0.0)) { hv_set_error("%s: quality_level %g (must be > 0)", who, quality); return HV_ERR_INVALID; }
    if (!(minDistance >= 0.0) || !std::isfinite(minDistance)) {
        hv_set_error("%s: min_distance %g (must be finite and >= 0)", who, minDistance);
        return HV_ERR_INVALID;
    }
    const HvLevel& L = pyr->desc.lv[0];
    if (mask && maskStride < (size_t)L.w) { hv_set_error("%s: mask stride %zu below the width %d", who, maskStride, L.w); return HV_ERR_INVALID; }
    if (mask && maskStride > (size_t)INT_MAX) { hv_set_error("%s: mask stride %zu too large", who, maskStride); return HV_ERR_INVALID; }
    memset(&a, 0, sizeof(a));
    a.gray = L.gray; a.pitch = L.gpitch; a.w = L.w; a.h = L.h;
    a.mask = mask; a.maskPitch = (int)maskStride;
    a.tilesX = (L.w + 31) / 32; a.tilesY = (L.h + 7) / 8;
    a.maxCorners = maxCorners; a.quality = quality;
    a.xy = (float2*)xy; a.response = response; a.capacity = capacity; a.count = count;
    a.useGrid = minDistance >= 1.0;
    size_t gridBytes = 0;
    if (a.useGrid) {
        // cell side s: the largest with 2 (s - 1)^2 < minDistance^2, so two corners in one cell are always too close and a cell holds at
        // most one kept corner; s - 1 <= 2896 keeps (s - 1)^2 exact in the fp32 distance test. reach: the largest |dx| that can be too close.
        const int big = L.w > L.h ? L.w : L.h;
        a.md2 = minDistance * minDistance;
        long long s = (long long)(minDistance / 1.4142135623730951);
        if (s > 2897) s = 2897;
        if (s < 1) s = 1;
        while (s > 1 && 2.0 * (double)(s - 1) * (double)(s - 1) >= a.md2) s--;
        while (s < 2897 && 2.0 * (double)s * (double)s < a.md2) s++;
        a.cell = (int)s;
        const double r = std::ceil(minDistance) - 1.0;
        a.reach = r > (double)big ? big : (int)r;
        a.gridW = (L.w + a.cell - 1) / a.cell; a.gridH = (L.h + a.cell - 1) / a.cell;
        gridBytes = align_up(sizeof(int) * (size_t)a.gridW * a.gridH, 256);
    }
    const size_t interior = L.w > 2 && L.h > 2 ? (size_t)(L.w - 2) * (L.h - 2) : 1;
    *scratch = align_up(sizeof(float) * (size_t)L.w * L.h, 256) + align_up(sizeof(unsigned long long) * interior, 256) + gridBytes;
    return HV_OK;
}

// points the jobs' words, maps, keys and grids into the context's scratch, grown (after the work that may still read it) as needed
static int gf_scratch(hv_ctx* c, GoodFeaturesArgs* jobs, const size_t* bytes, int njobs)
{
    size_t total = GF_WORDS;
    for (int j = 0; j < njobs; j++) total += bytes[j];
    if (total > c->gfScratchBytes) {
        if (c->d_gfScratch) { HV_CUDA(cudaStreamSynchronize(c->stream)); cudaFree(c->d_gfScratch); }
        c->d_gfScratch = nullptr; c->gfScratchBytes = 0;
        size_t cap = 1 << 20; while (cap < total) cap *= 2;
        HV_CUDA(cudaMalloc(&c->d_gfScratch, cap));
        c->gfScratchBytes = cap;
    }
    HV_CUDA(cudaMemsetAsync(c->d_gfScratch, 0, 2 * sizeof(unsigned) * (size_t)njobs, c->stream));
    uint8_t* p = (uint8_t*)c->d_gfScratch;
    unsigned* words = (unsigned*)p;
    p += GF_WORDS;
    for (int j = 0; j < njobs; j++) {
        GoodFeaturesArgs& a = jobs[j];
        a.maxWord = words + 2 * j;
        a.nCand = (int*)(words + 2 * j + 1);
        uint8_t* q = p;
        a.eig = (float*)q; q += align_up(sizeof(float) * (size_t)a.w * a.h, 256);
        a.maxCand = a.w > 2 && a.h > 2 ? (a.w - 2) * (a.h - 2) : 1;
        a.keys = (unsigned long long*)q; q += align_up(sizeof(unsigned long long) * (size_t)a.maxCand, 256);
        a.grid = a.useGrid ? (int*)q : nullptr;
        p += bytes[j];
    }
    return HV_OK;
}

int hv_good_features_device(hv_ctx* c, hv_pyr* pyr, int blockSize, int maxCorners, double quality, double minDistance,
                            const uint8_t* dMask, size_t maskStride, float* dXY, float* dResponse, int capacity, int* dCount)
{
    GoodFeaturesArgs a;
    size_t bytes = 0;
    int rc = gf_args("hv_good_features_device", c, pyr, blockSize, maxCorners, quality, minDistance, dMask, maskStride, dXY, dResponse,
                     capacity, dCount, a, &bytes);
    if (rc != HV_OK) return rc;
    HV_CUDA(cudaSetDevice(c->device));
    rc = gf_scratch(c, &a, &bytes, 1);
    if (rc != HV_OK) return rc;
    HV_CUDA(hv_launch_good_features(a, c->stream));
    c->launches += 3;
    return HV_OK;
}

int hv_good_features(hv_ctx* c, hv_pyr* pyr, int blockSize, int maxCorners, double quality, double minDistance, const uint8_t* mask,
                     size_t maskStride, float* xy, float* response, int capacity, int* count)
{
    GoodFeaturesArgs a;
    size_t bytes = 0;
    int rc = gf_args("hv_good_features", c, pyr, blockSize, maxCorners, quality, minDistance, mask, maskStride, xy, response, capacity,
                     count, a, &bytes);
    if (rc != HV_OK) return rc;
    HV_CUDA(cudaSetDevice(c->device));
    rc = gf_scratch(c, &a, &bytes, 1);
    if (rc != HV_OK) return rc;
    // staging block: [count (16 bytes) | xy 8 capacity | response 4 capacity | mask]
    const size_t oXY = 16, oResp = oXY + 8 * (size_t)capacity, oMask = align_up(oResp + (response ? 4 * (size_t)capacity : 0), 16);
    const size_t maskBytes = mask ? maskStride * (size_t)(a.h - 1) + (size_t)a.w : 0;
    rc = hv_ctx_reserve_stage(c, oMask + maskBytes);
    if (rc != HV_OK) return rc;
    uint8_t* hs = (uint8_t*)c->h_stage; uint8_t* ds = (uint8_t*)c->d_stage;
    if (mask) {
        memcpy(hs + oMask, mask, maskBytes);
        HV_CUDA(cudaMemcpyAsync(ds + oMask, hs + oMask, maskBytes, cudaMemcpyHostToDevice, c->stream));
        a.mask = ds + oMask;
    }
    a.count = (int*)ds; a.xy = (float2*)(ds + oXY); a.response = response ? (float*)(ds + oResp) : nullptr;
    HV_CUDA(hv_launch_good_features(a, c->stream));
    c->launches += 3;
    HV_CUDA(cudaMemcpyAsync(hs, ds, oMask, cudaMemcpyDeviceToHost, c->stream));
    HV_CUDA(cudaStreamSynchronize(c->stream));
    memcpy(count, hs, sizeof(int));
    memcpy(xy, hs + oXY, 8 * (size_t)capacity);
    if (response) memcpy(response, hs + oResp, 4 * (size_t)capacity);
    return HV_OK;
}

int hv_good_features_batch_device(hv_ctx* c, const hv_good_features_job* jobs, int njobs, int blockSize, double quality, double minDistance)
{
    int rc = corner_batch_check("hv_good_features_batch_device", c, jobs, njobs);
    if (rc != HV_OK) return rc;
    GoodFeaturesBatchArgs b;
    memset(&b, 0, sizeof(b));
    size_t bytes[HV_CORNER_BATCH_MAX];
    long long tiles = 0, strips = 0;
    for (int j = 0; j < njobs; j++) {
        const hv_good_features_job& J = jobs[j];
        char who[64];
        snprintf(who, sizeof(who), "hv_good_features_batch_device job %d", j);
        rc = gf_args(who, c, J.pyr, blockSize, J.max_corners, quality, minDistance, J.d_mask, J.mask_stride, J.d_xy, J.d_response,
                     J.capacity, J.d_count, b.job[j], &bytes[j]);
        if (rc != HV_OK) return rc;
        b.firstTile[j] = (int)tiles; b.firstStrip[j] = (int)strips;
        tiles += (long long)b.job[j].tilesX * b.job[j].tilesY;
        strips += (b.job[j].w + 31) / 32;
        if (tiles > INT_MAX) { hv_set_error("%s: more than %d tiles in one batch", who, INT_MAX); return HV_ERR_INVALID; }
    }
    for (int j = njobs; j <= HV_CORNER_BATCH_MAX; j++) { b.firstTile[j] = (int)tiles; b.firstStrip[j] = (int)strips; }
    HV_CUDA(cudaSetDevice(c->device));
    rc = gf_scratch(c, b.job, bytes, njobs);
    if (rc != HV_OK) return rc;
    HV_CUDA(hv_launch_good_features_batch(b, njobs, c->stream));
    c->launches += 3;
    return HV_OK;
}

// ------------------------------------------------------------------------------------------------ essential-matrix RANSAC (N3)
// The parameters of the batch: refused as cv::findEssentialMat 4.13 refuses them (prob outside (0, 1), NaN included), or as the device
// cannot run them (more than HV_ESSENTIAL_MAX_ITERS iterations; maxIters <= 0 runs one, as OpenCV does).
static int ess_params(const char* who, double prob, int maxIters)
{
    if (!(prob > 0.0 && prob < 1.0)) { hv_set_error("%s: prob %g outside (0, 1)", who, prob); return HV_ERR_INVALID; }
    if (maxIters > HV_ESSENTIAL_MAX_ITERS) {
        hv_set_error("%s: max_iters %d above %d", who, maxIters, HV_ESSENTIAL_MAX_ITERS);
        return HV_ERR_UNSUPPORTED;
    }
    return HV_OK;
}

// Checks one job and fills everything but the scratch.
static int ess_args(const char* who, const float* xy1, const float* xy2, const uint8_t* status, int n, double fx, double fy, double cx,
                    double cy, double* E, int* nsol, uint8_t* mask, int* inliers, EssentialArgs& a)
{
    if (!E || !nsol || !inliers) { hv_set_error("%s: NULL E, nsol or inliers", who); return HV_ERR_INVALID; }
    if (n < 0) { hv_set_error("%s: n = %d", who, n); return HV_ERR_INVALID; }
    if (n > 0 && (!xy1 || !xy2 || !mask)) { hv_set_error("%s: NULL xy1, xy2 or mask", who); return HV_ERR_INVALID; }
    if (n > HV_ESSENTIAL_MAX_POINTS) { hv_set_error("%s: %d points (at most %d)", who, n, HV_ESSENTIAL_MAX_POINTS); return HV_ERR_UNSUPPORTED; }
    if (!std::isfinite(fx) || !std::isfinite(fy) || !std::isfinite(cx) || !std::isfinite(cy) || fx == 0.0 || fy == 0.0 || fx + fy == 0.0) {
        hv_set_error("%s: intrinsics (%g, %g, %g, %g) not finite or a zero focal length", who, fx, fy, cx, cy);
        return HV_ERR_UNSUPPORTED;
    }
    memset(&a, 0, sizeof(a));
    a.xy1 = (const float2*)xy1; a.xy2 = (const float2*)xy2; a.status = status; a.n = n;
    a.fx = fx; a.fy = fy; a.cx = cx; a.cy = cy;
    a.E = E; a.nsol = nsol; a.mask = mask; a.inliers = inliers;
    return HV_OK;
}

// points the jobs' normalised points and indices into the context's scratch, grown (after the work that may still read it) as needed
static int ess_scratch(hv_ctx* c, EssentialArgs* jobs, int njobs)
{
    size_t total = 0;
    for (int j = 0; j < njobs; j++) total += align_up(32 * (size_t)jobs[j].n, 256) + align_up(4 * (size_t)jobs[j].n, 256);
    if (total > c->essScratchBytes) {
        if (c->d_essScratch) { HV_CUDA(cudaStreamSynchronize(c->stream)); cudaFree(c->d_essScratch); }
        c->d_essScratch = nullptr; c->essScratchBytes = 0;
        size_t cap = 1 << 16; while (cap < total) cap *= 2;
        HV_CUDA(cudaMalloc(&c->d_essScratch, cap));
        c->essScratchBytes = cap;
    }
    uint8_t* p = (uint8_t*)c->d_essScratch;
    for (int j = 0; j < njobs; j++) {
        jobs[j].q = (double*)p; p += align_up(32 * (size_t)jobs[j].n, 256);
        jobs[j].idx = (int*)p; p += align_up(4 * (size_t)jobs[j].n, 256);
    }
    return HV_OK;
}

int hv_find_essential_device(hv_ctx* c, const float* dXY1, const float* dXY2, const uint8_t* dStatus, int n, double fx, double fy,
                             double cx, double cy, double prob, double threshold, int maxIters, double* dE, int* dNsol, uint8_t* dMask,
                             int* dInliers)
{
    const char* who = "hv_find_essential_device";
    if (!c) { hv_set_error("%s: NULL context", who); return HV_ERR_INVALID; }
    int rc = ess_params(who, prob, maxIters);
    if (rc != HV_OK) return rc;
    EssentialBatchArgs b;
    memset(&b, 0, sizeof(b));
    rc = ess_args(who, dXY1, dXY2, dStatus, n, fx, fy, cx, cy, dE, dNsol, dMask, dInliers, b.job[0]);
    if (rc != HV_OK) return rc;
    b.prob = prob; b.threshold = threshold; b.maxIters = maxIters;
    HV_CUDA(cudaSetDevice(c->device));
    rc = ess_scratch(c, b.job, 1);
    if (rc != HV_OK) return rc;
    HV_CUDA(hv_launch_essential(b, 1, c->stream));
    c->launches += 1;
    return HV_OK;
}

int hv_find_essential(hv_ctx* c, const float* xy1, const float* xy2, const uint8_t* status, int n, double fx, double fy, double cx,
                      double cy, double prob, double threshold, int maxIters, double* E, int* nsol, uint8_t* mask, int* inliers)
{
    const char* who = "hv_find_essential";
    if (!c) { hv_set_error("%s: NULL context", who); return HV_ERR_INVALID; }
    int rc = ess_params(who, prob, maxIters);
    if (rc != HV_OK) return rc;
    EssentialBatchArgs b;
    memset(&b, 0, sizeof(b));
    rc = ess_args(who, xy1, xy2, status, n, fx, fy, cx, cy, E, nsol, mask, inliers, b.job[0]);
    if (rc != HV_OK) return rc;
    b.prob = prob; b.threshold = threshold; b.maxIters = maxIters;
    HV_CUDA(cudaSetDevice(c->device));
    rc = ess_scratch(c, b.job, 1);
    if (rc != HV_OK) return rc;
    // staging block: [E 80 doubles | nsol, inliers | mask n] back to the host, [xy1 8n | xy2 8n | status n] to the device
    const size_t oMask = 8 * 90 + 16, oXY1 = align_up(oMask + (size_t)n, 16);
    const size_t oXY2 = oXY1 + 8 * (size_t)n, oSt = oXY2 + 8 * (size_t)n, total = oSt + (status ? (size_t)n : 0);
    rc = hv_ctx_reserve_stage(c, total);
    if (rc != HV_OK) return rc;
    uint8_t* hs = (uint8_t*)c->h_stage; uint8_t* ds = (uint8_t*)c->d_stage;
    if (n > 0) {
        memcpy(hs + oXY1, xy1, 8 * (size_t)n);
        memcpy(hs + oXY2, xy2, 8 * (size_t)n);
        if (status) memcpy(hs + oSt, status, (size_t)n);
    }
    if (total > oXY1) HV_CUDA(cudaMemcpyAsync(ds + oXY1, hs + oXY1, total - oXY1, cudaMemcpyHostToDevice, c->stream));
    EssentialArgs& a = b.job[0];
    a.xy1 = (const float2*)(ds + oXY1); a.xy2 = (const float2*)(ds + oXY2); a.status = status ? ds + oSt : nullptr;
    a.E = (double*)ds; a.nsol = (int*)(ds + 8 * 90); a.inliers = (int*)(ds + 8 * 90 + 4); a.mask = ds + oMask;
    HV_CUDA(hv_launch_essential(b, 1, c->stream));
    c->launches += 1;
    HV_CUDA(cudaMemcpyAsync(hs, ds, oMask + (size_t)n, cudaMemcpyDeviceToHost, c->stream));
    HV_CUDA(cudaStreamSynchronize(c->stream));
    memcpy(E, hs, 8 * 90);
    memcpy(nsol, hs + 8 * 90, sizeof(int));
    memcpy(inliers, hs + 8 * 90 + 4, sizeof(int));
    if (n > 0) memcpy(mask, hs + oMask, (size_t)n);
    return HV_OK;
}

int hv_find_essential_batch_device(hv_ctx* c, const hv_essential_job* jobs, int njobs, double prob, double threshold, int maxIters)
{
    const char* who = "hv_find_essential_batch_device";
    if (!c || !jobs) { hv_set_error("%s: NULL context or jobs", who); return HV_ERR_INVALID; }
    if (njobs < 1 || njobs > HV_ESSENTIAL_BATCH_MAX) { hv_set_error("%s: %d jobs (1..%d per call)", who, njobs, HV_ESSENTIAL_BATCH_MAX); return HV_ERR_INVALID; }
    int rc = ess_params(who, prob, maxIters);
    if (rc != HV_OK) return rc;
    EssentialBatchArgs b;
    memset(&b, 0, sizeof(b));
    for (int j = 0; j < njobs; j++) {
        const hv_essential_job& J = jobs[j];
        char w[64];
        snprintf(w, sizeof(w), "%s job %d", who, j);
        rc = ess_args(w, J.d_xy1, J.d_xy2, J.d_status, J.n, J.fx, J.fy, J.cx, J.cy, J.d_E, J.d_nsol, J.d_mask, J.d_inliers, b.job[j]);
        if (rc != HV_OK) return rc;
    }
    b.prob = prob; b.threshold = threshold; b.maxIters = maxIters;
    HV_CUDA(cudaSetDevice(c->device));
    rc = ess_scratch(c, b.job, njobs);
    if (rc != HV_OK) return rc;
    HV_CUDA(hv_launch_essential(b, njobs, c->stream));
    c->launches += 1;
    return HV_OK;
}

// ------------------------------------------------------------------------------------------------ relative pose from E (N3)
// Checks one job and fills its arguments; the intrinsics are refused as ess_args refuses them.
static int pose_args(const char* who, const double* E, const int* nsol, const float* xy1, const float* xy2, const uint8_t* maskIn, int n,
                     double fx, double fy, double cx, double cy, double* R, double* t, uint8_t* maskOut, int* good, PoseArgs& a)
{
    if (!E || !R || !t || !good) { hv_set_error("%s: NULL E, R, t or good", who); return HV_ERR_INVALID; }
    if (n < 0) { hv_set_error("%s: n = %d", who, n); return HV_ERR_INVALID; }
    if (n > 0 && (!xy1 || !xy2 || !maskOut)) { hv_set_error("%s: NULL xy1, xy2 or mask_out", who); return HV_ERR_INVALID; }
    if (n > HV_ESSENTIAL_MAX_POINTS) { hv_set_error("%s: %d points (at most %d)", who, n, HV_ESSENTIAL_MAX_POINTS); return HV_ERR_UNSUPPORTED; }
    if (!std::isfinite(fx) || !std::isfinite(fy) || !std::isfinite(cx) || !std::isfinite(cy) || fx == 0.0 || fy == 0.0) {
        hv_set_error("%s: intrinsics (%g, %g, %g, %g) not finite or a zero focal length", who, fx, fy, cx, cy);
        return HV_ERR_UNSUPPORTED;
    }
    memset(&a, 0, sizeof(a));
    a.E = E; a.nsol = nsol;
    a.xy1 = (const float2*)xy1; a.xy2 = (const float2*)xy2; a.maskIn = maskIn; a.n = n;
    a.fx = fx; a.fy = fy; a.cx = cx; a.cy = cy;
    a.R = R; a.t = t; a.maskOut = maskOut; a.good = good;
    return HV_OK;
}

int hv_recover_pose_device(hv_ctx* c, const double* dE, const int* dNsol, const float* dXY1, const float* dXY2, const uint8_t* dMaskIn, int n,
                           double fx, double fy, double cx, double cy, double dist, double* dR, double* dT, uint8_t* dMaskOut, int* dGood)
{
    const char* who = "hv_recover_pose_device";
    if (!c) { hv_set_error("%s: NULL context", who); return HV_ERR_INVALID; }
    PoseBatchArgs b;
    memset(&b, 0, sizeof(b));
    int rc = pose_args(who, dE, dNsol, dXY1, dXY2, dMaskIn, n, fx, fy, cx, cy, dR, dT, dMaskOut, dGood, b.job[0]);
    if (rc != HV_OK) return rc;
    b.dist = dist;
    HV_CUDA(cudaSetDevice(c->device));
    HV_CUDA(hv_launch_pose(b, 1, c->stream));
    c->launches += 1;
    return HV_OK;
}

int hv_recover_pose(hv_ctx* c, const double* E, const float* xy1, const float* xy2, const uint8_t* maskIn, int n, double fx, double fy,
                    double cx, double cy, double dist, double* R, double* t, uint8_t* maskOut, int* good)
{
    const char* who = "hv_recover_pose";
    if (!c) { hv_set_error("%s: NULL context", who); return HV_ERR_INVALID; }
    PoseBatchArgs b;
    memset(&b, 0, sizeof(b));
    int rc = pose_args(who, E, nullptr, xy1, xy2, maskIn, n, fx, fy, cx, cy, R, t, maskOut, good, b.job[0]);
    if (rc != HV_OK) return rc;
    for (int k = 0; k < 9; k++)
        if (!std::isfinite(E[k])) { hv_set_error("%s: E[%d] = %g is not finite", who, k, E[k]); return HV_ERR_UNSUPPORTED; }
    b.dist = dist;
    HV_CUDA(cudaSetDevice(c->device));
    // staging block: [R 9 | t 3 doubles | good | mask_out n] back to the host, [E 9 doubles | xy1 8n | xy2 8n | mask_in n] to the device
    const size_t oGood = 8 * 12, oMask = oGood + 16, oE = align_up(oMask + (size_t)n, 16), oXY1 = oE + 8 * 9;
    const size_t oXY2 = oXY1 + 8 * (size_t)n, oMi = oXY2 + 8 * (size_t)n, total = oMi + (maskIn ? (size_t)n : 0);
    rc = hv_ctx_reserve_stage(c, total);
    if (rc != HV_OK) return rc;
    uint8_t* hs = (uint8_t*)c->h_stage; uint8_t* ds = (uint8_t*)c->d_stage;
    memcpy(hs + oE, E, 8 * 9);
    if (n > 0) {
        memcpy(hs + oXY1, xy1, 8 * (size_t)n);
        memcpy(hs + oXY2, xy2, 8 * (size_t)n);
        if (maskIn) memcpy(hs + oMi, maskIn, (size_t)n);
    }
    HV_CUDA(cudaMemcpyAsync(ds + oE, hs + oE, total - oE, cudaMemcpyHostToDevice, c->stream));
    PoseArgs& a = b.job[0];
    a.E = (const double*)(ds + oE); a.xy1 = (const float2*)(ds + oXY1); a.xy2 = (const float2*)(ds + oXY2);
    a.maskIn = maskIn ? ds + oMi : nullptr;
    a.R = (double*)ds; a.t = (double*)(ds + 8 * 9); a.good = (int*)(ds + oGood); a.maskOut = ds + oMask;
    HV_CUDA(hv_launch_pose(b, 1, c->stream));
    c->launches += 1;
    HV_CUDA(cudaMemcpyAsync(hs, ds, oMask + (size_t)n, cudaMemcpyDeviceToHost, c->stream));
    HV_CUDA(cudaStreamSynchronize(c->stream));
    memcpy(R, hs, 8 * 9);
    memcpy(t, hs + 8 * 9, 8 * 3);
    memcpy(good, hs + oGood, sizeof(int));
    if (n > 0) memcpy(maskOut, hs + oMask, (size_t)n);
    return HV_OK;
}

int hv_recover_pose_batch_device(hv_ctx* c, const hv_pose_job* jobs, int njobs, double dist)
{
    const char* who = "hv_recover_pose_batch_device";
    if (!c || !jobs) { hv_set_error("%s: NULL context or jobs", who); return HV_ERR_INVALID; }
    if (njobs < 1 || njobs > HV_ESSENTIAL_BATCH_MAX) { hv_set_error("%s: %d jobs (1..%d per call)", who, njobs, HV_ESSENTIAL_BATCH_MAX); return HV_ERR_INVALID; }
    PoseBatchArgs b;
    memset(&b, 0, sizeof(b));
    for (int j = 0; j < njobs; j++) {
        const hv_pose_job& J = jobs[j];
        char w[64];
        snprintf(w, sizeof(w), "%s job %d", who, j);
        const int rc = pose_args(w, J.d_E, J.d_nsol, J.d_xy1, J.d_xy2, J.d_mask_in, J.n, J.fx, J.fy, J.cx, J.cy, J.d_R, J.d_t, J.d_mask_out,
                                 J.d_good, b.job[j]);
        if (rc != HV_OK) return rc;
    }
    b.dist = dist;
    HV_CUDA(cudaSetDevice(c->device));
    HV_CUDA(hv_launch_pose(b, njobs, c->stream));
    c->launches += 1;
    return HV_OK;
}

// ------------------------------------------------------------------------------------------------ frame ingest (N4)
struct hv_ingest {
    hv_ctx* ctx = nullptr;
    int w = 0, h = 0;
    uint8_t* d_raw = nullptr; size_t rawBytes = 0;     // the frame as it arrived (device)
    uint8_t* d_gray = nullptr;                          // gray before the remap (w x h, pitch w: a remap tap right of the last column
                                                        // reads the next row's first pixel, as the reference's contiguous image does)
    HvRemapEntry* d_table = nullptr;
};

int hv_ingest_create(hv_ctx* c, int w, int h, hv_ingest** out)
{
    if (!c || !out || w <= 0 || h <= 0 || w > 32767 || h > 32767) { hv_set_error("hv_ingest_create: invalid argument"); return HV_ERR_INVALID; }
    HV_CUDA(cudaSetDevice(c->device));
    hv_ingest* g = new hv_ingest;
    g->ctx = c; g->w = w; g->h = h;
    cudaError_t e = cudaMalloc(&g->d_gray, (size_t)w * h);
    if (e != cudaSuccess) { delete g; hv_set_error("hv_ingest_create: %s", cudaGetErrorString(e)); return HV_ERR_OOM; }
    *out = g;
    return HV_OK;
}
int hv_ingest_destroy(hv_ingest* g)
{
    if (!g) return HV_OK;
    cudaStreamSynchronize(g->ctx->stream);
    cudaFree(g->d_raw); cudaFree(g->d_gray); cudaFree(g->d_table);
    delete g;
    return HV_OK;
}
int hv_ingest_set_remap(hv_ingest* g, const hv_remap_entry* table)
{
    if (!g) { hv_set_error("hv_ingest_set_remap: NULL handle"); return HV_ERR_INVALID; }
    static_assert(sizeof(hv_remap_entry) == sizeof(HvRemapEntry) && sizeof(HvRemapEntry) == 12, "remap entry layout");
    HV_CUDA(cudaSetDevice(g->ctx->device));
    HV_CUDA(cudaStreamSynchronize(g->ctx->stream));
    if (!table) { cudaFree(g->d_table); g->d_table = nullptr; return HV_OK; }
    const size_t bytes = sizeof(HvRemapEntry) * (size_t)g->w * g->h;
    if (!g->d_table) HV_CUDA(cudaMalloc(&g->d_table, bytes));
    HV_CUDA(cudaMemcpy(g->d_table, table, bytes, cudaMemcpyHostToDevice));
    return HV_OK;
}
// the four fp32 coefficients of a colour frame: the reference's defaults (image.cpp:360-366), or coeff[i] for the frame's channels and 0
// past them
static void ingest_coeff(const double* coeff, int channels, float cf[4])
{
    const float def[4] = {0.299f, 0.587f, 0.114f, 0.0f};
    for (int i = 0; i < 4; i++) cf[i] = coeff ? (i < channels ? (float)coeff[i] : 0.0f) : def[i];
}
// grows the staging buffer of the frame as it arrives to at least `need` bytes
static int ingest_reserve_raw(hv_ingest* g, size_t need)
{
    if (need <= g->rawBytes) return HV_OK;
    cudaStreamSynchronize(g->ctx->stream); cudaFree(g->d_raw); g->d_raw = nullptr; g->rawBytes = 0;
    HV_CUDA(cudaMalloc(&g->d_raw, need)); g->rawBytes = need;
    return HV_OK;
}
int hv_ingest_frame(hv_ingest* g, const uint8_t* src, size_t stride, int channels, const double* coeff, hv_pyr* dst, uint8_t* grayOut)
{
    if (!g || !src || !dst || channels < 1 || channels > 4 || dst->ctx != g->ctx || dst->w != g->w || dst->h != g->h || stride < (size_t)g->w * channels) {
        hv_set_error("hv_ingest_frame: invalid argument"); return HV_ERR_INVALID;
    }
    hv_ctx* c = g->ctx;
    HV_CUDA(cudaSetDevice(c->device));
    const int w = g->w, h = g->h;
    const HvLevel& L0 = dst->desc.lv[0];
    const bool colour = channels > 1, remap = g->d_table != nullptr;
    if (!colour && !remap) {                                     // plain gray frame: exactly hv_pyr_build
        int rc = hv_pyr_build(dst, src, stride);
        if (rc != HV_OK) return rc;
    } else {
        const size_t need = stride * (h - 1) + (size_t)w * channels;                               // up to the last pixel: no byte past it
        const int rc = ingest_reserve_raw(g, need);
        if (rc != HV_OK) return rc;
        HV_CUDA(cudaMemcpyAsync(g->d_raw, src, need, cudaMemcpyHostToDevice, c->stream));          // the only trip of the frame over PCIe
        const uint8_t* cur = g->d_raw; int curPitch = (int)stride;
        if (colour) {
            float cf[4];
            ingest_coeff(coeff, channels, cf);
            uint8_t* out = remap ? g->d_gray : L0.gray; const int op = remap ? w : L0.gpitch;
            HV_CUDA(hv_launch_gray(cur, curPitch, channels, w, h, cf, out, op, c->stream));
            c->launches += 1;
            cur = out; curPitch = op;
        }
        if (remap) { HV_CUDA(hv_launch_remap(cur, curPitch, w, h, g->d_table, L0.gray, L0.gpitch, c->stream)); c->launches += 1; }
        // level 0 of the pyramid now holds the ingested image: build the rest in place (no second copy of the frame)
        unsigned short idx = (unsigned short)dst->slot;
        const uint8_t* l0 = L0.gray; const int l0p = L0.gpitch, nl = dst->nlevels;
        HV_CUDA(hv_launch_pyr_fused(c->d_table, &idx, nullptr, nullptr, &l0, &l0p, &nl, 1, w, h, nl, c->stream));
        c->launches += 1;
    }
    if (grayOut) HV_CUDA(cudaMemcpy2DAsync(grayOut, (size_t)w, L0.gray, (size_t)L0.gpitch, (size_t)w, (size_t)h, cudaMemcpyDeviceToHost, c->stream));
    return HV_OK;
}

// ------------------------------------------------------------------------------------------------ frame ingest of many frames
static inline bool ingest_needs_kernel(const hv_ingest_job& J) { return J.channels > 1 || J.ing->d_table != nullptr; }
static inline size_t ingest_src_bytes(const hv_ingest_job& J) { return J.stride_bytes * (J.ing->h - 1) + (size_t)J.ing->w * J.channels; }

static int ingest_frames_check(const hv_ingest_job* jobs, int njobs, int srcIsDevice)
{
    const char* who = "hv_ingest_frames";
    if (!jobs || njobs < 1 || njobs > HV_INGEST_BATCH_MAX) { hv_set_error("%s: NULL jobs or %d jobs (1..%d per call)", who, njobs, HV_INGEST_BATCH_MAX); return HV_ERR_INVALID; }
    const hv_ctx* c = jobs[0].ing ? jobs[0].ing->ctx : nullptr;
    for (int j = 0; j < njobs; j++) {
        const hv_ingest_job& J = jobs[j];
        const hv_ingest* g = J.ing;
        const hv_pyr* p = J.dst;
        if (!g || !J.src || !p) { hv_set_error("%s: job %d: NULL ing, src or dst", who, j); return HV_ERR_INVALID; }
        if (J.channels < 1 || J.channels > 4 || J.stride_bytes < (size_t)g->w * J.channels) {
            hv_set_error("%s: job %d: %d channels, stride %zu for width %d", who, j, J.channels, J.stride_bytes, g->w); return HV_ERR_INVALID;
        }
        if (g->ctx != c || p->ctx != c) { hv_set_error("%s: job %d: ing or dst of another context than job 0", who, j); return HV_ERR_INVALID; }
        if (p->w != g->w || p->h != g->h) { hv_set_error("%s: job %d: pyramid %dx%d for frames of %dx%d", who, j, p->w, p->h, g->w, g->h); return HV_ERR_INVALID; }
        for (int k = 0; k < j; k++)
            if (jobs[k].ing == g || jobs[k].dst == p) { hv_set_error("%s: job %d: the hv_ingest or pyramid of job %d again", who, j, k); return HV_ERR_INVALID; }
    }
    if (srcIsDevice)        // the call writes every job's pyramid while it reads the sources
        for (int j = 0; j < njobs; j++) {
            const uintptr_t a = (uintptr_t)jobs[j].src, ae = a + ingest_src_bytes(jobs[j]);
            for (int k = 0; k < njobs; k++) {
                const uintptr_t b = (uintptr_t)jobs[k].dst->d_mem, be = b + jobs[k].dst->bytes;
                if (a < be && b < ae) { hv_set_error("%s: job %d: the device source overlaps the pyramid of job %d", who, j, k); return HV_ERR_INVALID; }
            }
        }
    return HV_OK;
}

int hv_ingest_frames(const hv_ingest_job* jobs, int njobs, int srcIsDevice)
{
    int rc = ingest_frames_check(jobs, njobs, srcIsDevice);
    if (rc != HV_OK) return rc;
    hv_ctx* c = jobs[0].ing->ctx;
    HV_CUDA(cudaSetDevice(c->device));
    // host sources: one copy each, into the hv_ingest's staging buffer (kernel jobs) or level 0 of the pyramid (gray jobs without a table)
    if (!srcIsDevice) {
        for (int j = 0; j < njobs; j++)
            if (ingest_needs_kernel(jobs[j]) && (rc = ingest_reserve_raw(jobs[j].ing, ingest_src_bytes(jobs[j]))) != HV_OK) return rc;
        for (int j = 0; j < njobs; j++) {
            const hv_ingest_job& J = jobs[j];
            const HvLevel& L0 = J.dst->desc.lv[0];
            if (ingest_needs_kernel(J))
                HV_CUDA(cudaMemcpyAsync(J.ing->d_raw, J.src, ingest_src_bytes(J), cudaMemcpyHostToDevice, c->stream));
            else if (J.stride_bytes == (size_t)L0.gpitch)                // as hv_pyr_build_batch copies a host frame
                HV_CUDA(cudaMemcpyAsync(L0.gray, J.src, (size_t)L0.gpitch * (L0.h - 1) + L0.w, cudaMemcpyHostToDevice, c->stream));
            else
                HV_CUDA(cudaMemcpy2DAsync(L0.gray, L0.gpitch, J.src, J.stride_bytes, (size_t)L0.w, (size_t)L0.h, cudaMemcpyHostToDevice, c->stream));
        }
    }
    // colour and / or remap into level 0: HV_CORNER_BATCH_MAX jobs per launch
    static_assert(HV_INGEST_BATCH_MAX <= 2 * HV_CORNER_BATCH_MAX, "at most two ingest launches per call");
    IngestBatchArgs b;
    int nb = 0, ctas = 0;
    for (int j = 0; j <= njobs; j++) {
        if (j < njobs && ingest_needs_kernel(jobs[j])) {
            const hv_ingest_job& J = jobs[j];
            const HvLevel& L0 = J.dst->desc.lv[0];
            if (nb == 0) memset(&b, 0, sizeof(b));
            IngestJob& K = b.job[nb];
            K.src = srcIsDevice ? J.src : J.ing->d_raw; K.srcPitch = (int)J.stride_bytes; K.channels = J.channels;
            ingest_coeff(J.coeff, J.channels, K.coeff);
            K.table = J.ing->d_table;
            K.dst = L0.gray; K.dstPitch = L0.gpitch; K.w = L0.w; K.h = L0.h;
            b.first[nb++] = ctas;
            ctas += (L0.w + 255) / 256 * L0.h;                                // at most 64 x 128 x 32767: no overflow
        }
        if (nb > 0 && (nb == HV_CORNER_BATCH_MAX || j == njobs)) {
            for (int k = nb; k <= HV_CORNER_BATCH_MAX; k++) b.first[k] = ctas;
            HV_CUDA(hv_launch_ingest_batch(b, nb, c->stream));
            c->launches += 1;
            nb = 0; ctas = 0;
        }
    }
    // the pyramids, one hv_launch_pyr_fused call per level-0 size (one launch per 32 frames)
    std::vector<char> built(njobs, 0);
    std::vector<unsigned short> idx;
    std::vector<const uint8_t*> src, l0;
    std::vector<int> srcPitch, l0Pitch, nls;
    for (int j = 0; j < njobs; j++) {
        if (built[j]) continue;
        const int w = jobs[j].dst->w, h = jobs[j].dst->h;
        idx.clear(); src.clear(); l0.clear(); srcPitch.clear(); l0Pitch.clear(); nls.clear();
        int maxNl = 0;
        for (int k = j; k < njobs; k++) {
            const hv_ingest_job& J = jobs[k];
            if (built[k] || J.dst->w != w || J.dst->h != h) continue;
            built[k] = 1;
            const bool inPlace = srcIsDevice && !ingest_needs_kernel(J);     // device gray frame: the pyramid kernel reads it in place
            const HvLevel& L0 = J.dst->desc.lv[0];
            idx.push_back((unsigned short)J.dst->slot);
            src.push_back(inPlace ? J.src : nullptr); srcPitch.push_back(inPlace ? (int)J.stride_bytes : 0);
            l0.push_back(L0.gray); l0Pitch.push_back(L0.gpitch); nls.push_back(J.dst->nlevels);
            if (J.dst->nlevels > maxNl) maxNl = J.dst->nlevels;
        }
        const int n = (int)idx.size();
        HV_CUDA(hv_launch_pyr_fused(c->d_table, idx.data(), src.data(), srcPitch.data(), l0.data(), l0Pitch.data(), nls.data(), n, w, h, maxNl, c->stream));
        c->launches += (n + 31) / 32;
    }
    for (int j = 0; j < njobs; j++) {
        const hv_ingest_job& J = jobs[j];
        const HvLevel& L0 = J.dst->desc.lv[0];
        if (J.gray_out) HV_CUDA(cudaMemcpy2DAsync(J.gray_out, (size_t)L0.w, L0.gray, (size_t)L0.gpitch, (size_t)L0.w, (size_t)L0.h, cudaMemcpyDeviceToHost, c->stream));
    }
    return HV_OK;
}

} // extern "C"
