// hybvio_b200/csrc/lk.cu -- pyramidal Lucas-Kanade tracker for sm_90a, one warp per feature, all levels in
// one launch. Compile with --fmad=false (the reference x86 build has no FMA; every fp32 op rounds separately).
//
// Replaces, for tracker::OpticalFlow::compute (src/tracker/optical_flow.cpp:10-59, 78-102), the reference's
//   SparsePyrLKOpticalFlowImpl::calc   OCV/video/src/lkpyramid.cpp:1236-1401  (level loop, criteria clamp)
//   LKTrackerInvoker::operator()       OCV/video/src/lkpyramid.cpp:183-724    (patch, 2x2 system, iterations)
// and the HybVIO status mapping of optical_flow.cpp:52-58.
//
// Mapping to the hardware
//   * lane x of the warp owns window column x (win <= 31, lane `win` carries the +1 bilinear column); the
//     31x31 I / (Ix,Iy) patch lives in registers (2 x 31 regs per lane) for the whole level.
//   * window rows are fetched as one coalesced 32-byte (gray) / 128-byte (gradient) warp load per row, all
//     rows issued back to back (32 independent loads in flight per lane) so a patch or an iteration costs
//     about one L2 round trip; the x+1 neighbour comes from __shfl_down, not from a second load.
//   * pyramid levels are stored unpadded; the reference's 31-px REFLECT_101 (gray) / zero (gradient) padding
//     (lkpyramid.cpp:761-808) is reproduced by per-lane column / per-row index reflection.
//   * fixed-point sample arithmetic (W_BITS 14, DESCALE 9 / 14) is integer and bit-exact with the reference.
//   * the 2x2 normal equations: per-lane int32 partial sums of the exact integer products (31 products per lane
//     cannot overflow), reduced across the warp with redux.sync on 16-bit halves into an exact int64 total,
//     rounded to fp32 ONCE. The reference accumulates the same products in fp32 SSE lanes
//     (lkpyramid.cpp:317-350, 556-562); the exact sum differs from it by <= ~1e-6 relative, which is what
//     the 1e-3 px end-point tolerance absorbs. The result is independent of reduction order => deterministic.
//   * all scalar float steps (D, minEig, delta, stop tests) are evaluated redundantly by every lane with
//     explicit round-to-nearest intrinsics, in the reference's operation order.
#include "hv_common.cuh"
#include <float.h>
#include <stdlib.h>

// search-window region of the next image staged per warp in shared memory: (32 + 2*margin) rows x 48 bytes
#define LK_REG_M 6
#define LK_REG_H (32 + 2 * LK_REG_M)
#define LK_REG_W 48

__device__ __forceinline__ int cv_floor(float v)
{
    // cvFloor (OCV/core/include/opencv2/core/fast_math.hpp:340-352) with the x86 out-of-range result
    if (!(fabsf(v) < 2147483648.f)) return INT_MIN;
    return __float2int_rd(v);
}

__device__ __forceinline__ long long warp_sum_exact(int v)
{
    // v = hi * 65536 + lo, lo in [0, 65535]; both partial sums fit int32 for 32 lanes
    int lo = v & 0xffff, hi = v >> 16;
    int slo = __reduce_add_sync(0xffffffffu, lo);
    int shi = __reduce_add_sync(0xffffffffu, hi);
    return (long long)shi * 65536 + (long long)slo;
}

__device__ __forceinline__ void bilin_weights(float a, float b, int& w00, int& w01, int& w10, int& w11)
{
    // lkpyramid.cpp:232-239; cvRound(float) = round-half-even
    const float oa = __fsub_rn(1.f, a), ob = __fsub_rn(1.f, b);
    w00 = __float2int_rn(__fmul_rn(__fmul_rn(oa, ob), 16384.f));
    w01 = __float2int_rn(__fmul_rn(__fmul_rn(a, ob), 16384.f));
    w10 = __float2int_rn(__fmul_rn(__fmul_rn(oa, b), 16384.f));
    w11 = 16384 - w00 - w01 - w10;
}

template <int WIN>
__global__ void __launch_bounds__(LK_WARPS_PER_CTA * 32) hv_lk_kernel(LkLaunch L)
{
    const LkJob& job = L.jobs[blockIdx.y];
    const int lane = threadIdx.x & 31;
    const int f = blockIdx.x * LK_WARPS_PER_CTA + (threadIdx.x >> 5);
    if (f >= job.n) return;

    const HvPyrDesc& PI = L.table[job.prevIdx];
    const HvPyrDesc& PJ = L.table[job.nextIdx];
    int maxLevel = min(L.maxLevel, min(PI.nlevels, PJ.nlevels) - 1);

    const float halfWin = (float)(WIN - 1) * 0.5f;
    const float FLT_SCALE = 1.f / (1 << 20);
    const int col = min(lane, WIN);            // lanes above WIN duplicate the last column (results unused)

    const float2 prevPt = job.prevPts[f];
    float2 outPt = job.useInitial ? (job.initPts ? job.initPts[f] : job.nextPts[f]) : prevPt;
    int status = 1;

    __shared__ __align__(16) uint8_t s_region[LK_WARPS_PER_CTA][LK_REG_H * LK_REG_W];
    uint8_t* reg = s_region[threadIdx.x >> 5];

    int Ipat[WIN];      // I patch column, x32 fixed point (lkpyramid.cpp:441)
    int dIpat[WIN];     // (Ix, Iy) packed as two int16

    for (int level = maxLevel; level >= 0; --level) {
        const HvLevel LI = PI.lv[level];
        const HvLevel LJ = PJ.lv[level];
        const float lscale = (float)(1. / (1 << level));
        float px = __fmul_rn(prevPt.x, lscale), py = __fmul_rn(prevPt.y, lscale);
        float nx, ny;
        if (level == maxLevel) {
            if (job.useInitial) { nx = __fmul_rn(outPt.x, lscale); ny = __fmul_rn(outPt.y, lscale); }
            else { nx = px; ny = py; }
        } else { nx = __fmul_rn(outPt.x, 2.f); ny = __fmul_rn(outPt.y, 2.f); }
        outPt.x = nx; outPt.y = ny;

        px = __fsub_rn(px, halfWin); py = __fsub_rn(py, halfWin);
        const int ipx = cv_floor(px), ipy = cv_floor(py);
        if (ipx < -WIN || ipx >= LI.w || ipy < -WIN || ipy >= LI.h) {
            if (level == 0) status = 0;
            continue;
        }
        int w00, w01, w10, w11;
        bilin_weights(__fsub_rn(px, (float)ipx), __fsub_rn(py, (float)ipy), w00, w01, w10, w11);

        // ---- template patch + gradient covariance (lkpyramid.cpp:272-471)
        int a11 = 0, a12 = 0, a22 = 0;
        {
            const int cx = ipx + col;
            const bool colOk = (unsigned)cx < (unsigned)LI.w;
            const int cxr = hv_reflect101(cx, LI.w);
            int v[WIN + 1], d[WIN + 1];
#pragma unroll
            for (int y = 0; y <= WIN; y++) {
                const int ry = ipy + y;
                const int ryr = hv_reflect101(ry, LI.h);
                v[y] = __ldg(LI.gray + (size_t)ryr * LI.gpitch + cxr);
                d[y] = (colOk && (unsigned)ry < (unsigned)LI.h)
                           ? __ldg(reinterpret_cast<const int*>(LI.deriv + (size_t)ry * LI.dpitch + cx)) : 0;
            }
            int vr0 = __shfl_down_sync(0xffffffffu, v[0], 1), dr0 = __shfl_down_sync(0xffffffffu, d[0], 1);
#pragma unroll
            for (int y = 0; y < WIN; y++) {
                const int vr1 = __shfl_down_sync(0xffffffffu, v[y + 1], 1);
                const int dr1 = __shfl_down_sync(0xffffffffu, d[y + 1], 1);
                const int ival = (v[y] * w00 + vr0 * w01 + v[y + 1] * w10 + vr1 * w11 + (1 << 8)) >> 9;
                const int x00 = (short)(d[y] & 0xffff), y00 = d[y] >> 16;
                const int x01 = (short)(dr0 & 0xffff), y01 = dr0 >> 16;
                const int x10 = (short)(d[y + 1] & 0xffff), y10 = d[y + 1] >> 16;
                const int x11 = (short)(dr1 & 0xffff), y11 = dr1 >> 16;
                const int ixv = (x00 * w00 + x01 * w01 + x10 * w10 + x11 * w11 + (1 << 13)) >> 14;
                const int iyv = (y00 * w00 + y01 * w01 + y10 * w10 + y11 * w11 + (1 << 13)) >> 14;
                Ipat[y] = ival;
                dIpat[y] = (ixv & 0xffff) | (iyv << 16);
                if (lane < WIN) { a11 += ixv * ixv; a12 += ixv * iyv; a22 += iyv * iyv; }
                vr0 = vr1; dr0 = dr1;
            }
        }
        const float A11 = __fmul_rn(__ll2float_rn(warp_sum_exact(a11)), FLT_SCALE);
        const float A12 = __fmul_rn(__ll2float_rn(warp_sum_exact(a12)), FLT_SCALE);
        const float A22 = __fmul_rn(__ll2float_rn(warp_sum_exact(a22)), FLT_SCALE);

        float D = __fsub_rn(__fmul_rn(A11, A22), __fmul_rn(A12, A12));
        const float dA = __fsub_rn(A11, A22);
        const float disc = __fadd_rn(__fmul_rn(dA, dA), __fmul_rn(__fmul_rn(4.f, A12), A12));
        const float minEig = __fdiv_rn(__fsub_rn(__fadd_rn(A22, A11), __fsqrt_rn(disc)), (float)(2 * WIN * WIN));
        if (minEig < L.minEig || D < FLT_EPSILON) {
            if (level == 0) status = 0;
            continue;
        }
        D = __fdiv_rn(1.f, D);

        // ---- Newton iterations (lkpyramid.cpp:492-681)
        nx = __fsub_rn(nx, halfWin); ny = __fsub_rn(ny, halfWin);
        float pdx = 0.f, pdy = 0.f;
        bool rgOk = false;          // the staged region belongs to this level's image
        int rx0 = 0, ry0 = 0;
        for (int j = 0; j < L.maxIter; j++) {
            const int inx = cv_floor(nx), iny = cv_floor(ny);
            if (inx < -WIN || inx >= LJ.w || iny < -WIN || iny >= LJ.h) {
                if (level == 0) status = 0;
                break;
            }
            bilin_weights(__fsub_rn(nx, (float)inx), __fsub_rn(ny, (float)iny), w00, w01, w10, w11);
            // The 32 x 32 search window is read from a (32 + 2*6)^2 region of the next image staged in shared memory; the
            // region is (re)filled only when the window leaves it, so an iteration costs shared-memory latency instead
            // of an L2 round trip. Region bytes are gray[reflect(y)][reflect(x)], i.e. exactly the reference's padded
            // image, so the samples are unchanged.
            if (!(rgOk && inx >= rx0 && inx + 32 <= rx0 + LK_REG_W && iny >= ry0 && iny + 32 <= ry0 + LK_REG_H)) {
                __syncwarp();
                rx0 = (inx - LK_REG_M) & ~3; ry0 = iny - LK_REG_M;
                if (rx0 >= 0 && rx0 + LK_REG_W <= LJ.w && ry0 >= 0 && ry0 + LK_REG_H <= LJ.h) {
                    const uint8_t* g0 = LJ.gray + (size_t)ry0 * LJ.gpitch + rx0;        // 4-byte aligned: gpitch % 4 == 0
#pragma unroll 6
                    for (int idx = lane; idx < LK_REG_H * (LK_REG_W / 4); idx += 32) {
                        const int row = idx / (LK_REG_W / 4), wd = idx - row * (LK_REG_W / 4);
                        reinterpret_cast<uint32_t*>(reg)[row * (LK_REG_W / 4) + wd] =
                            __ldg(reinterpret_cast<const uint32_t*>(g0 + (size_t)row * LJ.gpitch) + wd);
                    }
                } else {
                    // region touches the image border (common on the coarse levels): per-lane reflected columns once,
                    // rows reflected per row, all loads of 4 rows in flight
                    const int cA = hv_reflect101(rx0 + lane, LJ.w);
                    const bool hasB = lane + 32 < LK_REG_W;
                    const int cB = hv_reflect101(rx0 + (hasB ? lane + 32 : lane), LJ.w);
#pragma unroll 4
                    for (int row = 0; row < LK_REG_H; row++) {
                        const uint8_t* grow = LJ.gray + (size_t)hv_reflect101(ry0 + row, LJ.h) * LJ.gpitch;
                        const uint8_t a0 = __ldg(grow + cA), b0 = __ldg(grow + cB);
                        reg[row * LK_REG_W + lane] = a0;
                        if (hasB) reg[row * LK_REG_W + lane + 32] = b0;
                    }
                }
                rgOk = true;
                __syncwarp();
            }
            const uint8_t* rp = reg + (iny - ry0) * LK_REG_W + (inx - rx0) + col;
            int v[WIN + 1];
#pragma unroll
            for (int y = 0; y <= WIN; y++) v[y] = rp[y * LK_REG_W];
            int b1 = 0, b2 = 0;
            int vr0 = __shfl_down_sync(0xffffffffu, v[0], 1);
#pragma unroll
            for (int y = 0; y < WIN; y++) {
                const int vr1 = __shfl_down_sync(0xffffffffu, v[y + 1], 1);
                const int diff = ((v[y] * w00 + vr0 * w01 + v[y + 1] * w10 + vr1 * w11 + (1 << 8)) >> 9) - Ipat[y];
                b1 += diff * (int)(short)(dIpat[y] & 0xffff);
                b2 += diff * (dIpat[y] >> 16);
                vr0 = vr1;
            }
            if (lane >= WIN) { b1 = 0; b2 = 0; }
            const float fb1 = __fmul_rn(__ll2float_rn(warp_sum_exact(b1)), FLT_SCALE);
            const float fb2 = __fmul_rn(__ll2float_rn(warp_sum_exact(b2)), FLT_SCALE);
            const float dx = __fmul_rn(__fsub_rn(__fmul_rn(A12, fb2), __fmul_rn(A22, fb1)), D);
            const float dy = __fmul_rn(__fsub_rn(__fmul_rn(A12, fb1), __fmul_rn(A11, fb2)), D);
            nx = __fadd_rn(nx, dx); ny = __fadd_rn(ny, dy);
            outPt.x = __fadd_rn(nx, halfWin); outPt.y = __fadd_rn(ny, halfWin);
            if (__dadd_rn(__dmul_rn((double)dx, (double)dx), __dmul_rn((double)dy, (double)dy)) <= L.eps2) break;
            if (j > 0 && fabs((double)__fadd_rn(dx, pdx)) < 0.01 && fabs((double)__fadd_rn(dy, pdy)) < 0.01) {
                outPt.x = __fsub_rn(outPt.x, __fmul_rn(dx, 0.5f));
                outPt.y = __fsub_rn(outPt.y, __fmul_rn(dy, 0.5f));
                break;
            }
            pdx = dx; pdy = dy;
        }

        // ---- level-0 re-check of the final window position (lkpyramid.cpp:684-698; runs because HybVIO
        //      requests `err`, src/tracker/optical_flow.cpp:46-49)
        if (status && level == 0) {
            const int ix = cv_floor(__fsub_rn(outPt.x, halfWin)), iy = cv_floor(__fsub_rn(outPt.y, halfWin));
            if (ix < -WIN || ix >= LJ.w || iy < -WIN || iy >= LJ.h) status = 0;
        }
    }

    if (lane == 0) {
        job.nextPts[f] = outPt;
        job.status[f] = (uint8_t)status;
        if (job.trackStatus) {
            // src/tracker/optical_flow.cpp:52-58 against level 0 of the *next* pyramid
            int ts = status ? 0 /*TRACKED*/ : 2 /*FAILED_FLOW*/;
            const float W = (float)PJ.lv[0].w, H = (float)PJ.lv[0].h;
            if (outPt.x < 0.0f || outPt.x >= W || outPt.y < 0.0f || outPt.y >= H) ts = 4; /*FLOW_OUT_OF_RANGE*/
            job.trackStatus[f] = ts;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// CTA-per-feature variant (4 warps): the 31 window rows are split over the warps (8 rows each), so a patch build or an
// iteration is ~4x shorter; the per-warp exact integer partial sums meet in shared memory (one __syncthreads per
// iteration, double-buffered). Because the sums are exact integers, the result is BIT-IDENTICAL to the warp-per-feature
// kernel above for any split. Used when the launch has few features (one VIO session: 150 features on 132 SMs), where
// latency, not throughput, is what counts.
// Asynchronous global -> shared copies (LDGSTS): the search region of a level is requested before the template patch is loaded, so that
// the two dependent L2 round trips of a level become one (no registers in between). Plain copies on the host emulator.
__device__ __forceinline__ void lk_cp_async4(void* smemDst, const void* gsrc)
{
#ifdef HV_EMU
    *reinterpret_cast<uint32_t*>(smemDst) = *reinterpret_cast<const uint32_t*>(gsrc);
#else
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" :: "r"((unsigned)__cvta_generic_to_shared(smemDst)), "l"(gsrc) : "memory");
#endif
}
__device__ __forceinline__ void lk_cp_async_wait_all()
{
#ifndef HV_EMU
    asm volatile("cp.async.wait_all;" ::: "memory");
#endif
}

#define LKC_NW 4      // warps per feature
template <int WIN, int NW = LKC_NW>
__global__ void __launch_bounds__(NW * 32) hv_lk_cta_kernel(LkLaunch L)
{
    constexpr int RPW = (WIN + NW - 1) / NW;      // window rows per warp
#ifndef HV_EMU
    // Programmatic dependent launch: the next kernel of the stream (the stereo call behind the temporal one) may be scheduled now; this
    // one reads nothing (points, pyramids) before its predecessor has completed.
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");
#endif
    const LkJob& job = L.jobs[blockIdx.y];
    const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5, tid = threadIdx.x;
    const int f = blockIdx.x;
    if (f >= job.n) return;
    __shared__ __align__(16) uint8_t reg[LK_REG_H * LK_REG_W];
    __shared__ long long s_pa[NW][3];
    __shared__ long long s_pb[2][NW][2];

    const HvPyrDesc& PI = L.table[job.prevIdx];
    const HvPyrDesc& PJ = L.table[job.nextIdx];
    const int maxLevel = min(L.maxLevel, min(PI.nlevels, PJ.nlevels) - 1);
    const float halfWin = (float)(WIN - 1) * 0.5f;
    const float FLT_SCALE = 1.f / (1 << 20);
    const int col = min(lane, WIN);
    const int r0 = wrp * RPW;                               // first window row of this warp
    const int nr = max(0, min(RPW, WIN - r0));              // rows owned (the last warp may own fewer)

    const float2 prevPt = job.prevPts[f];
    float2 outPt = job.useInitial ? (job.initPts ? job.initPts[f] : job.nextPts[f]) : prevPt;
    int status = 1;
    int Ipat[RPW], dIpat[RPW];

    for (int level = maxLevel; level >= 0; --level) {
        const HvLevel LI = PI.lv[level];
        const HvLevel LJ = PJ.lv[level];
        const float lscale = (float)(1. / (1 << level));
        float px = __fmul_rn(prevPt.x, lscale), py = __fmul_rn(prevPt.y, lscale);
        float nx, ny;
        if (level == maxLevel) {
            if (job.useInitial) { nx = __fmul_rn(outPt.x, lscale); ny = __fmul_rn(outPt.y, lscale); }
            else { nx = px; ny = py; }
        } else { nx = __fmul_rn(outPt.x, 2.f); ny = __fmul_rn(outPt.y, 2.f); }
        outPt.x = nx; outPt.y = ny;

        px = __fsub_rn(px, halfWin); py = __fsub_rn(py, halfWin);
        const int ipx = cv_floor(px), ipy = cv_floor(py);
        if (ipx < -WIN || ipx >= LI.w || ipy < -WIN || ipy >= LI.h) {
            if (level == 0) status = 0;
            continue;
        }
        int w00, w01, w10, w11;
        bilin_weights(__fsub_rn(px, (float)ipx), __fsub_rn(py, (float)ipy), w00, w01, w10, w11);

        // ---- search region of the first iteration, requested NOW with cp.async (it only depends on the starting point of the level):
        // it arrives while the template patch below is being loaded and reduced. Same rx0 / ry0 as the iteration loop would choose.
        bool rgOk = false;
        int rx0 = 0, ry0 = 0;
        {
            lk_cp_async_wait_all();                          // a request of a level that was skipped after it was issued
            __syncthreads();
            const int inx0 = cv_floor(__fsub_rn(nx, halfWin)), iny0 = cv_floor(__fsub_rn(ny, halfWin));
            if (L.prefetch && !(inx0 < -WIN || inx0 >= LJ.w || iny0 < -WIN || iny0 >= LJ.h)) {
                const int qx = (inx0 - LK_REG_M) & ~3, qy = iny0 - LK_REG_M;
                if (qx >= 0 && qx + LK_REG_W <= LJ.w && qy >= 0 && qy + LK_REG_H <= LJ.h) {
                    const uint8_t* g0 = LJ.gray + (size_t)qy * LJ.gpitch + qx;
#pragma unroll
                    for (int u = 0; u < (LK_REG_H * (LK_REG_W / 4) + NW * 32 - 1) / (NW * 32); u++) {
                        const int idx = tid + u * NW * 32;
                        if (idx < LK_REG_H * (LK_REG_W / 4)) {
                            const int row = idx / (LK_REG_W / 4), wd = idx - row * (LK_REG_W / 4);
                            lk_cp_async4(reinterpret_cast<uint32_t*>(reg) + idx, reinterpret_cast<const uint32_t*>(g0 + (size_t)row * LJ.gpitch) + wd);
                        }
                    }
                    rgOk = true; rx0 = qx; ry0 = qy;
                }
            }
        }

        // ---- template patch rows r0 .. r0+nr-1 of this warp (+1 row for the bilinear tap)
        int a11 = 0, a12 = 0, a22 = 0;
        {
            const int cx = ipx + col;
            const bool colOk = (unsigned)cx < (unsigned)LI.w;
            const int cxr = hv_reflect101(cx, LI.w);
            int v[RPW + 1], d[RPW + 1];
#pragma unroll
            for (int y = 0; y <= RPW; y++) {
                const int ry = ipy + r0 + min(y, nr);
                const int ryr = hv_reflect101(ry, LI.h);
                v[y] = __ldg(LI.gray + (size_t)ryr * LI.gpitch + cxr);
                d[y] = (colOk && (unsigned)ry < (unsigned)LI.h)
                           ? __ldg(reinterpret_cast<const int*>(LI.deriv + (size_t)ry * LI.dpitch + cx)) : 0;
            }
            int vr0 = __shfl_down_sync(0xffffffffu, v[0], 1), dr0 = __shfl_down_sync(0xffffffffu, d[0], 1);
#pragma unroll
            for (int y = 0; y < RPW; y++) {
                const int vr1 = __shfl_down_sync(0xffffffffu, v[y + 1], 1);
                const int dr1 = __shfl_down_sync(0xffffffffu, d[y + 1], 1);
                const int ival = (v[y] * w00 + vr0 * w01 + v[y + 1] * w10 + vr1 * w11 + (1 << 8)) >> 9;
                const int x00 = (short)(d[y] & 0xffff), y00 = d[y] >> 16;
                const int x01 = (short)(dr0 & 0xffff), y01 = dr0 >> 16;
                const int x10 = (short)(d[y + 1] & 0xffff), y10 = d[y + 1] >> 16;
                const int x11 = (short)(dr1 & 0xffff), y11 = dr1 >> 16;
                const int ixv = (x00 * w00 + x01 * w01 + x10 * w10 + x11 * w11 + (1 << 13)) >> 14;
                const int iyv = (y00 * w00 + y01 * w01 + y10 * w10 + y11 * w11 + (1 << 13)) >> 14;
                Ipat[y] = ival;
                dIpat[y] = (ixv & 0xffff) | ((unsigned)iyv << 16);
                if (lane < WIN && y < nr) { a11 += ixv * ixv; a12 += ixv * iyv; a22 += iyv * iyv; }
                vr0 = vr1; dr0 = dr1;
            }
        }
        {
            const long long sa11 = warp_sum_exact(a11), sa12 = warp_sum_exact(a12), sa22 = warp_sum_exact(a22);
            lk_cp_async_wait_all();                          // own part of the search region has landed; the barrier publishes it
            __syncthreads();                                 // previous readers of s_pa are done
            if (lane == 0) { s_pa[wrp][0] = sa11; s_pa[wrp][1] = sa12; s_pa[wrp][2] = sa22; }
            __syncthreads();
        }
        long long tA11 = 0, tA12 = 0, tA22 = 0;
#pragma unroll
        for (int w = 0; w < NW; w++) { tA11 += s_pa[w][0]; tA12 += s_pa[w][1]; tA22 += s_pa[w][2]; }
        const float A11 = __fmul_rn(__ll2float_rn(tA11), FLT_SCALE);
        const float A12 = __fmul_rn(__ll2float_rn(tA12), FLT_SCALE);
        const float A22 = __fmul_rn(__ll2float_rn(tA22), FLT_SCALE);

        float D = __fsub_rn(__fmul_rn(A11, A22), __fmul_rn(A12, A12));
        const float dA = __fsub_rn(A11, A22);
        const float disc = __fadd_rn(__fmul_rn(dA, dA), __fmul_rn(__fmul_rn(4.f, A12), A12));
        const float minEig = __fdiv_rn(__fsub_rn(__fadd_rn(A22, A11), __fsqrt_rn(disc)), (float)(2 * WIN * WIN));
        if (minEig < L.minEig || D < FLT_EPSILON) {
            if (level == 0) status = 0;
            continue;
        }
        D = __fdiv_rn(1.f, D);

        nx = __fsub_rn(nx, halfWin); ny = __fsub_rn(ny, halfWin);
        float pdx = 0.f, pdy = 0.f;
        for (int j = 0; j < L.maxIter; j++) {
            const int inx = cv_floor(nx), iny = cv_floor(ny);
            if (inx < -WIN || inx >= LJ.w || iny < -WIN || iny >= LJ.h) {
                if (level == 0) status = 0;
                break;
            }
            bilin_weights(__fsub_rn(nx, (float)inx), __fsub_rn(ny, (float)iny), w00, w01, w10, w11);
            if (!(rgOk && inx >= rx0 && inx + 32 <= rx0 + LK_REG_W && iny >= ry0 && iny + 32 <= ry0 + LK_REG_H)) {
                __syncthreads();                             // everyone is done with the old region
                rx0 = (inx - LK_REG_M) & ~3; ry0 = iny - LK_REG_M;
                if (rx0 >= 0 && rx0 + LK_REG_W <= LJ.w && ry0 >= 0 && ry0 + LK_REG_H <= LJ.h) {
                    const uint8_t* g0 = LJ.gray + (size_t)ry0 * LJ.gpitch + rx0;
#pragma unroll
                    for (int u = 0; u < (LK_REG_H * (LK_REG_W / 4) + NW * 32 - 1) / (NW * 32); u++) {
                        const int idx = tid + u * NW * 32;
                        if (idx < LK_REG_H * (LK_REG_W / 4)) {
                            const int row = idx / (LK_REG_W / 4), wd = idx - row * (LK_REG_W / 4);
                            reinterpret_cast<uint32_t*>(reg)[idx] = __ldg(reinterpret_cast<const uint32_t*>(g0 + (size_t)row * LJ.gpitch) + wd);
                        }
                    }
                } else {
                    const int cA = hv_reflect101(rx0 + lane, LJ.w);
                    const bool hasB = lane + 32 < LK_REG_W;
                    const int cB = hv_reflect101(rx0 + (hasB ? lane + 32 : lane), LJ.w);
#pragma unroll 4
                    for (int row = wrp; row < LK_REG_H; row += NW) {
                        const uint8_t* grow = LJ.gray + (size_t)hv_reflect101(ry0 + row, LJ.h) * LJ.gpitch;
                        const uint8_t a0 = __ldg(grow + cA), b0 = __ldg(grow + cB);
                        reg[row * LK_REG_W + lane] = a0;
                        if (hasB) reg[row * LK_REG_W + lane + 32] = b0;
                    }
                }
                rgOk = true;
                __syncthreads();
            }
            const uint8_t* rp = reg + (iny - ry0 + r0) * LK_REG_W + (inx - rx0) + col;
            int v[RPW + 1];
#pragma unroll
            for (int y = 0; y <= RPW; y++) v[y] = rp[min(y, nr) * LK_REG_W];
            int b1 = 0, b2 = 0;
            int vr0 = __shfl_down_sync(0xffffffffu, v[0], 1);
#pragma unroll
            for (int y = 0; y < RPW; y++) {
                const int vr1 = __shfl_down_sync(0xffffffffu, v[y + 1], 1);
                const int diff = ((v[y] * w00 + vr0 * w01 + v[y + 1] * w10 + vr1 * w11 + (1 << 8)) >> 9) - Ipat[y];
                if (y < nr) { b1 += diff * (int)(short)(dIpat[y] & 0xffff); b2 += diff * (dIpat[y] >> 16); }
                vr0 = vr1;
            }
            if (lane >= WIN) { b1 = 0; b2 = 0; }
            const long long sb1 = warp_sum_exact(b1), sb2 = warp_sum_exact(b2);
            if (lane == 0) { s_pb[j & 1][wrp][0] = sb1; s_pb[j & 1][wrp][1] = sb2; }
            __syncthreads();
            long long tb1 = 0, tb2 = 0;
#pragma unroll
            for (int w = 0; w < NW; w++) { tb1 += s_pb[j & 1][w][0]; tb2 += s_pb[j & 1][w][1]; }
            const float fb1 = __fmul_rn(__ll2float_rn(tb1), FLT_SCALE);
            const float fb2 = __fmul_rn(__ll2float_rn(tb2), FLT_SCALE);
            const float dx = __fmul_rn(__fsub_rn(__fmul_rn(A12, fb2), __fmul_rn(A22, fb1)), D);
            const float dy = __fmul_rn(__fsub_rn(__fmul_rn(A12, fb1), __fmul_rn(A11, fb2)), D);
            nx = __fadd_rn(nx, dx); ny = __fadd_rn(ny, dy);
            outPt.x = __fadd_rn(nx, halfWin); outPt.y = __fadd_rn(ny, halfWin);
            if (__dadd_rn(__dmul_rn((double)dx, (double)dx), __dmul_rn((double)dy, (double)dy)) <= L.eps2) break;
            if (j > 0 && fabs((double)__fadd_rn(dx, pdx)) < 0.01 && fabs((double)__fadd_rn(dy, pdy)) < 0.01) {
                outPt.x = __fsub_rn(outPt.x, __fmul_rn(dx, 0.5f));
                outPt.y = __fsub_rn(outPt.y, __fmul_rn(dy, 0.5f));
                break;
            }
            pdx = dx; pdy = dy;
        }
        if (status && level == 0) {
            const int ix = cv_floor(__fsub_rn(outPt.x, halfWin)), iy = cv_floor(__fsub_rn(outPt.y, halfWin));
            if (ix < -WIN || ix >= LJ.w || iy < -WIN || iy >= LJ.h) status = 0;
        }
    }

    if (tid == 0) {
        job.nextPts[f] = outPt;
        job.status[f] = (uint8_t)status;
        if (job.trackStatus) {
            int ts = status ? 0 : 2;
            const float W = (float)PJ.lv[0].w, H = (float)PJ.lv[0].h;
            if (outPt.x < 0.0f || outPt.x >= W || outPt.y < 0.0f || outPt.y >= H) ts = 4;
            job.trackStatus[f] = ts;
        }
        if (L.done.hostFlag) {  // results may live in mapped host memory: make them visible, count, last one raises the flag
            __threadfence_system();
            hv_signal_done(L.done);
        }
    }
}

cudaError_t hv_launch_lk(const LkLaunch& L, int win, cudaStream_t stream)
{
    int maxN = 0;
    for (int i = 0; i < L.njobs; i++) maxN = max(maxN, L.jobs[i].n);
    if (maxN == 0) return cudaSuccess;
    // few features (one session): a CTA of 4 warps per feature minimises latency; many features: a warp per feature
    // maximises throughput. Both kernels produce identical bits (exact integer accumulation).
    long long total = 0;
    for (int i = 0; i < L.njobs; i++) total += L.jobs[i].n;
    if (hv_lk_uses_cta_kernel(total)) {          // the one predicate hv_lk_track's polling path relies on too (capi_internal.h)
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(maxN, L.njobs); cfg.blockDim = dim3(LKC_NW * 32); cfg.dynamicSmemBytes = 0; cfg.stream = stream;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[0].val.programmaticStreamSerializationAllowed = 1;
        static const bool pdl = getenv("HV_EKF_NO_PDL") == nullptr;       // one switch for every programmatic dependent launch of the library
        cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
        switch (win) {
            case 31: return cudaLaunchKernelEx(&cfg, hv_lk_cta_kernel<31>, L);
            case 21: return cudaLaunchKernelEx(&cfg, hv_lk_cta_kernel<21>, L);
            case 15: return cudaLaunchKernelEx(&cfg, hv_lk_cta_kernel<15>, L);
            case 11: return cudaLaunchKernelEx(&cfg, hv_lk_cta_kernel<11>, L);
            default: return cudaErrorInvalidValue;
        }
    }
    dim3 grid((maxN + LK_WARPS_PER_CTA - 1) / LK_WARPS_PER_CTA, L.njobs);
    dim3 block(LK_WARPS_PER_CTA * 32);
    switch (win) {
        case 31: hv_lk_kernel<31><<<grid, block, 0, stream>>>(L); break;
        case 21: hv_lk_kernel<21><<<grid, block, 0, stream>>>(L); break;
        case 15: hv_lk_kernel<15><<<grid, block, 0, stream>>>(L); break;
        case 11: hv_lk_kernel<11><<<grid, block, 0, stream>>>(L); break;
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}
