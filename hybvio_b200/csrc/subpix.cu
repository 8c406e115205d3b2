// hybvio_b200/csrc/subpix.cu -- sub-pixel corner refinement, cv::cornerSubPix (OCV/imgproc/src/cornersubpix.cpp), on the gray image that is
// already in HBM as pyramid level 0: the refinement the reference's SubPixelAdjuster runs on freshly detected corners (image.cpp:76-79).
//
// One warp (one CTA) per corner. Every iteration the lanes sample the (win_w + 2) x (win_h + 2) patch of cv::getRectSubPix(8U -> 32F)
// (OCV/imgproc/src/samplers.cpp: getRectSubPix_8u32f inside the image, getRectSubPix_Cn_ + adjustRect at the border) and the five
// per-tap double terms of the normal equations into shared memory -- elementwise, so in any order -- and lanes 0..4 then each run one
// of the five sums in OpenCV's row-major order. All lanes take the 2 x 2 step from the shuffled sums, so the stop tests are uniform.
// Every float and double operation is an explicitly rounded intrinsic (no FMA contraction) with OpenCV's casts: the result is
// bit-identical to oracle/hv_oracle_subpix.c, and with it to cv::cornerSubPix built without IPP. The mask (exp on the host) arrives
// with the arguments.
//
// hv_subpix_batch_kernel runs the same corner body for the points of up to HV_CORNER_BATCH_MAX lists (one per session, each on its own
// image) in one flattened grid: CTA g refines point g - first[j] of the job j with first[j] <= g < first[j + 1]. The window, criteria and
// mask are the batch's.
#include "hv_common.cuh"
#include <cfloat>

__device__ __forceinline__ double hv_dsub(double a, double b) { return __dadd_rn(a, -b); }

__host__ __device__ inline size_t hv_subpix_smem_bytes(int hw, int hh)
{
    const int taps = (2 * hw + 1) * (2 * hh + 1), patch = (2 * hw + 3) * (2 * hh + 3);
    return (size_t)5 * taps * sizeof(double) + (size_t)(patch + taps) * sizeof(float);
}

// cv::getRectSubPix(gray, Size(pw, ph), Point2f(cx, cy), patch, CV_32F), one element per lane and step
__device__ void hv_subpix_patch(const uint8_t* gray, int pitch, int w, int h, int pw, int ph, float cx, float cy, float* patch, int lane)
{
    const float x = __fsub_rn(cx, (float)(pw - 1) * 0.5f), y = __fsub_rn(cy, (float)(ph - 1) * 0.5f);
    const int ipx = __float2int_rd(x), ipy = __float2int_rd(y);
    if (0 <= ipx && ipx + pw < w && 0 <= ipy && ipy + ph < h) {
        // getRectSubPix_8u32f: the rectangle lies inside the image. Its running `prev` is the previous column's t scaled by s, so every
        // element can be formed on its own.
        float fa = __fsub_rn(x, (float)ipx);
        const float fb = __fsub_rn(y, (float)ipy);
        fa = fa < 0.0001f ? 0.0001f : fa;
        const float b1 = __fsub_rn(1.f, fb), b2 = fb, a12 = __fmul_rn(fa, b1), a22 = __fmul_rn(fa, fb);
        const double s = hv_dsub(1.0, (double)fa) / (double)fa;
        for (int e = lane; e < pw * ph; e += 32) {
            const int i = e / pw, j = e - i * pw;
            const uint8_t* r0 = gray + (size_t)(ipy + i) * pitch + ipx;
            const uint8_t* r1 = r0 + pitch;
            const float t = __fadd_rn(__fmul_rn(a12, (float)__ldg(r0 + j + 1)), __fmul_rn(a22, (float)__ldg(r1 + j + 1)));
            float prev;
            if (j == 0) {
                prev = __fmul_rn(__fsub_rn(1.f, fa), __fadd_rn(__fmul_rn(b1, (float)__ldg(r0)), __fmul_rn(b2, (float)__ldg(r1))));
            } else {
                const float tp = __fadd_rn(__fmul_rn(a12, (float)__ldg(r0 + j)), __fmul_rn(a22, (float)__ldg(r1 + j)));
                prev = (float)__dmul_rn((double)tp, s);
            }
            patch[e] = __fadd_rn(prev, t);
        }
        return;
    }
    // getRectSubPix_Cn_: rows and columns clamped into the image as adjustRect lays them out; columns left / right of the valid span
    // [rx, rw) take the two-tap blend of the edge column
    const float fa = __fsub_rn(x, (float)ipx), fb = __fsub_rn(y, (float)ipy), ia = __fsub_rn(1.f, fa), ib = __fsub_rn(1.f, fb);
    const float a11 = __fmul_rn(ia, ib), a12 = __fmul_rn(fa, ib), a21 = __fmul_rn(ia, fb), a22 = __fmul_rn(fa, fb), b1 = ib, b2 = fb;
    int col0 = ipx >= 0 ? ipx : 0, rx = ipx >= 0 ? 0 : (-ipx > pw ? pw : -ipx), rw;
    if (ipx < w - pw) rw = pw;
    else { rw = w - ipx - 1; if (rw < 0) { col0 += rw; rw = 0; } }
    int row0 = ipy >= 0 ? ipy : 0, ry = ipy >= 0 ? 0 : -ipy, rh;
    if (ipy < h - ph) rh = ph;
    else { rh = h - ipy - 1; if (rh < 0) { row0 += rh; rh = 0; } }
    for (int e = lane; e < pw * ph; e += 32) {
        const int i = e / pw, j = e - i * pw;
        // the source row advances after every patch row i with ry <= i < rh
        const int adv = (i < rh ? i : rh) - ry, row = row0 + (adv > 0 ? adv : 0), row2 = (i < ry || i >= rh) ? row : row + 1;
        const uint8_t* s1 = gray + (size_t)row * pitch + (col0 - rx);
        const uint8_t* s2 = gray + (size_t)row2 * pitch + (col0 - rx);
        float v;
        if (j >= rw) v = __fadd_rn(__fmul_rn((float)__ldg(s1 + rw), b1), __fmul_rn((float)__ldg(s2 + rw), b2));
        else if (j < rx) v = __fadd_rn(__fmul_rn((float)__ldg(s1 + rx), b1), __fmul_rn((float)__ldg(s2 + rx), b2));
        else v = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn((float)__ldg(s1 + j), a11), __fmul_rn((float)__ldg(s1 + j + 1), a12)),
                                     __fmul_rn((float)__ldg(s2 + j), a21)), __fmul_rn((float)__ldg(s2 + j + 1), a22));
        patch[e] = v;
    }
}

// the refined position of the corner *xy of the image (gray, pitch, w, h), with the window, criteria and mask of a, by one warp
__device__ __forceinline__ float2 hv_subpix_corner(const SubpixArgs& a, const uint8_t* gray, int pitch, int w, int h, const float2* xy)
{
    extern __shared__ __align__(16) unsigned char subpix_smem[];
    const int lane = threadIdx.x, hw = a.hw, hh = a.hh;
    const int ww = 2 * hw + 1, wh = 2 * hh + 1, taps = ww * wh, pw = ww + 2, ph = wh + 2;
    double* term = (double*)subpix_smem;                  // 5 x taps: gxx, gxy, gyy, gxx px + gxy py, gxy px + gyy py
    float* patch = (float*)(term + 5 * taps);             // ph x pw
    float* mask = patch + pw * ph;                        // wh x ww
    for (int k = lane; k < taps; k += 32) mask[k] = a.mask[k];
    const float2 cT = *xy;
    float cx = cT.x, cy = cT.y;
    // cv::cornerSubPix asserts a start inside the image (the host entry point checks it); the device entry point leaves such a point as it is
    if (cx >= 0.f && cx < (float)w && cy >= 0.f && cy < (float)h) {
        for (int iter = 0;;) {
            __syncwarp();
            hv_subpix_patch(gray, pitch, w, h, pw, ph, cx, cy, patch, lane);
            __syncwarp();
            for (int k = lane; k < taps; k += 32) {
                const int i = k / ww, j = k - i * ww;
                const float* sub = patch + (i + 1) * pw + (j + 1);
                const double tgx = (double)__fsub_rn(sub[1], sub[-1]), tgy = (double)__fsub_rn(sub[pw], sub[-pw]), m = (double)mask[k];
                const double gxx = __dmul_rn(__dmul_rn(tgx, tgx), m), gxy = __dmul_rn(__dmul_rn(tgx, tgy), m), gyy = __dmul_rn(__dmul_rn(tgy, tgy), m);
                const double px = (double)(j - hw), py = (double)(i - hh);
                term[k] = gxx; term[taps + k] = gxy; term[2 * taps + k] = gyy;
                term[3 * taps + k] = __dadd_rn(__dmul_rn(gxx, px), __dmul_rn(gxy, py));
                term[4 * taps + k] = __dadd_rn(__dmul_rn(gxy, px), __dmul_rn(gyy, py));
            }
            __syncwarp();
            double sum = 0.0;
            if (lane < 5) {
                const double* t = term + lane * taps;
#pragma unroll 8
                for (int k = 0; k < taps; k++) sum = __dadd_rn(sum, t[k]);
            }
            const double A = __shfl_sync(0xffffffffu, sum, 0), B = __shfl_sync(0xffffffffu, sum, 1), C = __shfl_sync(0xffffffffu, sum, 2);
            const double bb1 = __shfl_sync(0xffffffffu, sum, 3), bb2 = __shfl_sync(0xffffffffu, sum, 4);
            const double det = hv_dsub(__dmul_rn(A, C), __dmul_rn(B, B));
            if (fabs(det) <= DBL_EPSILON * DBL_EPSILON) break;
            const double scale = 1.0 / det;                                                 // IEEE division
            const float nx = (float)hv_dsub(__dadd_rn((double)cx, __dmul_rn(__dmul_rn(C, scale), bb1)), __dmul_rn(__dmul_rn(B, scale), bb2));
            const float ny = (float)__dadd_rn(hv_dsub((double)cy, __dmul_rn(__dmul_rn(B, scale), bb1)), __dmul_rn(__dmul_rn(A, scale), bb2));
            const float dx = __fsub_rn(nx, cx), dy = __fsub_rn(ny, cy);
            const float err = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));            // float, as OpenCV's Point2f arithmetic
            if (nx < 0.f || nx >= (float)w || ny < 0.f || ny >= (float)h) break;        // a step out of the image is not taken
            cx = nx; cy = ny;
            if (!(++iter < a.maxIters && (double)err > a.eps2)) break;
        }
        // moved more than the window: poor convergence, the start point stands
        if (fabsf(__fsub_rn(cx, cT.x)) > (float)hw || fabsf(__fsub_rn(cy, cT.y)) > (float)hh) { cx = cT.x; cy = cT.y; }
    }
    return make_float2(cx, cy);
}

__global__ void __launch_bounds__(32) hv_subpix_kernel(const __grid_constant__ SubpixArgs a)
{
    const float2 r = hv_subpix_corner(a, a.gray, a.pitch, a.w, a.h, a.xy + blockIdx.x);
    if (threadIdx.x == 0) {
        a.xy[blockIdx.x] = r;
        if (a.done.hostFlag) {
            __threadfence_system();
            hv_signal_done(a.done);
        }
    }
}

__global__ void __launch_bounds__(32) hv_subpix_batch_kernel(const __grid_constant__ SubpixBatchArgs b)
{
    const int g = blockIdx.x, j = hv_batch_job(b.first, g);
    const SubpixJob& J = b.job[j];
    float2* xy = J.xy + (g - b.first[j]);
    const float2 r = hv_subpix_corner(b.s, J.gray, J.pitch, J.w, J.h, xy);
    if (threadIdx.x == 0) *xy = r;
}

cudaError_t hv_launch_subpix(const SubpixArgs& a, cudaStream_t stream)
{
    if (a.n <= 0) return cudaSuccess;
    hv_subpix_kernel<<<a.n, 32, hv_subpix_smem_bytes(a.hw, a.hh), stream>>>(a);
    return cudaGetLastError();
}

cudaError_t hv_launch_subpix_batch(const SubpixBatchArgs& b, int njobs, cudaStream_t stream)
{
    const int ctas = b.first[njobs];
    if (ctas <= 0) return cudaSuccess;
    hv_subpix_batch_kernel<<<ctas, 32, hv_subpix_smem_bytes(b.s.hw, b.s.hh), stream>>>(b);
    return cudaGetLastError();
}
