// hybvio_b200/csrc/gftt.cu -- corner detection (SURVEY.md 8(f) N2) on the gray image that is already in HBM as pyramid level 0.
//
// Replaces, for tracker::FeatureDetector::detect on CPU images (src/tracker/feature_detector.cpp:566-682, the path
// FeatureDetector::build("GPU-GFTT") takes without OpenGL images), the device-side equivalent of
//   CpuCornerResponse::operator()       feature_detector.cpp:281-310  -> cv::cornerMinEigenVal(img, gfttBlockSize = 3, ksize 3)
//     cornerEigenValsVecs / calcMinEigenVal   OCV/imgproc/src/corner.cpp:238-320, 52-96   (Sobel 8U -> 32F with scale 1 / (4 * 3 * 255)
//                                             folded into the smoothing kernel, dx^2 / dx dy / dy^2, 3 x 3 box sum, min eigenvalue)
//   CollectMax::cpuImplementation       feature_detector.cpp:393-417  (best response of every bs x bs cell, GAIN 16, > gfttMinResponse)
// (the reference's own GPU version of exactly these two stages is the GLSL pipeline of feature_detector.cpp:31-470).
// The sort by response, the reference's resize quirk and applyMinDistance stay on the host (hybvio_b200/host/cuda_feature_detector.cpp):
// a few hundred key points.
//
// One CTA per cell (bs = 32: 23 x 15 = 345 CTAs for 752 x 480, 2.3 per SM). The CTA stages the (bs + 4)^2 gray pixels it needs
// (reflect-101 at the image border, exactly where cv::Sobel / cv::boxFilter reflect), forms dx, dy and the three products for the
// (bs + 2)^2 pixels around its cell in shared memory, then the 3 x 3 sums and the min eigenvalue of its bs x bs pixels, and reduces the
// arg max (first maximum in row-major order, as the reference's scan) with shuffles. fp32 in the reference's operation order, every
// operation an explicitly rounded intrinsic (no FMA contraction): the response is bit-identical to oracle/hv_oracle_gftt.c, which
// differs from the compiled reference only by the order of the box sum (running sums in OpenCV; <= 1e-9 absolute, tests/test_oracle_gftt.py).
// HBM traffic: the image is read once (each pixel by at most 4 cells through L2): w * h bytes in, 12 bytes per cell out.
//
// hv_gftt_batch_kernel runs the same cell body for the cells of up to HV_CORNER_BATCH_MAX images (one per session) in one flattened grid:
// CTA b belongs to the job j with first[j] <= b < first[j + 1] (a prefix sum of the cell counts, formed on the host; hv_batch_job).
#include "hv_common.cuh"

#define GFTT_NT 256
#define GFTT_MAX_CELL 32

// the key point of cell (cellX, cellY) of a grid cellsX cells wide, by one CTA of GFTT_NT threads
__device__ __forceinline__ void hv_gftt_cell(const GfttArgs& a, int cellX, int cellY, int cellsX)
{
    constexpr int R = GFTT_MAX_CELL + 4, C = GFTT_MAX_CELL + 2;
    __shared__ float g[R][R + 1];
    __shared__ float cxx[C][C + 1], cxy[C][C + 1], cyy[C][C + 1];
    __shared__ float s_val[GFTT_NT / 32];
    __shared__ int s_idx[GFTT_NT / 32];
    const int bs = a.cell, x0 = cellX * bs, y0 = cellY * bs, tid = threadIdx.x;
    const int rw = bs + 4, cw = bs + 2;
    // ---- gray region [x0 - 2, x0 + bs + 2) x [y0 - 2, y0 + bs + 2), reflected into the image
    for (int i = tid; i < rw * rw; i += GFTT_NT) {
        const int ly = i / rw, lx = i - ly * rw;
        const int gx = hv_reflect101(x0 - 2 + lx, a.w), gy = hv_reflect101(y0 - 2 + ly, a.h);
        g[ly][lx] = (float)__ldg(a.gray + (size_t)gy * a.pitch + gx);
    }
    __syncthreads();
    // ---- Sobel + products at the (bs + 2)^2 positions [x0 - 1, x0 + bs + 1) x ...: a position outside the image takes the values of
    // its reflection (cv::boxFilter reflects the covariance image), whose own 3 x 3 taps reflect again (cv::Sobel)
    for (int i = tid; i < cw * cw; i += GFTT_NT) {
        const int ly = i / cw, lx = i - ly * cw;
        const int gx = hv_reflect101(x0 - 1 + lx, a.w), gy = hv_reflect101(y0 - 1 + ly, a.h);
        const int xc = gx - (x0 - 2), xl = hv_reflect101(gx - 1, a.w) - (x0 - 2), xr = hv_reflect101(gx + 1, a.w) - (x0 - 2);
        const int yc = gy - (y0 - 2), yu = hv_reflect101(gy - 1, a.h) - (y0 - 2), yd = hv_reflect101(gy + 1, a.h) - (y0 - 2);
        // dx: row pass [-1 0 1] (exact), column pass [1 2 1] * scale:  d1 * k0 + (d0 + d2) * k1
        const float d0 = __fsub_rn(g[yu][xr], g[yu][xl]), d1 = __fsub_rn(g[yc][xr], g[yc][xl]), d2 = __fsub_rn(g[yd][xr], g[yd][xl]);
        const float dx = __fadd_rn(__fmul_rn(d1, a.k0), __fmul_rn(__fadd_rn(d0, d2), a.k1));
        // dy: row pass [1 2 1] * scale, column pass [-1 0 1]
        const float s0 = __fadd_rn(__fmul_rn(g[yu][xc], a.k0), __fmul_rn(__fadd_rn(g[yu][xl], g[yu][xr]), a.k1));
        const float s2 = __fadd_rn(__fmul_rn(g[yd][xc], a.k0), __fmul_rn(__fadd_rn(g[yd][xl], g[yd][xr]), a.k1));
        const float dy = __fsub_rn(s2, s0);
        cxx[ly][lx] = __fmul_rn(dx, dx); cxy[ly][lx] = __fmul_rn(dx, dy); cyy[ly][lx] = __fmul_rn(dy, dy);
    }
    __syncthreads();
    // ---- 3 x 3 sums, min eigenvalue, arg max of the cell (first maximum in row-major order)
    float best = -1e10f; int bidx = 0x7fffffff;
    for (int i = tid; i < bs * bs; i += GFTT_NT) {
        const int ly = i / bs, lx = i - ly * bs;
        if (x0 + lx >= a.w || y0 + ly >= a.h) continue;
        auto box = [&](float (*c)[C + 1]) {
            const float r0 = __fadd_rn(__fadd_rn(c[ly][lx], c[ly][lx + 1]), c[ly][lx + 2]);
            const float r1 = __fadd_rn(__fadd_rn(c[ly + 1][lx], c[ly + 1][lx + 1]), c[ly + 1][lx + 2]);
            const float r2 = __fadd_rn(__fadd_rn(c[ly + 2][lx], c[ly + 2][lx + 1]), c[ly + 2][lx + 2]);
            return __fadd_rn(__fadd_rn(r0, r1), r2);
        };
        const float A = __fmul_rn(box(cxx), 0.5f), Bq = box(cxy), Cq = __fmul_rn(box(cyy), 0.5f);
        const float t = __fsub_rn(A, Cq);
        const float resp = __fsub_rn(__fadd_rn(A, Cq), __fsqrt_rn(__fadd_rn(__fmul_rn(Bq, Bq), __fmul_rn(t, t))));
        const float r = __fmul_rn(resp, 16.0f);                        // CpuCornerResponse::GAIN
        if (r > a.minResponse && (r > best || (r == best && i < bidx))) { best = r; bidx = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bidx, o);
        if (ov > best || (ov == best && oi < bidx)) { best = ov; bidx = oi; }
    }
    if ((tid & 31) == 0) { s_val[tid >> 5] = best; s_idx[tid >> 5] = bidx; }
    __syncthreads();
    if (tid == 0) {
        for (int q = 1; q < GFTT_NT / 32; q++)
            if (s_val[q] > best || (s_val[q] == best && s_idx[q] < bidx)) { best = s_val[q]; bidx = s_idx[q]; }
        float* out = a.kp + 3 * ((size_t)cellY * cellsX + cellX);
        const bool found = best > -1e10f;
        out[0] = found ? (float)(x0 + bidx % bs) : 0.0f;               // the reference leaves (0, 0) when no pixel of the cell qualifies
        out[1] = found ? (float)(y0 + bidx / bs) : 0.0f;
        out[2] = best;
        if (a.done.hostFlag) {
            __threadfence_system();
            hv_signal_done(a.done);
        }
    }
}

__global__ void __launch_bounds__(GFTT_NT) hv_gftt_kernel(GfttArgs a)
{
    hv_gftt_cell(a, blockIdx.x, blockIdx.y, gridDim.x);
}

__global__ void __launch_bounds__(GFTT_NT) hv_gftt_batch_kernel(const __grid_constant__ GfttBatchArgs b)
{
    const int cta = blockIdx.x, j = hv_batch_job(b.first, cta);
    const int k = cta - b.first[j], cellsX = b.cellsX[j];
    hv_gftt_cell(b.job[j], k % cellsX, k / cellsX, cellsX);
}

cudaError_t hv_launch_gftt(const GfttArgs& a, cudaStream_t stream)
{
    const int cx = a.w / a.cell, cy = a.h / a.cell;                    // integer division, as the reference (feature_detector.cpp:395-396)
    if (cx <= 0 || cy <= 0) return cudaSuccess;
    hv_gftt_kernel<<<dim3(cx, cy), GFTT_NT, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t hv_launch_gftt_batch(const GfttBatchArgs& b, int njobs, cudaStream_t stream)
{
    const int ctas = b.first[njobs];
    if (ctas <= 0) return cudaSuccess;
    hv_gftt_batch_kernel<<<ctas, GFTT_NT, 0, stream>>>(b);
    return cudaGetLastError();
}
