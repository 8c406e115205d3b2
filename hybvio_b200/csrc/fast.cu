// hybvio_b200/csrc/fast.cu -- FAST corner detection, cv::FAST with FastFeatureDetector::TYPE_9_16 (OCV/features2d/src/fast.cpp: FAST_t<16>;
// fast_score.cpp: cornerScore<16>), on the gray image that is already in HBM as pyramid level 0: the detector the reference's
// FeatureDetector::build hands out for featureDetector = FAST (src/tracker/feature_detector_legacy.cpp).
//
// Two launches on the context's stream:
//   hv_fast_mark_kernel     one CTA per 32 x 8 tile. The CTA stages the tile's gray pixels with a 4-pixel apron, runs the segment test
//                           (and, with suppression, the score) for the tile plus a one-pixel ring in shared memory, suppresses, and writes
//                           one 32-bit keypoint mask per (row, tile) -- a warp ballot, bit b = column 32 tx + b -- and its tile's count.
//   hv_fast_scatter_kernel  one CTA per band of 8 rows (a row of tiles). Its first output slot is the sum of the counts of every tile above
//                           the band; a block scan over the band's masks in (row, tile) order then gives each keypoint its slot, so the list
//                           comes out in OpenCV's order (rows top to bottom, columns left to right). The response of a kept keypoint is its
//                           score, recomputed from the image; slots [count, capacity) get HV_CORNER_NONE and response 0.
// Every operation is on integers, so the list equals oracle/hv_oracle_fast.c bit for bit by construction.
//
// The batch kernels run the same tile and band bodies for up to HV_CORNER_BATCH_MAX images (one per session) in one flattened grid each:
// CTA b belongs to the job j with first[j] <= b < first[j + 1] (prefix sums of the tile and band counts, formed on the host; hv_batch_job).
#include "hv_common.cuh"

// makeOffsets(pixel, step, 16): the circle as (dx, dy)
__constant__ signed char c_fast_circle[16][2] = {{0, 3}, {1, 3}, {2, 2}, {3, 1}, {3, 0}, {3, -1}, {2, -2}, {1, -3},
                                                  {0, -3}, {-1, -3}, {-2, -2}, {-3, -1}, {-3, 0}, {-3, 1}, {-2, 2}, {-1, 3}};

// FAST_t<16>'s segment test and cornerScore<16> at *p (rows `stride` bytes apart): -1 when 9 contiguous circle pixels are neither all
// darker than v - t nor all brighter than v + t; otherwise the score (withScore) or 0.
__device__ __forceinline__ int hv_fast_pixel(const uint8_t* p, int stride, int t, bool withScore)
{
    const int v = p[0];
    int d[16];
    unsigned dark = 0u, bright = 0u;
#pragma unroll
    for (int k = 0; k < 16; k++) {
        const int q = p[c_fast_circle[k][1] * stride + c_fast_circle[k][0]];
        d[k] = v - q;
        dark |= (unsigned)(q < v - t) << k;
        bright |= (unsigned)(q > v + t) << k;
    }
    // a run of 9 on the circle: bit k of the result is set when bits k .. k + 8 (mod 16) are
    auto run9 = [](unsigned m) {
        m |= m << 16;
        unsigned r = m;
#pragma unroll
        for (int i = 1; i < 9; i++) r &= m >> i;
        return r & 0xffffu;
    };
    if (!run9(dark) && !run9(bright)) return -1;
    if (!withScore) return 0;
    // cornerScore<16>: max(t, the best arc's min(v - q), the best arc's min(q - v)) - 1 over the 16 arcs of 9 (the scalar code's pruned
    // loops visit the same arcs)
    int a0 = t, b0 = 255;
#pragma unroll
    for (int k = 0; k < 16; k++) {
        int mn = d[k], mx = d[k];
#pragma unroll
        for (int i = 1; i < 9; i++) { mn = min(mn, d[(k + i) & 15]); mx = max(mx, d[(k + i) & 15]); }
        a0 = max(a0, mn);
        b0 = min(b0, mx);
    }
    return max(a0, -b0) - 1;
}

#define FAST_TW 32                  // tile width: one warp per tile row, so a ballot is the row's mask
#define FAST_TH 8
#define FAST_NT (FAST_TW * FAST_TH)

// the masks and the count of tile (tx, ty) of job a
__device__ __forceinline__ void hv_fast_tile(const FastArgs& a, int tx, int ty)
{
    __shared__ uint8_t g[FAST_TH + 8][FAST_TW + 8];
    __shared__ int sc[FAST_TH + 2][FAST_TW + 2];        // -1: no corner (or outside [3, w - 3) x [3, h - 3)); else the score (or 0)
    __shared__ int warpCount[FAST_TH];
    const int tid = threadIdx.x, x0 = tx * FAST_TW, y0 = ty * FAST_TH;
    for (int i = tid; i < (FAST_TH + 8) * (FAST_TW + 8); i += FAST_NT) {
        const int ly = i / (FAST_TW + 8), lx = i - ly * (FAST_TW + 8), X = x0 - 4 + lx, Y = y0 - 4 + ly;
        g[ly][lx] = (X >= 0 && X < a.w && Y >= 0 && Y < a.h) ? __ldg(a.gray + (size_t)Y * a.pitch + X) : 0;
    }
    __syncthreads();
    for (int i = tid; i < (FAST_TH + 2) * (FAST_TW + 2); i += FAST_NT) {
        const int ly = i / (FAST_TW + 2), lx = i - ly * (FAST_TW + 2), X = x0 - 1 + lx, Y = y0 - 1 + ly;
        int s = -1;
        if (X >= 3 && X < a.w - 3 && Y >= 3 && Y < a.h - 3) s = hv_fast_pixel(&g[ly + 3][lx + 3], FAST_TW + 8, a.threshold, a.nonmax);
        sc[ly][lx] = s;
    }
    __syncthreads();
    const int lx = tid % FAST_TW, ly = tid / FAST_TW;
    const int s = sc[ly + 1][lx + 1];
    bool kp = s >= 0;
    if (kp && a.nonmax) {
        // FAST_t's 3 x 3 test: strictly above every neighbour, a neighbour without a corner counting as score 0
#pragma unroll
        for (int dy = 0; dy < 3; dy++)
#pragma unroll
            for (int dx = 0; dx < 3; dx++)
                if ((dx != 1 || dy != 1) && s <= max(sc[ly + dy][lx + dx], 0)) kp = false;
    }
    const unsigned word = __ballot_sync(0xffffffffu, kp);
    if (lx == 0) {
        a.mask[(size_t)(y0 + ly) * a.tilesX + tx] = word;
        warpCount[ly] = __popc(word);
    }
    __syncthreads();
    if (tid == 0) {
        int n = 0;
        for (int r = 0; r < FAST_TH; r++) n += warpCount[r];
        a.tileCount[(size_t)ty * a.tilesX + tx] = n;
    }
}

// exclusive scan of v over the CTA; *total = the sum
__device__ __forceinline__ int hv_fast_block_scan(int v, int* buf, int* total)
{
    const int tid = threadIdx.x;
    buf[tid] = v;
    __syncthreads();
    for (int o = 1; o < FAST_NT; o <<= 1) {
        const int add = tid >= o ? buf[tid - o] : 0;
        __syncthreads();
        buf[tid] += add;
        __syncthreads();
    }
    const int incl = buf[tid];
    *total = buf[FAST_NT - 1];
    __syncthreads();
    return incl - v;
}

// the keypoints of band ty (rows [8 ty, 8 ty + 8)) of job a into their slots; CTA `cta` of `ctas` also writes its share of the padding
__device__ __forceinline__ void hv_fast_band(const FastArgs& a, int ty, int cta, int ctas)
{
    __shared__ int buf[FAST_NT];
    const int tid = threadIdx.x, tiles = a.tilesX * a.tilesY, above = ty * a.tilesX;
    int all = 0, before = 0;
    for (int i = tid; i < tiles; i += FAST_NT) {
        const int c = a.tileCount[i];
        all += c;
        before += i < above ? c : 0;
    }
    int sumAll, base;
    hv_fast_block_scan(all, buf, &sumAll);
    hv_fast_block_scan(before, buf, &base);
    const int words = FAST_TH * a.tilesX;
    const unsigned* mask = a.mask + (size_t)ty * words;
    for (int c0 = 0; c0 < words; c0 += FAST_NT) {
        const int k = c0 + tid;
        unsigned word = k < words ? mask[k] : 0u;
        int chunk;
        int slot = base + hv_fast_block_scan(__popc(word), buf, &chunk);
        const int x0 = (k % a.tilesX) * FAST_TW, y = ty * FAST_TH + k / a.tilesX;
        while (word) {
            const int b = __ffs(word) - 1;
            word &= word - 1u;
            if (slot < a.capacity) {
                a.xy[slot] = make_float2((float)(x0 + b), (float)y);
                if (a.response) {
                    const int s = a.nonmax ? hv_fast_pixel(a.gray + (size_t)y * a.pitch + x0 + b, a.pitch, a.threshold, true) : 0;
                    a.response[slot] = (float)s;
                }
            }
            slot++;
        }
        base += chunk;
    }
    for (int i = sumAll + cta * FAST_NT + tid; i < a.capacity; i += ctas * FAST_NT) {
        a.xy[i] = make_float2(HV_CORNER_NONE_F, HV_CORNER_NONE_F);
        if (a.response) a.response[i] = 0.f;
    }
    if (cta == 0 && tid == 0) *a.count = sumAll;
}

__global__ void __launch_bounds__(FAST_NT) hv_fast_mark_kernel(FastArgs a)
{
    hv_fast_tile(a, blockIdx.x, blockIdx.y);
}

__global__ void __launch_bounds__(FAST_NT) hv_fast_scatter_kernel(FastArgs a)
{
    hv_fast_band(a, blockIdx.x, blockIdx.x, gridDim.x);
}

__global__ void __launch_bounds__(FAST_NT) hv_fast_mark_batch_kernel(const __grid_constant__ FastBatchArgs b)
{
    const int cta = blockIdx.x, j = hv_batch_job(b.firstTile, cta);
    const FastArgs& a = b.job[j];
    const int k = cta - b.firstTile[j];
    hv_fast_tile(a, k % a.tilesX, k / a.tilesX);
}

__global__ void __launch_bounds__(FAST_NT) hv_fast_scatter_batch_kernel(const __grid_constant__ FastBatchArgs b)
{
    const int cta = blockIdx.x, j = hv_batch_job(b.firstBand, cta);
    const FastArgs& a = b.job[j];
    const int k = cta - b.firstBand[j];
    hv_fast_band(a, k, k, a.tilesY);
}

cudaError_t hv_launch_fast(const FastArgs& a, cudaStream_t stream)
{
    hv_fast_mark_kernel<<<dim3(a.tilesX, a.tilesY), FAST_NT, 0, stream>>>(a);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    hv_fast_scatter_kernel<<<a.tilesY, FAST_NT, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t hv_launch_fast_batch(const FastBatchArgs& b, int njobs, cudaStream_t stream)
{
    hv_fast_mark_batch_kernel<<<b.firstTile[njobs], FAST_NT, 0, stream>>>(b);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    hv_fast_scatter_batch_kernel<<<b.firstBand[njobs], FAST_NT, 0, stream>>>(b);
    return cudaGetLastError();
}
