// hybvio_b200/csrc/good_features.cu -- Shi-Tomasi corner detection, cv::goodFeaturesToTrack(img, corners, maxCorners, qualityLevel,
// minDistance, mask, 3, 3, useHarrisDetector = false) (OCV/imgproc/src/featureselect.cpp, CPU path), on the gray image that is already in
// HBM as pyramid level 0: the primitive of the reference's featureDetector = GFTT setting.
//
// Three launches on the context's stream:
//   hv_gf_response_kernel   one warp per 32 columns, one thread per column, sweeping the column from the top down. boxFilter on CV_32F
//                           keeps one running double sum per column (ColumnSum<double, float>), so a response depends on every row above
//                           it and a column is a sequential recurrence. Per row each lane forms the Sobel products of its own column (and
//                           the lanes at the warp's ends one more), takes its neighbours' by shuffle, row-sums them in double and steps
//                           the running sum; cornerMinEigenVal goes into the response map (scratch). The maximum over the mask's pixels is
//                           reduced per warp and atomicMax'ed, as order-preserving bits, into the job's word.
//   hv_gf_candidate_kernel  one CTA per 32 x 8 tile. Threshold (v > (float)(maxVal * qualityLevel)), 3 x 3 dilation and the candidate
//                           test on the interior [1, w - 1) x [1, h - 1); each candidate appends one 64-bit key with a warp-aggregated
//                           atomic. The key is ~(the response's order-preserving bits) above ~(the pixel index y w + x): ascending key order
//                           is greaterThanPtr's order (response descending, ties by descending address), whatever the append order. The
//                           CTAs also clear the job's min-distance grid.
//   hv_gf_select_kernel     one CTA of 1024 threads per job. In rounds of up to HV_GF_CHUNK keys: when more keys remain than a round
//                           holds, a radix select (8 passes of 8 bits over the remaining keys, shared-memory histograms) finds the
//                           HV_GF_CHUNK-th smallest; the keys up to it are gathered into shared memory and sorted bitonically. Each round
//                           then runs the greedy filter in list order, 1024 keys at a time: a key tests the corners kept before its
//                           group on a grid whose cells (side s, 2 (s - 1)^2 < minDistance^2) hold at most one kept corner each, then
//                           the group's own conflicts are resolved in order (ballot: the first live key is kept, later keys near it
//                           die), as gftt_select.cu does. It stops at maxCorners and pads [count, capacity) with HV_CORNER_NONE / 0.
// The job's max word and candidate count are zeroed on the stream before the first launch.
// The response follows OpenCV's operation order (Sobel 8U -> 32F: RowFilter's ((k0 S0 + k1 S1) + k2 S2) for the row pass and
// SymmColumnSmallFilter for the column pass; boxFilter's RowSum ((c[x - 1] + c[x]) + c[x + 1]) in double and its running ColumnSum), every
// fp32 and fp64 operation an explicitly rounded intrinsic: bit-identical to oracle/hv_oracle_good_features.c. It differs from hv_gftt_cell
// (gftt.cu), whose dy row pass and box sum are fp32 forms of their own, so the two share no code.
//
// The batch kernels run the same bodies for up to HV_CORNER_BATCH_MAX images (one per session) over one flattened grid each (CTA b belongs to
// the job j with firstStrip[j] <= b < firstStrip[j + 1], or firstTile[]; hv_batch_job), and the select kernel runs one CTA per job.
#include "hv_common.cuh"

#define GF_TW 32
#define GF_TH 8
#define GF_NT (GF_TW * GF_TH)
#define GF_SEL_NT 1024

// unsigned order of the result = float order of v (NaN aside)
__device__ __forceinline__ unsigned hv_gf_ordered(float v)
{
    const unsigned u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float hv_gf_unordered(unsigned o)
{
    return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o);
}

// The Sobel products (dx dx, dx dy, dy dy) at column cx of row r (both inside the image): the taps reflect-101 as cv::Sobel's do
__device__ __forceinline__ void hv_gf_products(const GoodFeaturesArgs& a, int cx, int r, float c[3])
{
    const float k1 = (float)(1.0 / 3060.0), k0 = 2.0f * k1;               // [1 2 1] * scale as the fp32 kernel Sobel builds
    const int xl = hv_reflect101(cx - 1, a.w), xr = hv_reflect101(cx + 1, a.w);
    const uint8_t* up = a.gray + (size_t)hv_reflect101(r - 1, a.h) * a.pitch;
    const uint8_t* mid = a.gray + (size_t)r * a.pitch;
    const uint8_t* dn = a.gray + (size_t)hv_reflect101(r + 1, a.h) * a.pitch;
    const float u0 = __ldg(up + xl), u1 = __ldg(up + cx), u2 = __ldg(up + xr);
    const float m0 = __ldg(mid + xl), m2 = __ldg(mid + xr);
    const float d0 = __ldg(dn + xl), d1 = __ldg(dn + cx), d2 = __ldg(dn + xr);
    // dx: row pass [-1 0 1] (exact), column pass [s 2s s] (SymmColumnSmallFilter: S1 k0 + (S0 + S2) k1)
    const float dx = __fadd_rn(__fmul_rn(__fsub_rn(m2, m0), k0), __fmul_rn(__fadd_rn(__fsub_rn(u2, u0), __fsub_rn(d2, d0)), k1));
    // dy: row pass [s 2s s] (RowFilter: ((k1 S0 + k0 S1) + k1 S2)), column pass [-1 0 1]
    const float s0 = __fadd_rn(__fadd_rn(__fmul_rn(k1, u0), __fmul_rn(k0, u1)), __fmul_rn(k1, u2));
    const float s2 = __fadd_rn(__fadd_rn(__fmul_rn(k1, d0), __fmul_rn(k0, d1)), __fmul_rn(k1, d2));
    const float dy = __fsub_rn(s2, s0);
    c[0] = __fmul_rn(dx, dx); c[1] = __fmul_rn(dx, dy); c[2] = __fmul_rn(dy, dy);
}

__device__ __forceinline__ float hv_gf_shfl_up(float v) { return __uint_as_float((unsigned)__shfl_up_sync(0xffffffffu, (int)__float_as_uint(v), 1)); }
__device__ __forceinline__ float hv_gf_shfl_down(float v) { return __uint_as_float((unsigned)__shfl_down_sync(0xffffffffu, (int)__float_as_uint(v), 1)); }

// RowSum<float, double> with ksize 3 at this lane's column x of row r: ((c[x - 1] + c[x]) + c[x + 1]) in double, columns reflect-101.
// A lane's own column is reflect101(x), so the lane right of column w - 1 holds column w - 2, the reflection of w; the lanes at the
// warp's ends form their outer neighbour themselves (lane 0 also covers x = -1, which reflects to column 1). Every lane of the warp calls it.
__device__ __forceinline__ void hv_gf_rowsum(const GoodFeaturesArgs& a, int x, int r, double R[3])
{
    const int lane = threadIdx.x & 31;
    float own[3], extra[3];
    hv_gf_products(a, hv_reflect101(x, a.w), r, own);
    hv_gf_products(a, hv_reflect101(lane == 0 ? x - 1 : x + 1, a.w), r, extra);
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const float up = hv_gf_shfl_up(own[k]), down = hv_gf_shfl_down(own[k]);
        const float left = lane == 0 ? extra[k] : up, right = lane == 31 ? extra[k] : down;
        R[k] = __dadd_rn(__dadd_rn((double)left, (double)own[k]), (double)right);
    }
}

// the response map and the masked maximum of columns [32 strip, 32 strip + 32) of job a, by one warp
__device__ __forceinline__ void hv_gf_response_strip(const GoodFeaturesArgs& a, int strip)
{
    const int x = strip * 32 + (threadIdx.x & 31);
    const bool mine = x < a.w;
    // ColumnSum<double, float>: SUM = (0 + R[-1]) + R[0]; per row s0 = SUM + R[y + 1], out = (float)s0, SUM = s0 - R[y - 1]
    double Rm[3], R0[3], Rn[3], sum[3];
    hv_gf_rowsum(a, x, hv_reflect101(-1, a.h), Rm);
    hv_gf_rowsum(a, x, 0, R0);
#pragma unroll
    for (int k = 0; k < 3; k++) sum[k] = __dadd_rn(__dadd_rn(0.0, Rm[k]), R0[k]);
    unsigned best = 0u;
    for (int y = 0; y < a.h; y++) {
        hv_gf_rowsum(a, x, hv_reflect101(y + 1, a.h), Rn);
        float box[3];
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const double s0 = __dadd_rn(sum[k], Rn[k]);
            box[k] = __double2float_rn(s0);
            sum[k] = __dsub_rn(s0, Rm[k]);
            Rm[k] = R0[k];
            R0[k] = Rn[k];
        }
        if (mine) {
            const float A = __fmul_rn(box[0], 0.5f), B = box[1], C = __fmul_rn(box[2], 0.5f);
            const float t = __fsub_rn(A, C);
            const float e = __fsub_rn(__fadd_rn(A, C), __fsqrt_rn(__fadd_rn(__fmul_rn(t, t), __fmul_rn(B, B))));
            a.eig[(size_t)y * a.w + x] = e;
            if (!a.mask || __ldg(a.mask + (size_t)y * a.maskPitch + x)) best = max(best, hv_gf_ordered(e));
        }
    }
    best = __reduce_max_sync(0xffffffffu, best);
    if ((threadIdx.x & 31) == 0 && best) atomicMax(a.maxWord, best);
}

// the candidates of tile (tx, ty) of job a, appended to a.keys; CTA `cta` of `ctas` also clears its share of the grid
__device__ __forceinline__ void hv_gf_candidate_tile(const GoodFeaturesArgs& a, int tx, int ty, int cta, int ctas)
{
    if (a.useGrid)
        for (long long i = (long long)cta * GF_NT + threadIdx.x; i < (long long)a.gridW * a.gridH; i += (long long)ctas * GF_NT) a.grid[i] = -1;
    const int tid = threadIdx.x, x = tx * GF_TW + tid % GF_TW, y = ty * GF_TH + tid / GF_TW;
    const unsigned mw = *a.maxWord;
    const float maxVal = mw ? hv_gf_unordered(mw) : 0.0f;
    const float thresh = __double2float_rn(__dmul_rn((double)maxVal, a.quality));      // threshold(eig, eig, maxVal * q, 0, TOZERO)
    bool cand = false;
    float v = 0.0f;
    if (x >= 1 && x < a.w - 1 && y >= 1 && y < a.h - 1 && (!a.mask || __ldg(a.mask + (size_t)y * a.maskPitch + x))) {
        const float* e = a.eig + (size_t)y * a.w + x;
        v = __ldg(e);
        v = v > thresh ? v : 0.0f;
        if (v != 0.0f) {
            float m = v;                                                 // dilate(eig, tmp, 3 x 3)
#pragma unroll
            for (int dy = -1; dy <= 1; dy++)
#pragma unroll
                for (int dx = -1; dx <= 1; dx++) {
                    float u = __ldg(e + dy * a.w + dx);
                    u = u > thresh ? u : 0.0f;
                    m = u > m ? u : m;
                }
            cand = v == m;
        }
    }
    const unsigned b = __ballot_sync(0xffffffffu, cand);
    if (!b) return;
    const int lane = tid & 31;
    int base = 0;
    if (lane == 0) base = atomicAdd(a.nCand, __popc(b));
    base = __shfl_sync(0xffffffffu, base, 0);
    const int slot = base + __popc(b & ((1u << lane) - 1u));
    if (cand && slot < a.maxCand)
        a.keys[slot] =
            ((unsigned long long)~hv_gf_ordered(v) << 32) | (unsigned)~(unsigned)(y * a.w + x);
}

// does a corner kept before the current group lie within minDistance of (x, y)?
__device__ __forceinline__ bool hv_gf_near_grid(const GoodFeaturesArgs& a, int x, int y)
{
    const int cx0 = max(x - a.reach, 0) / a.cell, cx1 = min(x + a.reach, a.w - 1) / a.cell;
    const int cy0 = max(y - a.reach, 0) / a.cell, cy1 = min(y + a.reach, a.h - 1) / a.cell;
    for (int cy = cy0; cy <= cy1; cy++)
        for (int cx = cx0; cx <= cx1; cx++) {
            const int k = a.grid[(size_t)cy * a.gridW + cx];
            if (k < 0) continue;
            const int ky = k / a.w, kx = k - ky * a.w;
            const float ddx = __fsub_rn((float)x, (float)kx), ddy = __fsub_rn((float)y, (float)ky);
            if ((double)__fadd_rn(__fmul_rn(ddx, ddx), __fmul_rn(ddy, ddy)) < a.md2) return true;
        }
    return false;
}

__device__ __forceinline__ bool hv_gf_near(const GoodFeaturesArgs& a, int x, int y, int k)
{
    const int ky = k / a.w, kx = k - ky * a.w;
    const float ddx = __fsub_rn((float)x, (float)kx), ddy = __fsub_rn((float)y, (float)ky);
    return (double)__fadd_rn(__fmul_rn(ddx, ddx), __fmul_rn(ddy, ddy)) < a.md2;
}

// the list of job a, by one CTA of GF_SEL_NT threads with HV_GF_CHUNK keys of dynamic shared memory
__device__ __forceinline__ void hv_gf_select_list(const GoodFeaturesArgs& a)
{
    extern __shared__ __align__(16) unsigned char gf_smem[];
    unsigned long long* key = (unsigned long long*)gf_smem;
    __shared__ unsigned hist[256];
    __shared__ unsigned s_live[GF_SEL_NT / 32];
    __shared__ unsigned long long s_prefix;
    __shared__ int s_need, s_fill, s_kept;
    const int tid = threadIdx.x, lane = tid & 31;
    const int n = min(*a.nCand, a.maxCand);
    const unsigned long long* K = a.keys;
    unsigned long long lo = 0ull;                      // every key is > 0; the keys <= lo have been consumed
    int remaining = n, kept = 0;
    while (remaining > 0 && kept < a.maxCorners) {
        unsigned long long hi = ~0ull;                 // no key is ~0: its response bits would be a NaN's
        int take = remaining;
        if (remaining > HV_GF_CHUNK) {
            // radix select: hi = the HV_GF_CHUNK-th smallest key above lo (keys are unique)
            unsigned long long prefix = 0ull;
            int need = HV_GF_CHUNK;
            for (int shift = 56; shift >= 0; shift -= 8) {
                if (tid < 256) hist[tid] = 0u;
                __syncthreads();
                const unsigned long long himask = shift == 56 ? 0ull : ~0ull << (shift + 8);
                for (int i = tid; i < n; i += GF_SEL_NT) {
                    const unsigned long long k = K[i];
                    if (k > lo && ((k ^ prefix) & himask) == 0ull) atomicAdd(&hist[(unsigned)(k >> shift) & 255u], 1u);
                }
                __syncthreads();
                if (tid < 32) {
                    unsigned c[8], sum = 0u;
#pragma unroll
                    for (int j = 0; j < 8; j++) { c[j] = hist[8 * lane + j]; sum += c[j]; }
                    unsigned incl = sum;
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
                        const unsigned t = (unsigned)__shfl_up_sync(0xffffffffu, (int)incl, o);
                        if (lane >= o) incl += t;
                    }
                    unsigned before = incl - sum;
                    if (before < (unsigned)need && (unsigned)need <= incl) {
                        int j = 0;
                        while (before + c[j] < (unsigned)need) before += c[j++];
                        s_prefix = prefix | ((unsigned long long)(8 * lane + j) << shift);
                        s_need = need - (int)before;
                    }
                }
                __syncthreads();
                prefix = s_prefix;
                need = s_need;
            }
            hi = prefix;
            take = HV_GF_CHUNK;
        }
        // gather the keys in (lo, hi] and sort them
        int P = 2;
        while (P < take) P <<= 1;
        for (int i = tid; i < P; i += GF_SEL_NT) key[i] = ~0ull;
        if (tid == 0) s_fill = 0;
        __syncthreads();
        for (int i = tid; i < n; i += GF_SEL_NT) {
            const unsigned long long k = K[i];
            if (k > lo && k <= hi) {
                const int slot = atomicAdd(&s_fill, 1);
                if (slot < P) key[slot] = k;
            }
        }
        __syncthreads();
        for (int kk = 2; kk <= P; kk <<= 1)
            for (int j = kk >> 1; j > 0; j >>= 1) {
                for (int t = tid; t < P / 2; t += GF_SEL_NT) {
                    const int l = 2 * t - (t & (j - 1)), r = l + j;
                    const unsigned long long u = key[l], w = key[r];
                    if ((u > w) == ((l & kk) == 0)) { key[l] = w; key[r] = u; }
                }
                __syncthreads();
            }
        // the greedy filter in list order, GF_SEL_NT keys at a time
        for (int c0 = 0; c0 < take && kept < a.maxCorners; c0 += GF_SEL_NT) {
            const int i = c0 + tid;
            const bool has = i < take;
            const unsigned long long k = has ? key[i] : 0ull;
            const int idx = (int)~(unsigned)k, y = has ? idx / a.w : 0, x = has ? idx - y * a.w : 0;
            const float v = hv_gf_unordered(~(unsigned)(k >> 32));
            if (!a.useGrid) {                                            // minDistance < 1: every candidate in order
                const int slot = kept + tid;
                if (has && slot < a.maxCorners) {
                    a.xy[slot] = make_float2((float)x, (float)y);
                    if (a.response) a.response[slot] = v;
                }
                kept = min(a.maxCorners, kept + min(GF_SEL_NT, take - c0));
                continue;
            }
            bool alive = has && !hv_gf_near_grid(a, x, y);
            for (;;) {
                const unsigned b = __ballot_sync(0xffffffffu, alive);
                if (lane == 0) s_live[tid >> 5] = b;
                __syncthreads();
                int first = -1;
                for (int w = 0; w < GF_SEL_NT / 32; w++)
                    if (s_live[w]) { first = 32 * w + __ffs(s_live[w]) - 1; break; }
                if (first < 0) break;
                if (tid == first) {
                    a.grid[(size_t)(y / a.cell) * a.gridW + x / a.cell] = idx;
                    a.xy[kept] = make_float2((float)x, (float)y);
                    if (a.response) a.response[kept] = v;
                    s_kept = idx;
                    alive = false;
                }
                __syncthreads();
                const int q = s_kept;
                kept++;
                if (alive && hv_gf_near(a, x, y, q)) alive = false;
                if (kept >= a.maxCorners) break;
            }
            __syncthreads();                                             // s_live is rewritten by the next group
        }
        __syncthreads();                                                 // key[] is rewritten by the next round
        lo = hi;
        remaining -= take;
    }
    for (int i = kept + tid; i < a.capacity; i += GF_SEL_NT) {
        a.xy[i] = make_float2(HV_CORNER_NONE_F, HV_CORNER_NONE_F);
        if (a.response) a.response[i] = 0.0f;
    }
    if (tid == 0) *a.count = kept;
}

__global__ void __launch_bounds__(32) hv_gf_response_kernel(GoodFeaturesArgs a)
{
    hv_gf_response_strip(a, blockIdx.x);
}

__global__ void __launch_bounds__(GF_NT) hv_gf_candidate_kernel(GoodFeaturesArgs a)
{
    hv_gf_candidate_tile(a, blockIdx.x, blockIdx.y, blockIdx.y * gridDim.x + blockIdx.x, gridDim.x * gridDim.y);
}

__global__ void __launch_bounds__(GF_SEL_NT, 1) hv_gf_select_kernel(const __grid_constant__ GoodFeaturesArgs a)
{
    hv_gf_select_list(a);
}

__global__ void __launch_bounds__(32) hv_gf_response_batch_kernel(const __grid_constant__ GoodFeaturesBatchArgs b)
{
    const int cta = blockIdx.x, j = hv_batch_job(b.firstStrip, cta);
    hv_gf_response_strip(b.job[j], cta - b.firstStrip[j]);
}

__global__ void __launch_bounds__(GF_NT) hv_gf_candidate_batch_kernel(const __grid_constant__ GoodFeaturesBatchArgs b)
{
    const int cta = blockIdx.x, j = hv_batch_job(b.firstTile, cta);
    const GoodFeaturesArgs& a = b.job[j];
    const int k = cta - b.firstTile[j];
    hv_gf_candidate_tile(a, k % a.tilesX, k / a.tilesX, k, a.tilesX * a.tilesY);
}

__global__ void __launch_bounds__(GF_SEL_NT, 1) hv_gf_select_batch_kernel(const __grid_constant__ GoodFeaturesBatchArgs b)
{
    hv_gf_select_list(b.job[blockIdx.x]);
}

#include "hv_device_once.cuh"

static bool g_gf_attr_set[64], g_gf_batch_attr_set[64];
static const int GF_SMEM = HV_GF_CHUNK * (int)sizeof(unsigned long long);

cudaError_t hv_launch_good_features(const GoodFeaturesArgs& a, cudaStream_t stream)
{
    if (hv_first_use_on_device(g_gf_attr_set)) {
        cudaError_t e = cudaFuncSetAttribute(hv_gf_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, GF_SMEM);
        if (e != cudaSuccess) return e;
    }
    hv_gf_response_kernel<<<(a.w + 31) / 32, 32, 0, stream>>>(a);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    hv_gf_candidate_kernel<<<dim3(a.tilesX, a.tilesY), GF_NT, 0, stream>>>(a);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    hv_gf_select_kernel<<<1, GF_SEL_NT, GF_SMEM, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t hv_launch_good_features_batch(const GoodFeaturesBatchArgs& b, int njobs, cudaStream_t stream)
{
    if (hv_first_use_on_device(g_gf_batch_attr_set)) {
        cudaError_t e = cudaFuncSetAttribute(hv_gf_select_batch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, GF_SMEM);
        if (e != cudaSuccess) return e;
    }
    hv_gf_response_batch_kernel<<<b.firstStrip[njobs], 32, 0, stream>>>(b);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    hv_gf_candidate_batch_kernel<<<b.firstTile[njobs], GF_NT, 0, stream>>>(b);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    hv_gf_select_batch_kernel<<<njobs, GF_SEL_NT, GF_SMEM, stream>>>(b);
    return cudaGetLastError();
}
