// hybvio_b200/csrc/gftt_select.cu -- corner selection (SURVEY.md 8(f) N2): the tail of tracker::FeatureDetector::detect after CollectMax
// (src/tracker/feature_detector.cpp:625-638) on the key points hv_gftt_kernel left in HBM, so that the new corners can go on to
// cv::cornerSubPix (subpix.cu) and the stereo LK call without a host round trip:
//   std::stable_sort by response, descending                     feature_detector.cpp:625-630
//   corners.clear(); corners.resize(n); push_back(...)           feature_detector.cpp:631-634 (n points at (0, 0) in front: a quirk kept)
//   applyMinDistance(corners, prevCorners, maskRadius)            feature_detector.cpp:636-637, src/tracker/feature_detector_legacy.cpp
// Bit-identical to orc_gftt_corners (oracle/hv_oracle_gftt.c), the restatement the golden lists of the compiled reference pin.
//
// One CTA of 1024 threads.
//  * Sort: a unique 64-bit key per key point, the response's orderable bits (inverted: descending) above the cell index, so an ascending
//    bitonic sort of the keys in shared memory is the stable sort. -0.0 is canonicalised first: the reference's `<` finds it equal to +0.0.
//  * The n quirk points at (0, 0): the first is kept iff no previous corner lies within the radius; every later one lies at distance
//    0 < r^2 of it (r >= 1), so the block contributes at most that one point.
//  * Greedy filter, in list order, chunks of 1024 sorted points, one per thread: each tests its point against the previous corners and
//    against the points kept so far (in parallel); conflicts inside the chunk are then resolved in order -- the first point still alive
//    is kept (ballot), every later live point within the radius of it dies -- until the chunk is exhausted or max_tracks points are kept.
//    The kept points are a subsequence of the sorted list, so they are compacted into the front of the same shared array.
//  * Distance test as the reference writes it, (c.x - p.x)^2 + (c.y - p.y)^2 < (float)(r * r) with c the other point, in fp32 with every
//    operation an explicitly rounded intrinsic (no FMA contraction).
// NaN responses (which the detector never produces) are outside the contract: the reference's insertion order around them is not a sort.
//
// hv_gftt_select_batch_kernel runs the same list body for up to HV_CORNER_BATCH_MAX lists (one per session): CTA j is list j.
#include "hv_common.cuh"

#define SEL_NT 1024

// ascending order of the keys = descending response, ties in cell order
__device__ __forceinline__ unsigned long long hv_select_key(float r, int i)
{
    unsigned u = __float_as_uint(r == 0.0f ? 0.0f : r);
    u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);                  // unsigned order of u = float order of r
    return ((unsigned long long)~u << 32) | (unsigned)i;
}

// applyMinDistance's test of point (cx, cy) against an earlier point (ox, oy)
__device__ __forceinline__ bool hv_select_near(float ox, float oy, float cx, float cy, float r2)
{
    const float dx = __fsub_rn(ox, cx), dy = __fsub_rn(oy, cy);
    return __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)) < r2;
}

// list a, by one CTA of SEL_NT threads
__device__ __forceinline__ void hv_gftt_select_list(const GfttSelectArgs& a)
{
    extern __shared__ __align__(16) unsigned char select_smem[];
    unsigned long long* key = (unsigned long long*)select_smem;       // pow2 sort keys; afterwards slot k holds sorted point k ...
    float2* pt = (float2*)select_smem;                                 // ... and, in the greedy phase, kept point k
    __shared__ unsigned s_live[SEL_NT / 32];
    const int tid = threadIdx.x, n = a.nkp, P = a.pow2;

    for (int i = tid; i < P; i += SEL_NT) key[i] = i < n ? hv_select_key(__ldg(a.kp + 3 * i + 2), i) : ~0ull;
    __syncthreads();
    for (int k = 2; k <= P; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int t = tid; t < P / 2; t += SEL_NT) {
                const int lo = 2 * t - (t & (j - 1)), hi = lo + j;
                const unsigned long long x = key[lo], y = key[hi];
                if ((x > y) == ((lo & k) == 0)) { key[lo] = y; key[hi] = x; }
            }
            __syncthreads();
        }
    for (int i = tid; i < n; i += SEL_NT) {                           // every thread rewrites only the slots it reads
        const int c = (int)(unsigned)key[i];
        pt[i] = make_float2(__ldg(a.kp + 3 * c), __ldg(a.kp + 3 * c + 1));
    }
    __syncthreads();

    int count, zero = 0, kept = 0;
    if (a.maskRadius <= 0) {
        count = 2 * n;                                                 // no filter, no cap
        zero = n;
    } else {
        const float r2 = a.r2;
        int near0 = 0;
        for (int k = tid; k < a.nprev; k += SEL_NT) near0 |= hv_select_near(__ldg(a.prev + 2 * k), __ldg(a.prev + 2 * k + 1), 0.f, 0.f, r2);
        zero = (n > 0 && !__syncthreads_or(near0)) ? 1 : 0;
        bool full = zero >= a.maxTracks;
        for (int c0 = 0; c0 < n && !full; c0 += SEL_NT) {
            const int i = c0 + tid;
            const float2 me = i < n ? pt[i] : make_float2(0.f, 0.f);    // slots >= c0 are not written before the first barrier below
            bool alive = i < n;
            if (alive && zero) alive = !hv_select_near(0.f, 0.f, me.x, me.y, r2);
            for (int k = 0; alive && k < kept; k++) alive = !hv_select_near(pt[k].x, pt[k].y, me.x, me.y, r2);
            for (int k = 0; alive && k < a.nprev; k++) alive = !hv_select_near(__ldg(a.prev + 2 * k), __ldg(a.prev + 2 * k + 1), me.x, me.y, r2);
            for (;;) {
                const unsigned b = __ballot_sync(0xffffffffu, alive);
                if ((tid & 31) == 0) s_live[tid >> 5] = b;
                __syncthreads();
                int first = -1;
                for (int w = 0; w < SEL_NT / 32; w++)
                    if (s_live[w]) { first = 32 * w + __ffs(s_live[w]) - 1; break; }
                if (first < 0) break;
                // kept point `kept` goes to slot kept <= c0 + first: a slot whose point has been decided (or is this one)
                if (tid == first) { pt[kept] = me; alive = false; }
                __syncthreads();
                const float2 q = pt[kept];
                kept++;
                if (alive && hv_select_near(q.x, q.y, me.x, me.y, r2)) alive = false;
                if (zero + kept >= a.maxTracks) { full = true; break; }
            }
            __syncthreads();                                           // s_live is rewritten by the next chunk
        }
        count = zero + kept;
    }

    for (int i = tid; i < a.capacity; i += SEL_NT) {
        float x = HV_CORNER_NONE_F, y = HV_CORNER_NONE_F;
        if (i < zero) x = y = 0.f;
        else if (i < count) { const float2 p = pt[i - zero]; x = p.x; y = p.y; }
        a.out[2 * i] = x; a.out[2 * i + 1] = y;
    }
    if (tid == 0) *a.count = count;
    if (a.done.hostFlag) {
        __threadfence_system();
        __syncthreads();
        if (tid == 0) hv_signal_done(a.done);
    }
}

__global__ void __launch_bounds__(SEL_NT) hv_gftt_select_kernel(const __grid_constant__ GfttSelectArgs a)
{
    hv_gftt_select_list(a);
}

// one list per CTA; each CTA sorts its own pow2 keys in the dynamic shared memory sized for the largest
__global__ void __launch_bounds__(SEL_NT) hv_gftt_select_batch_kernel(const __grid_constant__ GfttSelectBatchArgs b)
{
    hv_gftt_select_list(b.job[blockIdx.x]);
}

#include "hv_device_once.cuh"

static bool g_select_attr_set[64], g_select_batch_attr_set[64];

cudaError_t hv_launch_gftt_select(const GfttSelectArgs& a, cudaStream_t stream)
{
    if (hv_first_use_on_device(g_select_attr_set)) {
        cudaError_t e = cudaFuncSetAttribute(hv_gftt_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)(HV_GFTT_SELECT_MAX_KP * sizeof(unsigned long long)));
        if (e != cudaSuccess) return e;
    }
    hv_gftt_select_kernel<<<1, SEL_NT, (size_t)a.pow2 * sizeof(unsigned long long), stream>>>(a);
    return cudaGetLastError();
}

cudaError_t hv_launch_gftt_select_batch(const GfttSelectBatchArgs& b, int njobs, int maxPow2, cudaStream_t stream)
{
    if (hv_first_use_on_device(g_select_batch_attr_set)) {
        cudaError_t e = cudaFuncSetAttribute(hv_gftt_select_batch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)(HV_GFTT_SELECT_MAX_KP * sizeof(unsigned long long)));
        if (e != cudaSuccess) return e;
    }
    hv_gftt_select_batch_kernel<<<njobs, SEL_NT, (size_t)maxPow2 * sizeof(unsigned long long), stream>>>(b);
    return cudaGetLastError();
}
