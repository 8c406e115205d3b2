// hybvio_b200/csrc/ekf_cluster2.cu -- kernels and launchers of the second-generation cluster update (ekf_cluster2.cuh):
// P column blocks resident in shared memory, small inter-CTA exchanges through distributed shared memory.
#include <cooperative_groups.h>
#include "hv_device_once.cuh"
#include <math.h>
#include <stdlib.h>
namespace cg = cooperative_groups;

#ifdef HV_EKF_TIMING
// phase timestamps (globaltimer, ns) into res[8 + i] (tools/ekf_phases.py)
#define EK2_PHASE(i) do { if (c == 0 && tid == 0) { unsigned long long t_; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_)); a.b.res[8 + (i)] = (double)t_; } } while (0)
#endif
#include "ekf_cluster2.cuh"

__global__ void __launch_bounds__(EK2_NT) ekf_update_cluster2_kernel(EkfUpdateArgs a)
{
    extern __shared__ __align__(16) double ek2_sm[];
    ek2_body<false>(a, ek2_sm, cg::this_cluster());
}

// The row-chunked form (a.rowChunk > 0): a dense visual op whose whole tableau does not fit beside the P blocks
__global__ void __launch_bounds__(EK2_NT) ekf_update_cluster2_chunked_kernel(EkfUpdateArgs a)
{
    extern __shared__ __align__(16) double ek2_sm[];
    ek2_body<true>(a, ek2_sm, cg::this_cluster());
}

// Item of the batch that runs the j-th check of one form (compact: on one CTA; otherwise on a cluster of its own), in item order;
// past the last: -1 for the compact form, b.count (the augmentation) for the other
__device__ __forceinline__ int ek2_batch_item(const EkfCheckBatch& b, int compact, int j)
{
    for (int i = 0; i < b.count; i++)
        if (b.it[i].compact == compact && j-- == 0) return i;
    return compact ? -1 : b.count;
}

// Batched outlier checks against the same state (read-only), each with its own result words (index = item). The clusters, in order:
//   ceil(b.compact / 8) clusters whose CTA r runs the (8q + r)-th compact check on its own (ek2_check_cta: 8 checks per 8 SMs);
//   one cluster per check that does not fit one CTA (ek2_body, as a single check);
//   aug != a: one more cluster runs the pose augmentation that FOLLOWS the checks in the caller's sequence (aug: its argument block).
// The checks only read (m, P) and the augmentation writes its result to the second buffers (aug.specP / aug.specM, adopted by the
// host with a pointer swap), so the two are independent and share the launch instead of queueing behind each other.
__global__ void __launch_bounds__(EK2_NT) ekf_check_batch_cluster2_kernel(EkfUpdateArgs a, EkfCheckBatch b, EkfUpdateArgs aug)
{
    extern __shared__ __align__(16) double ek2_sm[];
    cg::cluster_group cluster = cg::this_cluster();
    const int k = blockIdx.x / EK2_C, compactClusters = (b.compact + EK2_C - 1) / EK2_C;
    const bool compact = k < compactClusters;
    const int inst = compact ? ek2_batch_item(b, 1, k * EK2_C + (int)cluster.block_rank()) : ek2_batch_item(b, 0, k - compactClusters);
    if (inst < 0) return;                                       // the last compact cluster has fewer than 8 checks
    if (inst >= b.count) a = aug;                               // (one call of the body: its code is 340 KB)
    else {
        const EkfCheckItem& it = b.it[inst];
        a.H = it.H; a.f = it.f; a.y = it.y; a.n = it.n; a.l = it.l;
        a.Rdiag = it.Rdiag; a.chi2Thr = it.chi2Thr; a.rmseThr = it.rmseThr; a.skipChi2 = it.skipChi2;
        if (a.sig) a.sig += 4 * inst;
        if (a.slot) a.slot += 4 * inst;
    }
    a.b.res += (size_t)EKF_RES_STRIDE * inst;
    if (compact) { ek2_check_cta(a, ek2_sm); return; }
    a.b.cwork += (size_t)inst * 10 * a.b.N * a.b.N;           // own exchange area (Z | reduced S | partial S)
    ek2_body<false>(a, ek2_sm, cluster);
}
static_assert(2 * sizeof(EkfUpdateArgs) + sizeof(EkfCheckBatch) <= 4096, "ekf_check_batch_cluster2_kernel: arguments beyond 4 KB of parameter space");

// The state mean of the pose augmentation on one CTA (ek2_aug_mean_cta), while a cluster elsewhere forms the covariance
__global__ void __launch_bounds__(EK2_NT) ekf_aug_mean_kernel(EkfUpdateArgs a)
{
    extern __shared__ __align__(16) double ek2_sm[];
    ek2_aug_mean_cta(a, ek2_sm);
}

// Group launch (hv_ekf_group_run_device): cluster i runs args[i], an instance of any filter of the group. The blocks live in device
// memory (hundreds of clusters do not fit the parameter space); no cluster waits for another, so a grid of many clusters runs in waves.
__global__ void __launch_bounds__(EK2_NT) ekf_group_cluster2_kernel(const EkfUpdateArgs* __restrict__ args)
{
    extern __shared__ __align__(16) double ek2_sm[];
    ek2_group_body(args, blockIdx.x / EK2_C, ek2_sm, cg::this_cluster());
}

#define EK2_STATIC_SMEM (sizeof(double) * (2 + EK2_LINV_DOUBLES + 2 + EK2_MAXN) + 256)
#define EK2_SMEM_LIMIT (227 * 1024)

bool ekf_cluster2_fits(int n, int l, int N, bool joseph)
{
    return N <= EK2_MAXN && ek2_smem_bytes(n, l, N, joseph) + EK2_STATIC_SMEM <= EK2_SMEM_LIMIT;
}

int ekf_cluster2_chunk_rows(int n, int l, int N)
{
    if (N > EK2_MAXN) return 0;
    for (int h = n; h >= 1 && h >= (n < EK2_MIN_CHUNK ? n : EK2_MIN_CHUNK); h--)      // (the working set grows with h)
        if (ek2_smem_bytes_chunked(h, n, l, N) + EK2_STATIC_SMEM <= EK2_SMEM_LIMIT) return h;
    return 0;
}

template <class K, class... Args>
static cudaError_t ek2_launch(K kernel, int nclusters, size_t smem, cudaStream_t s, Args... args)
{
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(EK2_C * nclusters); cfg.blockDim = dim3(EK2_NT); cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute at[2];
    at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = EK2_C; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    // programmatic dependent launch: this kernel may start while the previous KERNEL of the stream is still running (it waits
    // in griddepcontrol.wait before it reads the filter state); HV_EKF_NO_PDL=1 switches it off (A/B)
    static const bool pdl = getenv("HV_EKF_NO_PDL") == nullptr;
    at[1].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = pdl ? 2 : 1;
    return cudaLaunchKernelEx(&cfg, kernel, args...);
}

template <class K>
static cudaError_t ek2_prepare(K kernel)
{
    return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(EK2_SMEM_LIMIT - EK2_STATIC_SMEM));
}

cudaError_t ekf_launch_update_cluster2(const EkfUpdateArgs& a, cudaStream_t s)
{
    static bool seen[64], seenChunked[64];            // per device (hv_common.cuh)
    if (a.rowChunk > 0) {
        if (hv_first_use_on_device(seenChunked)) { cudaError_t e = ek2_prepare(ekf_update_cluster2_chunked_kernel); if (e != cudaSuccess) return e; }
        const size_t smem = ek2_smem_bytes_chunked(a.rowChunk < a.n ? a.rowChunk : a.n, a.n, a.l, a.b.N);
        return ek2_launch(ekf_update_cluster2_chunked_kernel, 1, smem, s, a);
    }
    if (hv_first_use_on_device(seen)) { cudaError_t e = ek2_prepare(ekf_update_cluster2_kernel); if (e != cudaSuccess) return e; }
    const size_t smem = ek2_smem_bytes(a.n, a.l, a.b.N, a.op == EKF_OP_AUGMENT);
    return ek2_launch(ekf_update_cluster2_kernel, 1, smem, s, a);
}

// A check runs on one CTA iff its working set fits and its size n l^2 is at most EK2_CTA_CHECK_MAX. One CTA does the work of eight
// serially: at the bench's n = 84, l = 160 (n l^2 = 2.15e6) a batch took 80 us instead of 38 us on an H100 SXM (700 W), which the
// host-buffer entry points wait for; n = 40, l = 90 (3.2e5) and below gain. Larger checks keep a cluster of their own.
#define EK2_CTA_CHECK_MAX (1 << 20)
static bool ekf_check_on_one_cta(int n, int l, int N)
{
    return l <= N && (long long)n * l * l <= EK2_CTA_CHECK_MAX && ek2_check_cta_smem_bytes(n, l, N) + EK2_STATIC_SMEM <= EK2_SMEM_LIMIT;
}

cudaError_t ekf_launch_check_batch2(const EkfUpdateArgs& a, const EkfCheckBatch& b0, cudaStream_t s, const EkfUpdateArgs* aug)
{
    static bool seen[64];
    if (hv_first_use_on_device(seen)) { cudaError_t e = ek2_prepare(ekf_check_batch_cluster2_kernel); if (e != cudaSuccess) return e; }
    EkfCheckBatch b = b0;
    b.compact = 0;
    int clusters = aug ? 1 : 0;
    size_t smem = 0;
    for (int i = 0; i < b.count; i++) {
        EkfCheckItem& it = b.it[i];
        it.compact = ekf_check_on_one_cta(it.n, it.l, a.b.N) ? 1 : 0;
        const size_t v = it.compact ? ek2_check_cta_smem_bytes(it.n, it.l, a.b.N) : ek2_smem_bytes(it.n, it.l, a.b.N, false);
        if (v > smem) smem = v;
        b.compact += it.compact;
        clusters += 1 - it.compact;
    }
    clusters += (b.compact + EK2_C - 1) / EK2_C;
    if (aug) { const size_t v = ek2_smem_bytes(aug->n, aug->l, a.b.N, true); if (v > smem) smem = v; }
    return ek2_launch(ekf_check_batch_cluster2_kernel, clusters, smem, s, a, b, aug ? *aug : a);
}

bool ekf_aug_mean_fits(int N)
{
    return N <= EK2_MAXN && ek2_aug_mean_smem_bytes(EKF_POSE, EKF_CAM + EKF_POSE, N) <= EK2_SMEM_LIMIT;
}

cudaError_t ekf_launch_aug_mean(const EkfUpdateArgs& a, cudaStream_t s)
{
    static bool seen[64];
    if (hv_first_use_on_device(seen)) {
        cudaError_t e = cudaFuncSetAttribute(ekf_aug_mean_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)EK2_SMEM_LIMIT);
        if (e != cudaSuccess) return e;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(1); cfg.blockDim = dim3(EK2_NT); cfg.dynamicSmemBytes = ek2_aug_mean_smem_bytes(a.n, a.l, a.b.N); cfg.stream = s;
    cudaLaunchAttribute at[1];
    static const bool pdl = getenv("HV_EKF_NO_PDL") == nullptr;          // (as ek2_launch)
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, ekf_aug_mean_kernel, a);
}

cudaError_t ekf_launch_group_cluster2(const EkfUpdateArgs* hArgs, const EkfUpdateArgs* dArgs, int count, cudaStream_t s)
{
    static bool seen[64];
    if (hv_first_use_on_device(seen)) { cudaError_t e = ek2_prepare(ekf_group_cluster2_kernel); if (e != cudaSuccess) return e; }
    size_t smem = 0;
    for (int i = 0; i < count; i++) { const size_t v = ek2_smem_bytes(hArgs[i].n, hArgs[i].l, hArgs[i].b.N, hArgs[i].op == EKF_OP_AUGMENT); if (v > smem) smem = v; }
    return ek2_launch(ekf_group_cluster2_kernel, count, smem, s, dArgs);
}
