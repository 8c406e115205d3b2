// tools/ubench_update_twice.cu -- how much of the update kernel's time is instruction fetch? The body of ekf_cluster2.cuh is run several
// times INSIDE one launch on an 8-CTA cluster (same measurement, the filter state evolves): the first pass fetches its ~80 KB of
// executed code from L2, the later ones find whatever the instruction caches of the SM keep.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -Ihybvio_b200/csrc -o tools/ubench_update_twice tools/ubench_update_twice.cu
#include <cooperative_groups.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <vector>
#include <cuda_runtime.h>
namespace cg = cooperative_groups;
#include "ekf_cluster2.cuh"

#define REPS 4
__global__ void __launch_bounds__(EK2_NT) k_rep(EkfUpdateArgs a, unsigned long long* stamps)
{
    extern __shared__ __align__(16) double sm[];
    cg::cluster_group cluster = cg::this_cluster();
    for (int rep = 0; rep < REPS; rep++) {
        if (cluster.block_rank() == 0 && threadIdx.x == 0) { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); stamps[rep] = t; }
        EkfUpdateArgs b = a;
        ek2_body(b, sm, cluster);
        cluster.sync();
    }
    if (cluster.block_rank() == 0 && threadIdx.x == 0) { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); stamps[REPS] = t; }
}

int main()
{
    const int trail = 20, N = 20 + 7 * trail;
    for (int n : {8, 20, 40, 84}) {
        const int l = n == 84 ? 160 : 20 + 7 * (n / 4 > 1 ? n / 4 : 1);
        srand(3);
        std::vector<double> B((size_t)N * N), P((size_t)N * N), m(N), H((size_t)n * l), f(n), y(n);
        for (auto& x : B) x = rand() / (double)RAND_MAX - 0.5;
        for (int i = 0; i < N; i++) for (int j = 0; j < N; j++) { double s = 0; for (int k = 0; k < N; k++) s += B[i + (size_t)k * N] * B[j + (size_t)k * N]; P[i + (size_t)j * N] = 0.05 * s + (i == j ? 0.5 : 0.0); }
        for (auto& x : m) x = 0.3 * (rand() / (double)RAND_MAX - 0.5);
        m[6] = 1; m[7] = m[8] = m[9] = 0;
        for (int p = 0; p < trail; p++) { m[20 + 7 * p + 3] = 1; m[20 + 7 * p + 4] = m[20 + 7 * p + 5] = m[20 + 7 * p + 6] = 0; }
        for (auto& x : H) x = 0.1 * (rand() / (double)RAND_MAX - 0.5);
        for (int i = 0; i < n; i++) { f[i] = 0.5 * (rand() / (double)RAND_MAX - 0.5); y[i] = f[i] + 0.02 * (rand() / (double)RAND_MAX - 0.5); }
        double *dP, *dm, *dH, *df, *dy, *dres, *dcw; unsigned long long* dst;
        cudaMalloc(&dP, P.size() * 8); cudaMalloc(&dm, N * 8); cudaMalloc(&dH, H.size() * 8); cudaMalloc(&df, n * 8); cudaMalloc(&dy, n * 8);
        cudaMalloc(&dres, 64 * 8); cudaMalloc(&dcw, (size_t)10 * N * N * 8); cudaMalloc(&dst, (REPS + 1) * 8);
        cudaMemcpy(dP, P.data(), P.size() * 8, cudaMemcpyHostToDevice); cudaMemcpy(dm, m.data(), N * 8, cudaMemcpyHostToDevice);
        cudaMemcpy(dH, H.data(), H.size() * 8, cudaMemcpyHostToDevice); cudaMemcpy(df, f.data(), n * 8, cudaMemcpyHostToDevice); cudaMemcpy(dy, y.data(), n * 8, cudaMemcpyHostToDevice);
        EkfUpdateArgs a; memset(&a, 0, sizeof(a));
        a.b.m = dm; a.b.P = dP; a.b.res = dres; a.b.cwork = dcw; a.b.N = N; a.b.trail = trail;
        a.op = EKF_OP_DENSE; a.n = n; a.l = l; a.mode = EKF_MODE_UPDATE; a.noiseScale = 1e4; a.rmseThr = -1.0; a.H = dH; a.f = df; a.y = dy;
        a.Rdiag = 0.05 * 0.05 * 1e4; a.normalizeAll = 1;
        const size_t smem = ek2_smem_bytes(n, l, N, false);
        { cudaError_t e0 = cudaFuncSetAttribute(k_rep, cudaFuncAttributeMaxDynamicSharedMemorySize, 212 * 1024); if (e0 != cudaSuccess) { printf("attr: %s\n", cudaGetErrorString(e0)); return 1; } }
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(8); cfg.blockDim = dim3(EK2_NT); cfg.dynamicSmemBytes = smem;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = 8; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
        unsigned long long st[REPS + 1];
        for (int launch = 0; launch < 3; launch++) {
            cudaError_t e = cudaLaunchKernelEx(&cfg, k_rep, a, dst);
            if (e == cudaSuccess) e = cudaDeviceSynchronize();
            if (e != cudaSuccess) { printf("n=%d: %s\n", n, cudaGetErrorString(e)); return 1; }
            cudaMemcpy(st, dst, sizeof(st), cudaMemcpyDeviceToHost);
            printf("n=%2d l=%3d launch %d: passes", n, l, launch);
            for (int r = 0; r < REPS; r++) printf(" %6.2f", (st[r + 1] - st[r]) / 1e3);
            printf(" us\n");
        }
        std::vector<double> Pout(P.size());
        cudaMemcpy(Pout.data(), dP, P.size() * 8, cudaMemcpyDeviceToHost);
        double tr = 0; for (int i = 0; i < N; i++) tr += Pout[i + (size_t)i * N];
        printf("   trace(P) after %d updates: %.6f (finite: %d)\n", 3 * REPS, tr, (int)std::isfinite(tr));
        cudaFree(dP); cudaFree(dm); cudaFree(dH); cudaFree(df); cudaFree(dy); cudaFree(dres); cudaFree(dcw); cudaFree(dst);
    }
    return 0;
}
