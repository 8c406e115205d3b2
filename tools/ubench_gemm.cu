// tools/ubench_gemm.cu -- the three dense products of the n = 84 update in isolation on one CTA (cycles, clock64): are they bound by the
// fp64 tensor rate (64 FMA/clk/SM: one DMMA per 4 cycles) or by something around it?
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -Ihybvio_b200/csrc -o tools/ubench_gemm tools/ubench_gemm.cu
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <cuda_runtime.h>
#include "ekf_cluster2.cuh"

__global__ void __launch_bounds__(EK2_NT) k_gemm(double* gS, long long* out, int variant)
{
    extern __shared__ __align__(16) double sm[];
    const int tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5;
    const int n = 84, l = 160, N = 160, Bc = 20, J0 = 0;
    const Ek2Geom g = ek2_geom(n, l, N, false);
    double* X = sm; double* T = X + g.X; double* PB = T + g.T;
    const int W = g.W, LD = g.LD;
    for (int i = tid; i < g.X; i += EK2_NT) X[i] = 1e-3 * (i % 17);
    for (int i = tid; i < g.T; i += EK2_NT) T[i] = 1e-3 * (i % 13);
    for (int i = tid; i < g.PB; i += EK2_NT) PB[i] = 1e-3 * (i % 11);
    __syncthreads();
    const double* Hs = X;
    for (int rep = 0; rep < 3; rep++) {
        __syncthreads();
        const long long t0 = clock64();
        if (variant == 0)        // HP[:, J_c] = H P[0:l, J_c]   (84 x 20 x 160)
            ek2_dmma_gemm(n, Bc, l, wrp, lane, Hs, 1, n, PB, 1, LD, [](int, int) { return 0.0; },
                          [&](int i, int j, double v0, double v1) { T[(size_t)i * W + n + j] = v0; if (j + 1 < Bc) T[(size_t)i * W + n + j + 1] = v1; });
        else if (variant == 1)   // partial S, upper tiles, stored tile-ordered to GLOBAL memory (84 x 84 x 20)
            ek2_dmma_gemm<true>(n, n, Bc, wrp, lane, T + n, W, 1, Hs + (size_t)J0 * n, n, 1, [](int, int) { return 0.0; },
                          [&](int i, int j, double v0, double v1) { const int mt = i >> 3, nt = j >> 3; double* dst = gS + 64 * (nt * (nt + 1) / 2 + mt) + 8 * (i & 7) + (j & 7); dst[0] = v0; dst[1] = v1; });
        else if (variant == 2)   // partial S, stored into the tableau (shared memory)
            ek2_dmma_gemm<true>(n, n, Bc, wrp, lane, T + n, W, 1, Hs + (size_t)J0 * n, n, 1, [](int, int) { return 0.0; },
                          [&](int i, int j, double v0, double v1) { T[(size_t)i * W + j] = v0; if (j + 1 < n) T[(size_t)i * W + j + 1] = v1; });
        else                     // downdate P[:, J_c] -= Z' Z[:, J_c]   (160 x 21 x 84)
            ek2_dmma_gemm(N, Bc + 1, n, wrp, lane, X, 1, LD, X + J0, LD, 1, [&](int i, int j) { return -PB[i + (size_t)min(j, Bc - 1) * LD]; },
                          [&](int i, int j, double v0, double v1) { if (j < Bc) PB[i + (size_t)j * LD] = -v0; if (j + 1 < Bc) PB[i + (size_t)(j + 1) * LD] = -v1; });
        __syncthreads();
        const long long t1 = clock64();
        if (tid == 0) out[variant * 3 + rep] = t1 - t0;
    }
}

int main()
{
    double* gS; long long* out;
    cudaMalloc(&gS, 8 * 8192); cudaMalloc(&out, 8 * 16);
    cudaFuncSetAttribute(k_gemm, cudaFuncAttributeMaxDynamicSharedMemorySize, 218 * 1024);
    const size_t smem = ek2_smem_bytes(84, 160, 160, false);
    const char* names[4] = {"HP 84 x 20 x 160 (1320 DMMA: 5280 cycles at the tensor rate)", "partial S 84 x 84 x 20, upper tiles -> global (330 DMMA: 1320 cycles)",
                            "partial S -> shared memory", "downdate 160 x 21 x 84 (1260 DMMA: 5040 cycles)"};
    for (int v = 0; v < 4; v++) {
        k_gemm<<<1, EK2_NT, smem>>>(gS, out, v);
        cudaError_t e = cudaGetLastError(); if (e == cudaSuccess) e = cudaDeviceSynchronize();
        long long h[12]; cudaMemcpy(h, out, sizeof(h), cudaMemcpyDeviceToHost);
        printf("%-75s: %s  cycles %lld %lld %lld\n", names[v], cudaGetErrorString(e), h[v * 3], h[v * 3 + 1], h[v * 3 + 2]);
    }
    return 0;
}
