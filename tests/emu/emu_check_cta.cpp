// tests/emu/emu_check_cta.cpp -- the one-CTA outlier check (ek2_check_cta, ekf_cluster2.cuh) on the host emulator against the
// cluster body (ek2_body, mode EKF_MODE_CHECK) on the same inputs: the three result words (status, chi2, numeric flag) must be
// bitwise equal, and (m, P) untouched. Sweeps n over 1 .. 84 across the 8-row pivot blocks and the one-stage / two-stage S boundary
// (n * n <= 1024), l below one column block, l = N and l not a multiple of 4, N = 62 / 160 / 202, f given or NULL (v = y - H m), and
// the early exits: RMSE gate, skipChi2, a non-positive pivot.
#include "emu_cluster.h"
#include "ekf_cluster2.cuh"
namespace cg = cooperative_groups;

#if !defined(EMU_CLUSTER_THREADS) || defined(EMU_AS_LIB)
EMU_CLUSTER_BODY(emu_check_cluster_body) { EkfUpdateArgs aa = *(const EkfUpdateArgs*)ctx; ek2_body<false>(aa, dyn, cg::this_cluster()); }
EMU_CLUSTER_BODY(emu_check_cta_body) { ek2_check_cta(*(const EkfUpdateArgs*)ctx, dyn); }
#endif
#ifndef EMU_AS_LIB

static double rnd() { return rand() / (double)RAND_MAX - 0.5; }

// special: 0 none, 1 RMSE gate trips, 2 RMSE gate passes, 3 skipChi2, 4 S not positive definite
struct Case { int N, n, l, fNull, special; double yscale; };

int main(int argc, char** argv)
{
    std::vector<Case> cases;
    const int Ns[] = {62, 160, 202}, ns[] = {1, 7, 8, 9, 31, 32, 33, 84};
    for (int N : Ns) {
        const int B = (N + EK2_C - 1) / EK2_C;
        const int ls[] = {B - 3, N, 37, N - 2 * B + 1};       // below one block; all of N; odd; ending inside a block
        int q = 0;
        for (int n : ns) {
            if (n > N) continue;
            cases.push_back({N, n, ls[q % 4], q % 3 == 1, 0, q % 4 == 3 ? 40.0 : 0.02});
            q++;
        }
    }
    cases.push_back({160, 84, 160, 0, 0, 40.0});              // the largest bench check, outlier
    cases.push_back({160, 20, 55, 0, 1, 0.02});
    cases.push_back({160, 20, 55, 1, 2, 0.02});
    cases.push_back({62, 8, 34, 0, 3, 0.02});
    cases.push_back({160, 40, 90, 0, 4, 0.02});
    cases.push_back({202, 9, 202, 1, 4, 0.02});
    const int only = argc > 1 ? atoi(argv[1]) : -1;
    int fails = 0;
    for (int idx = 0; idx < (int)cases.size(); idx++) {
        if (only >= 0 && idx != only) continue;
        const Case& cs = cases[idx];
        const int N = cs.N, n = cs.n, l = cs.l;
        srand(500 + idx);
        emu::Arena arena((size_t)64 << 20);
        double* m = arena.alloc<double>(N); double* P = arena.alloc<double>((size_t)N * N);
        double* H = arena.alloc<double>((size_t)n * l); double* f = arena.alloc<double>(n); double* y = arena.alloc<double>(n);
        double* resC = arena.alloc<double>(EKF_RES_STRIDE); double* resT = arena.alloc<double>(EKF_RES_STRIDE);
        double* cwork = arena.alloc<double>((size_t)10 * N * N);
        {
            std::vector<double> Bm((size_t)N * N);
            for (auto& x : Bm) x = rnd();
            for (int i = 0; i < N; i++)
                for (int j = 0; j < N; j++) {
                    double s = 0; for (int k = 0; k < N; k++) s += Bm[i + (size_t)k * N] * Bm[j + (size_t)k * N];
                    P[i + (size_t)j * N] = 0.4 * s / N + (i == j ? 0.5 : 0.0);
                }
            if (cs.special == 4) for (int i = 0; i < N; i++) P[i + (size_t)i * N] -= 400.0;
            for (int i = 0; i < N; i++) m[i] = 0.3 * rnd();
        }
        for (size_t i = 0; i < (size_t)n * l; i++) H[i] = 0.2 * rnd();
        for (int i = 0; i < n; i++) { f[i] = 0.5 * rnd(); y[i] = f[i] + cs.yscale * rnd(); }
        const std::vector<double> P0(P, P + (size_t)N * N), m0(m, m + N);

        EkfUpdateArgs a; memset(&a, 0, sizeof(a));
        a.b.m = m; a.b.P = P; a.b.cwork = cwork; a.b.N = N; a.b.trail = (N - EKF_CAM) / EKF_POSE;
        a.op = EKF_OP_DENSE; a.mode = EKF_MODE_CHECK; a.n = n; a.l = l; a.H = H; a.f = cs.fNull ? nullptr : f; a.y = y;
        a.noiseScale = 1e-4; a.Rdiag = 0.0025 * a.noiseScale; a.chi2Thr = 3.0 * n + 5.0;
        a.rmseThr = cs.special == 1 ? 1e-3 : cs.special == 2 ? 1e3 : -1.0;
        a.skipChi2 = cs.special == 3;
        for (int i = 0; i < 8; i++) resC[i] = resT[i] = -7.0;
        EkfUpdateArgs ac = a, at = a;
        ac.b.res = resC; at.b.res = resT;
        const size_t smemC = ek2_smem_bytes(n, l, N, false), smemT = ek2_check_cta_smem_bytes(n, l, N);
        const int badC = EMU_LAUNCH_CLUSTER(arena, EK2_C, EK2_NT, smemC, emu_check_cluster_body, &ac);
        const int badT = EMU_LAUNCH_CLUSTER(arena, 1, EK2_NT, smemT, emu_check_cta_body, &at);
        bool ok = badC == 0 && badT == 0 && memcmp(resC, resT, 3 * sizeof(double)) == 0 && resC[0] != -7.0;
        ok = ok && memcmp(P0.data(), P, sizeof(double) * (size_t)N * N) == 0 && memcmp(m0.data(), m, sizeof(double) * N) == 0;
        const int want = cs.special == 1 ? 2 : cs.special == 4 ? 1 : -1;
        if (want >= 0) ok = ok && (int)resC[0] == want;
        if (cs.special == 4) ok = ok && resC[2] == 1.0;
        printf("[%2d] N=%3d n=%2d l=%3d f %-4s special %d smem %6.1f / %6.1f KB: cluster %g %.17g %g  cta %g %.17g %g  %s\n", idx, N, n, l,
               cs.fNull ? "NULL" : "set", cs.special, smemC / 1024.0, smemT / 1024.0, resC[0], resC[1], resC[2], resT[0], resT[1], resT[2], ok ? "ok" : "FAIL");
        fflush(stdout);
        fails += !ok;
        munmap(arena.base, arena.size);
    }
    return fails;
}
#endif  // EMU_AS_LIB
