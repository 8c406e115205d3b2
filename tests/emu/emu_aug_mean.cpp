// tests/emu/emu_aug_mean.cpp -- the one-CTA mean of the pose augmentation (ek2_aug_mean_cta, ekf_cluster2.cuh) on the host emulator
// against the cluster body (ek2_body, EKF_OP_AUGMENT with second buffers) on the same inputs: the state mean both leave in specM and the
// three result words (status, chi2, numeric flag) must be bitwise equal, and (m, P) untouched. Sweeps N = 62 / 160 / 202, a pose trail
// that is not yet full (the unused slots as the filter creates them: zero mean, diagonal covariance) and a full one, the discarded pose
// (the last one, what index -1 means, and one in the middle), the deferred symmetrisation on and off, and a non-positive pivot.
#include "emu_cluster.h"
#include "ekf_cluster2.cuh"
namespace cg = cooperative_groups;

#if !defined(EMU_CLUSTER_THREADS) || defined(EMU_AS_LIB)
EMU_CLUSTER_BODY(emu_aug_cluster_body) { EkfUpdateArgs aa = *(const EkfUpdateArgs*)ctx; ek2_body<false>(aa, dyn, cg::this_cluster()); }
EMU_CLUSTER_BODY(emu_aug_mean_body) { ek2_aug_mean_cta(*(const EkfUpdateArgs*)ctx, dyn); }
#endif
#ifndef EMU_AS_LIB

static double rnd() { return rand() / (double)RAND_MAX - 0.5; }

struct Case { int N, full, dropMid, symFirst, bad; };

int main(int argc, char** argv)
{
    std::vector<Case> cases;
    for (int N : {62, 160, 202})
        for (int full = 0; full < 2; full++)
            for (int dropMid = 0; dropMid < 2; dropMid++)
                for (int sym = 0; sym < 2; sym++) cases.push_back({N, full, dropMid, sym, 0});
    cases.push_back({160, 1, 1, 1, 1});
    const int only = argc > 1 ? atoi(argv[1]) : -1;
    int fails = 0;
    for (int idx = 0; idx < (int)cases.size(); idx++) {
        if (only >= 0 && idx != only) continue;
        const Case& cs = cases[idx];
        const int N = cs.N, trail = (N - EKF_CAM) / EKF_POSE, n = EKF_POSE, l = EKF_CAM + EKF_POSE;
        const int used = cs.full ? N : EKF_CAM + EKF_POSE * (trail / 3);       // states that carry data; the rest as hv_ekf_create leaves them
        srand(900 + idx);
        emu::Arena arena((size_t)96 << 20);
        double* m = arena.alloc<double>(N); double* P = arena.alloc<double>((size_t)N * N);
        double* P2 = arena.alloc<double>((size_t)N * N);
        double* mC = arena.alloc<double>(N); double* mT = arena.alloc<double>(N);
        double* resC = arena.alloc<double>(EKF_RES_STRIDE); double* resT = arena.alloc<double>(EKF_RES_STRIDE);
        double* cwork = arena.alloc<double>((size_t)10 * N * N);
        {
            std::vector<double> Bm((size_t)used * used);
            for (auto& x : Bm) x = rnd();
            for (int i = 0; i < N; i++)
                for (int j = 0; j < N; j++) {
                    double s = 0.0;
                    if (i < used && j < used) {
                        for (int k = 0; k < used; k++) s += Bm[i + (size_t)k * used] * Bm[j + (size_t)k * used];
                        s = 0.4 * s / used;
                        if (j > i) s *= 1.0 + 1e-13 * rnd();      // slightly asymmetric, as P drifts between symmetrisations
                    }
                    P[i + (size_t)j * N] = s + (i == j ? (i < used ? 0.5 : 1e4) : 0.0);
                }
            for (int i = 0; i < N; i++) m[i] = i < used ? 0.3 * rnd() : 0.0;
            m[EKF_ORI] = 1.0 + 0.1 * rnd();
            for (int q = 0; q < trail; q++) if (EKF_CAM + EKF_POSE * q < used) m[EKF_CAM + EKF_POSE * q + 3] += 1.0;
        }
        for (int i = 0; i < N; i++) mC[i] = mT[i] = -7.0;
        const std::vector<double> P0(P, P + (size_t)N * N), m0(m, m + N);

        EkfUpdateArgs a; memset(&a, 0, sizeof(a));
        a.b.m = m; a.b.P = P; a.b.P2 = P2; a.b.cwork = cwork; a.b.N = N; a.b.trail = trail;
        a.op = EKF_OP_AUGMENT; a.mode = EKF_MODE_UPDATE; a.n = n; a.l = l; a.rmseThr = -1.0;
        a.noiseScale = 1e4; a.Rdiag = 1e-9 * a.noiseScale;
        a.symFirst = cs.symFirst; a.dropIdx = cs.dropMid ? trail / 2 : trail - 1;
        a.augNoisePos = 1e4 * a.noiseScale; a.augNoiseOri = 10.0 * a.noiseScale;
        if (cs.bad) a.augNoisePos = -a.augNoisePos;          // S = P_pose + visAugQ + R is then not positive definite
        a.normalizeAll = 1; a.symmetrize = 1;
        for (int i = 0; i < 8; i++) resC[i] = resT[i] = -7.0;
        EkfUpdateArgs ac = a, at = a;
        ac.b.res = resC; ac.specP = P2; ac.specM = mC;
        at.b.res = resT; at.specP = nullptr; at.specM = mT;
        const size_t smemC = ek2_smem_bytes(n, l, N, true), smemT = ek2_aug_mean_smem_bytes(n, l, N);
        const int badC = EMU_LAUNCH_CLUSTER(arena, EK2_C, EK2_NT, smemC, emu_aug_cluster_body, &ac);
        const int badT = EMU_LAUNCH_CLUSTER(arena, 1, EK2_NT, smemT, emu_aug_mean_body, &at);
        bool ok = badC == 0 && badT == 0 && memcmp(resC, resT, 3 * sizeof(double)) == 0 && resC[0] != -7.0;
        ok = ok && memcmp(mC, mT, sizeof(double) * N) == 0 && mC[0] != -7.0;
        ok = ok && memcmp(P0.data(), P, sizeof(double) * (size_t)N * N) == 0 && memcmp(m0.data(), m, sizeof(double) * N) == 0;
        ok = ok && (cs.bad ? resC[0] == 1.0 && resC[2] == 1.0 && memcmp(mT, m, sizeof(double) * N) == 0 : resC[0] == 0.0);
        int diff = 0;
        for (int i = 0; i < N; i++) diff += memcmp(&mC[i], &mT[i], sizeof(double)) != 0;
        printf("[%2d] N=%3d trail %-8s drop %2d symFirst %d bad %d smem %6.1f / %6.1f KB: chi2 %.17g / %.17g, m[%d] %.17g / %.17g, %d entries differ  %s\n",
               idx, N, cs.full ? "full" : "not full", a.dropIdx, cs.symFirst, cs.bad, smemC / 1024.0, smemT / 1024.0, resC[1], resT[1],
               EKF_CAM, mC[EKF_CAM], mT[EKF_CAM], diff, ok ? "ok" : "FAIL");
        fflush(stdout);
        fails += !ok;
        munmap(arena.base, arena.size);
    }
    return fails;
}
#endif  // EMU_AS_LIB
