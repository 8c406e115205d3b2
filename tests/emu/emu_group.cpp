// tests/emu/emu_group.cpp -- runs the body of the group cluster kernel (ek2_group_body, hybvio_b200/csrc/ekf_cluster2.cuh) on the host
// emulator: three clusters of one launch from two filters at N = 62, each on its own argument block -- filter A: a check+update in place;
// filter B: an outlier check and the augmentation into the second buffers, with their own exchange areas and result words (the layout
// hv_ekf_group_run_device gives a run of checks with the augmentation behind it) -- and compares every result with the C oracle.
#include "emu_cluster.h"
#include "ekf_cluster2.cuh"
namespace cg = cooperative_groups;

extern "C" {
struct orc_params { int camera_trail_length, hybrid_map_size; double v[20]; };
struct orc_ekf;
void orc_ekf_default_params(orc_params*);
orc_ekf* orc_ekf_create(const orc_params*);
void orc_ekf_destroy(orc_ekf*);
void orc_ekf_upload(orc_ekf*, const double*, const double*);
void orc_ekf_download(const orc_ekf*, double*, double*);
int orc_ekf_state_dim(const orc_ekf*);
double orc_chi2inv95(int);
int orc_ekf_visual_check(const orc_ekf*, const double*, int, int, const double*, const double*, double, double, double*);
void orc_ekf_visual_update(orc_ekf*, const double*, int, int, const double*, const double*, double);
void orc_ekf_augment(orc_ekf*, int);
}

struct GroupLaunch { const EkfUpdateArgs* args; int inst; };

#if !defined(EMU_CLUSTER_THREADS) || defined(EMU_AS_LIB)
EMU_CLUSTER_BODY(emu_group_body) { const GroupLaunch* g = (const GroupLaunch*)ctx; ek2_group_body(g->args, g->inst, dyn, cg::this_cluster()); }
#endif
#ifndef EMU_AS_LIB

static double rnd() { return rand() / (double)RAND_MAX - 0.5; }
static double gauss() { double s = 0; for (int i = 0; i < 12; i++) s += rand() / (double)RAND_MAX; return s - 6.0; }

struct Filter { double *m, *P, *m2, *P2, *res, *cwork, *slot; };

static void random_state(int N, int trail, double* m, double* P)
{
    std::vector<double> Bm((size_t)N * N);
    for (auto& x : Bm) x = rnd();
    for (int i = 0; i < N; i++) for (int j = 0; j < N; j++) { double s = 0; for (int k = 0; k < N; k++) s += Bm[i + (size_t)k * N] * Bm[j + (size_t)k * N]; P[i + (size_t)j * N] = 0.05 * s + (i == j ? 0.5 : 0.0); }
    for (int i = 0; i < N; i++) m[i] = 0.3 * rnd();
    for (int p = 0; p <= trail; p++) {
        double* q = p == 0 ? m + EKF_ORI : m + EKF_CAM + EKF_POSE * (p - 1) + 3;
        double nn = 0; for (int i = 0; i < 4; i++) { q[i] = rnd() + (i == 0); nn += q[i] * q[i]; }
        for (int i = 0; i < 4; i++) q[i] /= std::sqrt(nn);
    }
}

static double max_rel(const double* a, const double* b, size_t n)
{
    double e = 0, mx = 1e-300;
    for (size_t i = 0; i < n; i++) { e = std::fmax(e, std::fabs(a[i] - b[i])); mx = std::fmax(mx, std::fabs(b[i])); }
    return e / mx;
}

int main()
{
    srand(7);
    const int trail = 6;
    orc_params prm; orc_ekf_default_params(&prm);
    prm.camera_trail_length = trail;
    orc_ekf* oa = orc_ekf_create(&prm); orc_ekf* ob = orc_ekf_create(&prm);
    const int N = orc_ekf_state_dim(oa);
    const size_t NN = (size_t)N * N;
    const double noiseScale = prm.v[0] * prm.v[0], r = 0.05;
    emu::Arena arena((size_t)64 << 20);
    Filter F[2];
    for (Filter& f : F) {
        f.m = arena.alloc<double>(N); f.P = arena.alloc<double>(NN); f.m2 = arena.alloc<double>(N); f.P2 = arena.alloc<double>(NN);
        f.res = arena.alloc<double>(EKF_RES_STRIDE * 2); f.cwork = arena.alloc<double>(2 * 10 * NN); f.slot = arena.alloc<double>(8);
        random_state(N, trail, f.m, f.P);
        for (size_t i = 0; i < NN; i++) f.P2[i] = -3.0;
        for (int i = 0; i < N; i++) f.m2[i] = -3.0;
        for (int i = 0; i < 8; i++) f.slot[i] = -7.0;
    }
    orc_ekf_upload(oa, F[0].m, F[0].P); orc_ekf_upload(ob, F[1].m, F[1].P);
    const std::vector<double> mB(F[1].m, F[1].m + N), PB(F[1].P, F[1].P + NN);
    // measurements: A n = 13 l = 41 (check+update), B n = 8 l = 34 (check)
    const int nA = 13, lA = 41, nB = 8, lB = 34;
    double* HA = arena.alloc<double>(nA * lA); double* fA = arena.alloc<double>(nA); double* yA = arena.alloc<double>(nA);
    double* HB = arena.alloc<double>(nB * lB); double* fB = arena.alloc<double>(nB); double* yB = arena.alloc<double>(nB);
    for (int i = 0; i < nA * lA; i++) HA[i] = 0.1 * gauss();
    for (int i = 0; i < nA; i++) { fA[i] = 0.5 * gauss(); yA[i] = fA[i] + 0.02 * gauss(); }
    for (int i = 0; i < nB * lB; i++) HB[i] = 0.1 * gauss();
    for (int i = 0; i < nB; i++) { fB[i] = 0.5 * gauss(); yB[i] = fB[i] + 0.02 * gauss(); }

    EkfUpdateArgs* args = arena.alloc<EkfUpdateArgs>(3);
    memset(args, 0, 3 * sizeof(EkfUpdateArgs));
    auto bufs = [&](EkfUpdateArgs& a, const Filter& f, int inst) {
        a.b.m = f.m; a.b.P = f.P; a.b.P2 = f.P2; a.b.N = N; a.b.trail = trail; a.b.mapDim = 0;
        a.b.res = f.res + EKF_RES_STRIDE * inst; a.b.cwork = f.cwork + (size_t)inst * 10 * NN;
        a.noiseScale = noiseScale; a.rmseThr = -1.0;
    };
    auto dense = [&](EkfUpdateArgs& a, const double* H, const double* f, const double* y, int n, int l, int mode) {
        a.op = EKF_OP_DENSE; a.H = H; a.f = f; a.y = y; a.n = n; a.l = l; a.mode = mode; a.Rdiag = r * r * noiseScale;
        a.chi2Thr = orc_chi2inv95(n); a.normalizeAll = 1;
    };
    bufs(args[0], F[0], 0); dense(args[0], HA, fA, yA, nA, lA, EKF_MODE_CHECK_UPDATE); args[0].slot = F[0].slot;
    bufs(args[1], F[1], 0); dense(args[1], HB, fB, yB, nB, lB, EKF_MODE_CHECK); args[1].slot = F[1].slot;
    bufs(args[2], F[1], 1);
    {
        EkfUpdateArgs& a = args[2];
        a.op = EKF_OP_AUGMENT; a.n = EKF_POSE; a.l = EKF_CAM + EKF_POSE; a.mode = EKF_MODE_UPDATE; a.Rdiag = prm.v[17] * noiseScale;
        a.dropIdx = trail - 1; a.augNoisePos = prm.v[9] * prm.v[9] * noiseScale; a.augNoiseOri = prm.v[10] * prm.v[10] * noiseScale;
        a.normalizeAll = 1; a.symmetrize = 1; a.specP = F[1].P2; a.specM = F[1].m2;
    }
    // oracle: A check then update iff inlier; B check and augmentation, both of the state as it was
    double chiA = 0, chiB = 0;
    const int stA = orc_ekf_visual_check(oa, HA, nA, lA, fA, yA, r, -1.0, &chiA);
    if (stA == 0) orc_ekf_visual_update(oa, HA, nA, lA, fA, yA, r);
    const int stB = orc_ekf_visual_check(ob, HB, nB, lB, fB, yB, r, -1.0, &chiB);
    orc_ekf_augment(ob, trail - 1);

    int fails = 0;
    for (int inst = 2; inst >= 0; inst--) {             // the augmentation first: the check of the same filter must still see (m, P)
        GroupLaunch g = {args, inst};
        const size_t smem = ek2_smem_bytes(args[inst].n, args[inst].l, N, args[inst].op == EKF_OP_AUGMENT);
        const int bad = EMU_LAUNCH_CLUSTER(arena, EK2_C, EK2_NT, smem, emu_group_body, &g);
        printf("cluster %d: %s\n", inst, bad == 0 ? "ran" : "FAIL"); fails += bad != 0;
    }
    std::vector<double> om(N), oP(NN);
    orc_ekf_download(oa, om.data(), oP.data());
    const double eA = std::fmax(max_rel(F[0].m, om.data(), N), max_rel(F[0].P, oP.data(), NN));
    bool ok = (int)F[0].res[0] == stA && std::fabs(F[0].res[1] - chiA) <= 1e-9 * std::fmax(1.0, chiA) && eA < 1e-9 &&
              F[0].slot[0] == F[0].res[0] && F[0].slot[1] == F[0].res[1] && F[0].slot[2] == F[0].res[2];
    printf("filter A check+update: status %d/%d chi2 %.6g/%.6g err %.2e  %s\n", (int)F[0].res[0], stA, F[0].res[1], chiA, eA, ok ? "ok" : "FAIL");
    fails += !ok;
    ok = (int)F[1].res[0] == stB && std::fabs(F[1].res[1] - chiB) <= 1e-9 * std::fmax(1.0, chiB) &&
         F[1].slot[0] == F[1].res[0] && F[1].slot[1] == F[1].res[1] && F[1].slot[2] == F[1].res[2] &&
         memcmp(F[1].m, mB.data(), N * sizeof(double)) == 0 && memcmp(F[1].P, PB.data(), NN * sizeof(double)) == 0;
    printf("filter B check: status %d/%d chi2 %.6g/%.6g, (m, P) untouched  %s\n", (int)F[1].res[0], stB, F[1].res[1], chiB, ok ? "ok" : "FAIL");
    fails += !ok;
    orc_ekf_download(ob, om.data(), oP.data());
    const double eB = std::fmax(max_rel(F[1].m2, om.data(), N), max_rel(F[1].P2, oP.data(), NN));
    ok = eB < 1e-9 && F[1].slot[4] == -7.0;           // (the augmentation has no slot: the check's neighbour slot stays as it was)
    printf("filter B augmentation into the second buffers: err %.2e  %s\n", eB, ok ? "ok" : "FAIL");
    fails += !ok;
    orc_ekf_destroy(oa); orc_ekf_destroy(ob);
    munmap(arena.base, arena.size);
    return fails;
}
#endif  // EMU_AS_LIB
