// tests/emu/emu_update.cpp -- runs the REAL body of the cluster update kernel (hybvio_b200/csrc/ekf_cluster2.cuh) on the
// host emulator (one process per CTA, distributed shared memory = a shared mapping) and compares it with the C oracle.
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
void orc_ekf_symmetrize(orc_ekf*);
void orc_ekf_update_position(orc_ekf*, const double*, double);
void orc_ekf_update_zupt(orc_ekf*, double);
}

// the code one CTA of the cluster runs (not compiled into the driver executable of the all-CTAs-in-one-process mode, emu_cluster.h)
#if !defined(EMU_CLUSTER_THREADS) || defined(EMU_AS_LIB)
EMU_CLUSTER_BODY(emu_update_body) { EkfUpdateArgs aa = *(const EkfUpdateArgs*)ctx; ek2_body(aa, dyn, cg::this_cluster()); }
#endif
#ifndef EMU_AS_LIB

static double rnd() { return rand() / (double)RAND_MAX - 0.5; }
static double gauss() { double s = 0; for (int i = 0; i < 12; i++) s += rand() / (double)RAND_MAX; return s - 6.0; }

// gate: 0 none; 1 device-side gates present and satisfied (+ lateH, slot, bump); 2 / 3 / 4: gated off by the int flag / the counter / the double flag
struct Case { const char* name; int trail, op, n, l, mode; double yscale; int symFirst, drop; int gate = 0; double r2 = 0.0; int second = 0; };   // second: results into specP / specM, P and m untouched   // r2 > 0: the update uses its own noise level (two-R check+update)

// File mode (tests/test_ekf_ops_ref.py): one fixed-H update or augmentation of a given state. The input holds 17 doubles (op code
// 1..7 = zupt, zrupt, pseudo-velocity, position, zero height, orientation, augmentation; N, trail, mapDim, drop index, symFirst,
// normalizeAll, symmetrize, Rdiag, noiseScale, augNoisePos, augNoiseOri, defaultSpeed, ysmall[4]), then m (N) and P (N x N,
// column-major); the output holds m and P after the kernel body.
static int run_file(const char* in, const char* out)
{
    FILE* fi = fopen(in, "rb");
    if (!fi) { printf("cannot open %s\n", in); return 1; }
    double h[17];
    if (fread(h, sizeof(double), 17, fi) != 17) { fclose(fi); return 1; }
    const int code = (int)h[0], N = (int)h[1];
    static const int ops[8] = {-1, EKF_OP_ZUPT, EKF_OP_ZRUPT, EKF_OP_PSEUDO_VELOCITY, EKF_OP_POSITION, EKF_OP_ZERO_HEIGHT, EKF_OP_ORIENTATION, EKF_OP_AUGMENT};
    static const int ns[8] = {0, 3, 3, 1, 3, 1, 4, 7}, ls[8] = {0, EKF_VEL + 3, EKF_BGA + 3, EKF_VEL + 2, EKF_POS + 3, EKF_POS + 3, EKF_ORI + 4, EKF_CAM + EKF_POSE};
    if (code < 1 || code > 7 || N < EKF_CAM + EKF_POSE || N > EK2_MAXN) { fclose(fi); printf("bad header\n"); return 1; }
    emu::Arena arena((size_t)64 << 20);
    double* m = arena.alloc<double>(N); double* P = arena.alloc<double>((size_t)N * N);
    double* res = arena.alloc<double>(64); double* cwork = arena.alloc<double>((size_t)10 * N * N);
    const bool ok = fread(m, sizeof(double), N, fi) == (size_t)N && fread(P, sizeof(double), (size_t)N * N, fi) == (size_t)N * N;
    fclose(fi);
    if (!ok) return 1;
    EkfUpdateArgs a; memset(&a, 0, sizeof(a));
    a.b.m = m; a.b.P = P; a.b.res = res; a.b.cwork = cwork; a.b.N = N; a.b.trail = (int)h[2]; a.b.mapDim = (int)h[3];
    a.op = ops[code]; a.n = ns[code]; a.l = ls[code]; a.mode = EKF_MODE_UPDATE; a.rmseThr = -1.0;
    a.dropIdx = (int)h[4]; a.symFirst = (int)h[5]; a.normalizeAll = (int)h[6]; a.symmetrize = (int)h[7];
    a.Rdiag = h[8]; a.noiseScale = h[9]; a.augNoisePos = h[10]; a.augNoiseOri = h[11]; a.defaultSpeed = h[12];
    for (int i = 0; i < 4; i++) a.ysmall[i] = h[13 + i];
    const int bad = EMU_LAUNCH_CLUSTER(arena, EK2_C, EK2_NT, ek2_smem_bytes(a.n, a.l, N, a.op == EKF_OP_AUGMENT), emu_update_body, &a);
    FILE* fo = fopen(out, "wb");
    if (!fo) return 1;
    fwrite(m, sizeof(double), N, fo); fwrite(P, sizeof(double), (size_t)N * N, fo);
    fclose(fo);
    printf("file mode: op %d N=%d %s\n", code, N, bad == 0 ? "ok" : "FAIL");
    munmap(arena.base, arena.size);
    return bad;
}

int main(int argc, char** argv)
{
    if (argc == 4 && strcmp(argv[1], "file") == 0) return run_file(argv[2], argv[3]);
    const Case cases[] = {
        {"dense n=8 check+update", 20, EKF_OP_DENSE, 8, 34, EKF_MODE_CHECK_UPDATE, 0.02, 0, 0},
        {"dense n=20 check (outlier)", 20, EKF_OP_DENSE, 20, 55, EKF_MODE_CHECK, 40.0, 0, 0},
        {"dense n=40 update", 20, EKF_OP_DENSE, 40, 90, EKF_MODE_UPDATE, 0.02, 0, 0},
        {"dense n=84 check+update", 20, EKF_OP_DENSE, 84, 160, EKF_MODE_CHECK_UPDATE, 0.02, 0, 0},
        {"dense n=20 update N=62", 6, EKF_OP_DENSE, 20, 55, EKF_MODE_UPDATE, 0.02, 0, 0},
        {"augment drop last + deferred symmetrise", 20, EKF_OP_AUGMENT, 7, 27, EKF_MODE_UPDATE, 0, 1, -1},
        {"augment drop 3 N=62", 6, EKF_OP_AUGMENT, 7, 27, EKF_MODE_UPDATE, 0, 0, 3},
        {"position update (symmetrise)", 20, EKF_OP_POSITION, 3, 3, EKF_MODE_UPDATE, 0, 0, 0},
        {"zupt", 6, EKF_OP_ZUPT, 3, 6, EKF_MODE_UPDATE, 0, 0, 0},
        {"dense n=120 update (batch visual update)", 30, EKF_OP_DENSE, 120, 160, EKF_MODE_UPDATE, 0.02, 0, 0},
        {"dense n=13 check+update N=62 (odd sizes)", 6, EKF_OP_DENSE, 13, 41, EKF_MODE_CHECK_UPDATE, 0.02, 0, 0},
        {"gated chain link: gates open, late H, update", 20, EKF_OP_DENSE, 24, 97, EKF_MODE_UPDATE, 0.02, 0, 0, 1},
        {"gated chain link: gates open, check", 20, EKF_OP_DENSE, 24, 97, EKF_MODE_CHECK, 0.02, 0, 0, 1},
        {"gated off by the model flag", 20, EKF_OP_DENSE, 24, 97, EKF_MODE_CHECK, 0.02, 0, 0, 2},
        {"gated off by the success counter", 20, EKF_OP_DENSE, 24, 97, EKF_MODE_CHECK, 0.02, 0, 0, 3},
        {"update gated off by the check result", 20, EKF_OP_DENSE, 24, 97, EKF_MODE_UPDATE, 0.02, 0, 0, 4},
        {"two-R check+update n=24 (inlier)", 20, EKF_OP_DENSE, 24, 97, EKF_MODE_CHECK_UPDATE, 0.02, 0, 0, 0, 0.004},
        {"two-R check+update n=24 (outlier)", 20, EKF_OP_DENSE, 24, 97, EKF_MODE_CHECK_UPDATE, 40.0, 0, 0, 0, 0.004},
        {"two-R check+update n=84 l=160", 20, EKF_OP_DENSE, 84, 160, EKF_MODE_CHECK_UPDATE, 0.02, 0, 0, 0, 0.01},
        {"two-R check+update n=8 (one-stage S), gated", 20, EKF_OP_DENSE, 8, 34, EKF_MODE_CHECK_UPDATE, 0.02, 0, 0, 1, 0.2},
        {"two-R check+update n=13 N=62", 6, EKF_OP_DENSE, 13, 41, EKF_MODE_CHECK_UPDATE, 0.02, 0, 0, 0, 0.004},
        {"augment + deferred symmetrise into the second buffers", 20, EKF_OP_AUGMENT, 7, 27, EKF_MODE_UPDATE, 0, 1, -1, 0, 0.0, 1},
        {"augment drop 2 N=62 into the second buffers", 6, EKF_OP_AUGMENT, 7, 27, EKF_MODE_UPDATE, 0, 0, 2, 0, 0.0, 1},
        {"two-R check+update n=40 into the second buffers", 20, EKF_OP_DENSE, 40, 90, EKF_MODE_CHECK_UPDATE, 0.02, 0, 0, 0, 0.004, 1},
    };
    const int only = argc > 1 ? atoi(argv[1]) : -1;
    int fails = 0, idx = -1;
    for (const Case& cs : cases) {
        idx++;
        if (only >= 0 && idx != only) continue;
        srand(100 + idx);
        orc_params prm; orc_ekf_default_params(&prm);
        prm.camera_trail_length = cs.trail;
        orc_ekf* o = orc_ekf_create(&prm);
        const int N = orc_ekf_state_dim(o);
        const double noiseScale = prm.v[0] * prm.v[0];
        emu::Arena arena((size_t)64 << 20);
        double* m = arena.alloc<double>(N); double* P = arena.alloc<double>((size_t)N * N);
        double* H = arena.alloc<double>((size_t)cs.n * N); double* f = arena.alloc<double>(cs.n); double* y = arena.alloc<double>(cs.n);
        double* res = arena.alloc<double>(64);
        double* cwork = arena.alloc<double>((size_t)10 * N * N);
        {   // random SPD covariance (slightly asymmetric for the symmetrisation cases) and a plausible mean
            std::vector<double> Bm((size_t)N * N);
            for (auto& x : Bm) x = rnd();
            for (int i = 0; i < N; i++) for (int j = 0; j < N; j++) { double s = 0; for (int k = 0; k < N; k++) s += Bm[i + (size_t)k * N] * Bm[j + (size_t)k * N]; P[i + (size_t)j * N] = 0.05 * s + (i == j ? 0.5 : 0.0); }
            if (cs.symFirst || cs.op == EKF_OP_POSITION) for (int i = 0; i < N; i++) for (int j = 0; j < i; j++) P[i + (size_t)j * N] *= 1.0 + 1e-9 * rnd();
            for (int i = 0; i < N; i++) m[i] = 0.3 * rnd();
            for (int p = 0; p <= cs.trail; p++) {
                double* q = p == 0 ? m + EKF_ORI : m + EKF_CAM + EKF_POSE * (p - 1) + 3;
                double nn = 0; for (int i = 0; i < 4; i++) { q[i] = rnd() + (i == 0); nn += q[i] * q[i]; }
                for (int i = 0; i < 4; i++) q[i] /= std::sqrt(nn);
            }
        }
        orc_ekf_upload(o, m, P);
        if (cs.symFirst) orc_ekf_symmetrize(o);
        for (size_t i = 0; i < (size_t)cs.n * cs.l; i++) H[i] = 0.1 * gauss();
        for (int i = 0; i < cs.n; i++) { f[i] = 0.5 * gauss(); y[i] = f[i] + cs.yscale * gauss(); }

        EkfUpdateArgs a; memset(&a, 0, sizeof(a));
        a.b.m = m; a.b.P = P; a.b.res = res; a.b.cwork = cwork; a.b.N = N; a.b.trail = cs.trail; a.b.mapDim = 0;
        a.op = cs.op; a.n = cs.n; a.l = cs.l; a.mode = cs.mode; a.noiseScale = noiseScale; a.rmseThr = -1.0;
        int ost = 0; double ochi2 = 0;
        const double r = 0.05;
        int* gflag = arena.alloc<int>(4); double* gslot = arena.alloc<double>(8);      // [0] model flag, [1] counter; slots: [0..2] of this kernel, [4] the check result it is gated on
        gflag[0] = 0; gflag[1] = 2; gslot[0] = gslot[1] = gslot[2] = -7.0; gslot[4] = 0.0;
        const bool gatedOff = cs.gate >= 2;
        if (cs.gate) {
            a.gateI = &gflag[0]; a.gateIExpect = 0; a.counter = &gflag[1]; a.counterMax = 5; a.gateD = &gslot[4]; a.gateDExpect = 0.0;
            a.bump = &gflag[1]; a.slot = gslot; a.lateH = 1;
            if (cs.gate == 2) gflag[0] = 3;            // the model kernel reported a failure
            if (cs.gate == 3) gflag[1] = 5;            // enough successful updates already
            if (cs.gate == 4) gslot[4] = 3.0;          // the check said CHI2 outlier
        }
        if (cs.op == EKF_OP_DENSE) {
            a.H = H; a.f = f; a.y = y; a.Rdiag = r * r * noiseScale; a.normalizeAll = 1;
            a.chi2Thr = cs.mode == EKF_MODE_UPDATE ? 0.0 : orc_chi2inv95(cs.n);
            if (gatedOff) ost = 1;                     // NOT_COMPUTED, filter untouched
            else {
                if (cs.mode != EKF_MODE_UPDATE) ost = orc_ekf_visual_check(o, H, cs.n, cs.l, f, y, r, -1.0, &ochi2);
                if (cs.mode == EKF_MODE_UPDATE || (cs.mode == EKF_MODE_CHECK_UPDATE && ost == 0)) orc_ekf_visual_update(o, H, cs.n, cs.l, f, y, cs.r2 > 0 ? cs.r2 : r);
            }
            if (cs.r2 > 0) a.Rdiag2 = cs.r2 * cs.r2 * noiseScale;
        } else if (cs.op == EKF_OP_AUGMENT) {
            const int drop = cs.drop == -1 ? cs.trail - 1 : cs.drop;
            a.Rdiag = prm.v[17] * noiseScale; a.dropIdx = drop; a.symFirst = cs.symFirst;
            a.augNoisePos = prm.v[9] * prm.v[9] * noiseScale; a.augNoiseOri = prm.v[10] * prm.v[10] * noiseScale;
            a.normalizeAll = 1; a.symmetrize = 1;
            orc_ekf_augment(o, drop);
        } else if (cs.op == EKF_OP_POSITION) {
            const double yy[3] = {0.1, -0.2, 0.05};
            a.Rdiag = 1e-3 * noiseScale; for (int i = 0; i < 3; i++) a.ysmall[i] = yy[i];
            a.symmetrize = 1;
            orc_ekf_update_position(o, yy, 1e-3);
        } else if (cs.op == EKF_OP_ZUPT) {
            a.Rdiag = 1e-2 * noiseScale;
            orc_ekf_update_zupt(o, 1e-2);
        }
        const size_t smem = ek2_smem_bytes(cs.n, cs.l, N, cs.op == EKF_OP_AUGMENT);
        double* P2 = nullptr; double* m2 = nullptr;
        std::vector<double> P0, m0;
        if (cs.second) {
            P2 = arena.alloc<double>((size_t)N * N); m2 = arena.alloc<double>(N);
            for (size_t i = 0; i < (size_t)N * N; i++) P2[i] = -3.0;
            for (int i = 0; i < N; i++) m2[i] = -3.0;
            a.specP = P2; a.specM = m2;
            P0.assign(P, P + (size_t)N * N); m0.assign(m, m + N);
        }
        int bad = EMU_LAUNCH_CLUSTER(arena, EK2_C, EK2_NT, smem, emu_update_body, &a);
        if (cs.second) {                                                   // the first buffers must be untouched; compare the second ones
            if (memcmp(P0.data(), P, sizeof(double) * (size_t)N * N) != 0 || memcmp(m0.data(), m, sizeof(double) * N) != 0) bad |= 64;
            P = P2; m = m2;
        }
        std::vector<double> om(N), oP((size_t)N * N);
        orc_ekf_download(o, om.data(), oP.data());
        double em = 0, eP = 0, pmax = 0, asym = 0;
        for (int i = 0; i < N; i++) em = std::fmax(em, std::fabs(om[i] - m[i]));
        for (size_t i = 0; i < oP.size(); i++) { eP = std::fmax(eP, std::fabs(oP[i] - P[i])); pmax = std::fmax(pmax, std::fabs(oP[i])); }
        if (a.symmetrize) for (int i = 0; i < N; i++) for (int j = 0; j < i; j++) asym = std::fmax(asym, std::fabs(P[i + (size_t)j * N] - P[j + (size_t)i * N]));
        bool ok = bad == 0 && em < 1e-9 && eP / pmax < 1e-9 && asym == 0.0;
        if (cs.op == EKF_OP_DENSE && (cs.mode != EKF_MODE_UPDATE || gatedOff)) ok = ok && (int)res[0] == ost && std::fabs(res[1] - ochi2) <= 1e-9 * std::fmax(1.0, std::fabs(ochi2));
        if (cs.gate) {
            ok = ok && gslot[0] == res[0] && gslot[1] == res[1] && gslot[2] == res[2];                     // the slot mirrors the result words
            const int expectCounter = (cs.gate == 3 ? 5 : 2) + ((cs.gate == 1 && (cs.mode == EKF_MODE_UPDATE || (cs.mode == EKF_MODE_CHECK_UPDATE && ost == 0))) ? 1 : 0);
            ok = ok && gflag[1] == expectCounter;                                                          // bumped only by an applied update
        }
        printf("[%2d] %-42s N=%3d smem %6.1f KB: status %d/%d chi2 %.6g/%.6g  max|dm| %.2e  max|dP|/max|P| %.2e  %s\n", idx, cs.name, N, smem / 1024.0,
               (int)res[0], ost, res[1], ochi2, em, eP / pmax, ok ? "ok" : "FAIL");
        fflush(stdout);
        fails += !ok;
        orc_ekf_destroy(o);
        munmap(arena.base, arena.size);
    }
    return fails;
}
#endif  // EMU_AS_LIB
