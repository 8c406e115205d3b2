// tests/emu/emu_update_chunked.cpp -- the row-chunked form of the cluster update (EkfUpdateArgs::rowChunk, ekf_cluster2.cuh) on the
// host emulator: the REAL ek2_body with chunk heights chosen here, against the C oracle's visualTrackOutlierCheck / updateVisualTrack
// on states the size of long trails and hybrid maps (N = 202 .. 400). Covers chunk heights 8 / 16 / n - 8 and heights that do not
// divide n, check / update / check+update with one and with two noise levels, the device-side gates of the visual-update chain, and
// an innovation covariance that is positive definite in the first chunk only (the numeric flag, nothing written back).
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
}

#if !defined(EMU_CLUSTER_THREADS) || defined(EMU_AS_LIB)
EMU_CLUSTER_BODY(emu_chunked_body) { EkfUpdateArgs aa = *(const EkfUpdateArgs*)ctx; ek2_body(aa, dyn, cg::this_cluster()); }
#endif
#ifndef EMU_AS_LIB

static double rnd() { return rand() / (double)RAND_MAX - 0.5; }
static double gauss() { double s = 0; for (int i = 0; i < 12; i++) s += rand() / (double)RAND_MAX; return s - 6.0; }

// gate: 0 none; 1 device-side gates present and satisfied (+ lateH, slot, bump); 2 gated off by the model flag
// r2 > 0: the update uses its own noise level (two-R check+update); indefinite: S is positive definite on the first chunk's rows only
struct Case { const char* name; int trail, map, n, l, mode, chunk; double yscale; double r2 = 0.0; int gate = 0; int indefinite = 0; };

int main(int argc, char** argv)
{
    const Case cases[] = {
        {"update n=84 chunk 8 N=301", 20, 47, 84, 160, EKF_MODE_UPDATE, 8, 0.02},
        {"update n=84 chunk 16 N=301", 20, 47, 84, 160, EKF_MODE_UPDATE, 16, 0.02},
        {"update n=84 chunk n-8 N=301", 20, 47, 84, 160, EKF_MODE_UPDATE, 76, 0.02},
        {"update n=84 chunk 40 (40+40+4) N=400", 20, 80, 84, 160, EKF_MODE_UPDATE, 40, 0.02},
        {"update n=60 chunk 41 (41+19) N=230", 30, 0, 60, 230, EKF_MODE_UPDATE, 41, 0.02},
        {"check n=84 chunk 16 (inlier) N=301", 20, 47, 84, 160, EKF_MODE_CHECK, 16, 0.02},
        {"check n=84 chunk 16 (outlier) N=301", 20, 47, 84, 160, EKF_MODE_CHECK, 16, 40.0},
        {"check+update n=72 chunk 24 N=202", 20, 14, 72, 160, EKF_MODE_CHECK_UPDATE, 24, 0.02},
        {"two-R check+update n=84 chunk 16 N=301", 20, 47, 84, 160, EKF_MODE_CHECK_UPDATE, 16, 0.02, 0.004},
        {"two-R check+update n=84 chunk 16 (outlier)", 20, 47, 84, 160, EKF_MODE_CHECK_UPDATE, 16, 40.0, 0.004},
        {"two-R check+update n=44 chunk 8 N=400, gated", 20, 80, 44, 160, EKF_MODE_CHECK_UPDATE, 8, 0.02, 0.004, 1},
        {"check n=44 chunk 8 N=400, gated off", 20, 80, 44, 160, EKF_MODE_CHECK, 8, 0.02, 0.0, 2},
        {"one chunk (rowChunk = n) n=20 N=202", 20, 14, 20, 97, EKF_MODE_CHECK_UPDATE, 20, 0.02, 0.004},
        {"S indefinite in chunk 2 only: update", 20, 47, 48, 160, EKF_MODE_UPDATE, 24, 0.02, 0.0, 0, 1},
        {"S indefinite in chunk 2 only: two-R", 20, 47, 48, 160, EKF_MODE_CHECK_UPDATE, 24, 0.02, 0.004, 0, 1},
    };
    const int only = argc > 1 ? atoi(argv[1]) : -1;
    int fails = 0, idx = -1;
    for (const Case& cs : cases) {
        idx++;
        if (only >= 0 && idx != only) continue;
        srand(300 + idx);
        orc_params prm; orc_ekf_default_params(&prm);
        prm.camera_trail_length = cs.trail; prm.hybrid_map_size = cs.map;
        orc_ekf* o = orc_ekf_create(&prm);
        const int N = orc_ekf_state_dim(o);
        const double noiseScale = prm.v[0] * prm.v[0];
        emu::Arena arena((size_t)96 << 20);
        double* m = arena.alloc<double>(N); double* P = arena.alloc<double>((size_t)N * N);
        double* H = arena.alloc<double>((size_t)cs.n * cs.l); double* f = arena.alloc<double>(cs.n); double* y = arena.alloc<double>(cs.n);
        double* res = arena.alloc<double>(64);
        double* cwork = arena.alloc<double>((size_t)10 * N * N);
        const int split = cs.l / 2;                                        // indefinite: chunk 1 sees columns [0, split), chunk 2 the rest
        {   // random SPD covariance and a plausible mean
            std::vector<double> Bm((size_t)N * N);
            for (auto& x : Bm) x = rnd();
            for (int i = 0; i < N; i++) for (int j = 0; j < N; j++) { double s = 0; for (int k = 0; k < N; k++) s += Bm[i + (size_t)k * N] * Bm[j + (size_t)k * N]; P[i + (size_t)j * N] = 0.05 * s / N * 8 + (i == j ? 0.5 : 0.0); }
            if (cs.indefinite) for (int i = split; i < cs.l; i++) P[i + (size_t)i * N] -= 50.0;
            for (int i = 0; i < N; i++) m[i] = 0.3 * rnd();
            for (int p = 0; p <= cs.trail; p++) {
                double* q = p == 0 ? m + EKF_ORI : m + EKF_CAM + EKF_POSE * (p - 1) + 3;
                double nn = 0; for (int i = 0; i < 4; i++) { q[i] = rnd() + (i == 0); nn += q[i] * q[i]; }
                for (int i = 0; i < 4; i++) q[i] /= std::sqrt(nn);
            }
        }
        orc_ekf_upload(o, m, P);
        for (int k = 0; k < cs.l; k++) for (int i = 0; i < cs.n; i++) {
            double h = 0.1 * gauss();
            if (cs.indefinite && ((i < cs.chunk) != (k < split))) h = 0.0;
            H[i + (size_t)k * cs.n] = h;
        }
        for (int i = 0; i < cs.n; i++) { f[i] = 0.5 * gauss(); y[i] = f[i] + cs.yscale * gauss(); }
        const std::vector<double> P0(P, P + (size_t)N * N), m0(m, m + N);

        EkfUpdateArgs a; memset(&a, 0, sizeof(a));
        a.b.m = m; a.b.P = P; a.b.res = res; a.b.cwork = cwork; a.b.N = N; a.b.trail = cs.trail; a.b.mapDim = 3 * cs.map;
        a.op = EKF_OP_DENSE; a.n = cs.n; a.l = cs.l; a.mode = cs.mode; a.noiseScale = noiseScale; a.rmseThr = -1.0; a.normalizeAll = 1;
        a.H = H; a.f = f; a.y = y; a.rowChunk = cs.chunk;
        const double r = 0.05;
        a.Rdiag = r * r * noiseScale; a.chi2Thr = cs.mode == EKF_MODE_UPDATE ? 0.0 : orc_chi2inv95(cs.n);
        if (cs.r2 > 0) a.Rdiag2 = cs.r2 * cs.r2 * noiseScale;
        int* gflag = arena.alloc<int>(4); double* gslot = arena.alloc<double>(8);      // [0] model flag, [1] counter
        gflag[0] = 0; gflag[1] = 2; gslot[0] = gslot[1] = gslot[2] = -7.0;
        if (cs.gate) {
            a.gateI = &gflag[0]; a.gateIExpect = 0; a.counter = &gflag[1]; a.counterMax = 5; a.bump = &gflag[1]; a.slot = gslot; a.lateH = 1;
            if (cs.gate == 2) gflag[0] = 3;            // the model kernel reported a failure
        }
        // the oracle: NOT_COMPUTED when gated off; numeric failure expected (and nothing to compare) for the indefinite cases
        int ost = 0; double ochi2 = 0;
        bool applied = false;
        if (cs.gate == 2) ost = 1;
        else if (!cs.indefinite) {
            if (cs.mode != EKF_MODE_UPDATE) ost = orc_ekf_visual_check(o, H, cs.n, cs.l, f, y, r, -1.0, &ochi2);
            if (cs.mode == EKF_MODE_UPDATE || (cs.mode == EKF_MODE_CHECK_UPDATE && ost == 0)) {
                orc_ekf_visual_update(o, H, cs.n, cs.l, f, y, cs.r2 > 0 ? cs.r2 : r);
                applied = true;
            }
        }
        const size_t smem = ek2_smem_bytes_chunked(std::min(cs.chunk, cs.n), cs.n, cs.l, N);
        const int bad = EMU_LAUNCH_CLUSTER(arena, EK2_C, EK2_NT, smem, emu_chunked_body, &a);
        bool ok = bad == 0;
        double em = 0, eP = 0, pmax = 0, ec = 0;
        if (cs.indefinite) {                           // non-positive pivot in the second chunk: flag set, (m, P) bit-identical
            ok = ok && res[0] == 1.0 && res[2] == 1.0;
            ok = ok && memcmp(P0.data(), P, sizeof(double) * (size_t)N * N) == 0 && memcmp(m0.data(), m, sizeof(double) * N) == 0;
        } else {
            std::vector<double> om(N), oP((size_t)N * N);
            orc_ekf_download(o, om.data(), oP.data());
            for (int i = 0; i < N; i++) em = std::fmax(em, std::fabs(om[i] - m[i]));
            for (size_t i = 0; i < oP.size(); i++) { eP = std::fmax(eP, std::fabs(oP[i] - P[i])); pmax = std::fmax(pmax, std::fabs(oP[i])); }
            ok = ok && em <= 1e-9 && eP / pmax <= 1e-9 && res[2] == 0.0;
            if (!applied) ok = ok && memcmp(P0.data(), P, sizeof(double) * (size_t)N * N) == 0 && memcmp(m0.data(), m, sizeof(double) * N) == 0;
            if (cs.mode != EKF_MODE_UPDATE || cs.gate == 2) {
                ec = std::fabs(res[1] - ochi2) / std::fmax(1.0, std::fabs(ochi2));
                ok = ok && (int)res[0] == ost && ec <= 1e-8;
            }
        }
        if (cs.gate) {
            ok = ok && gslot[0] == res[0] && gslot[1] == res[1] && gslot[2] == res[2];
            ok = ok && gflag[1] == 2 + (applied ? 1 : 0);                 // bumped only by an applied update
        }
        printf("[%2d] %-46s N=%3d chunk %2d smem %6.1f KB: status %d/%d chi2 %.6g/%.6g (rel %.1e)  max|dm| %.2e  max|dP|/max|P| %.2e  %s\n", idx, cs.name, N,
               cs.chunk, smem / 1024.0, (int)res[0], ost, res[1], ochi2, ec, em, pmax > 0 ? eP / pmax : 0.0, ok ? "ok" : "FAIL");
        fflush(stdout);
        fails += !ok;
        orc_ekf_destroy(o);
        munmap(arena.base, arena.size);
    }
    return fails;
}
#endif  // EMU_AS_LIB
