// tests/emu/emu_chain.cpp -- the device side of hv_ekf_visual_tracks on the host emulator: for a list of tracks, in order,
//   tm_body (one CTA, counter gate)  ->  ek2_body check (gated by the model's status word and the success counter, H staged late)
//   ->  ek2_body update (gated by the check's result word, bumps the counter),
// all kernels talking through words in "global memory" (a shared mapping) exactly as the chain on the GPU does, and compares the
// decisions and the final filter state with the same loop driven track by track through the C oracles
// (oracle/hv_oracle_tri.c, oracle/hv_oracle_ekf.c). Test infrastructure.
#include <algorithm>
#include "emu_cluster.h"
#include "ekf_cluster2.cuh"
#include "track_model.cuh"
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
int orc_track_model(const double* m, int trail, int useStereo, const int* poseTrailIndex, int npose, const double* imuToCam,
                    const double* imuToCam2, const double* ip, const double* vel, int estimateTimeShift, int* triStatus, double* pf,
                    double* dpf, double* depth, int* vuStatus, int* rows, int* cols, double* H, double* f);
}

#if !defined(EMU_CLUSTER_THREADS) || defined(EMU_AS_LIB)
EMU_CLUSTER_BODY(emu_chain_update_body) { EkfUpdateArgs aa = *(const EkfUpdateArgs*)ctx; ek2_body(aa, dyn, cg::this_cluster()); }
#endif
#ifndef EMU_AS_LIB

static double urand() { return rand() / (double)RAND_MAX; }
static double nrand() { double s = 0; for (int i = 0; i < 12; i++) s += urand(); return s - 6.0; }

int main(int argc, char**)
{
    const bool fused = argc > 1;        // any argument: check and update of a track in ONE kernel (two noise levels)
    srand(77);
    const int trail = 20, N = 20 + 7 * trail, ntracks = 9, maxSucc = 3, stereo = 1;
    const double chiR = 0.01, visR = 0.004;
    orc_params prm; orc_ekf_default_params(&prm); prm.camera_trail_length = trail;
    orc_ekf* o = orc_ekf_create(&prm);
    const double noiseScale = prm.v[0] * prm.v[0];
    emu::Arena arena((size_t)96 << 20);
    double* m = arena.alloc<double>(N); double* P = arena.alloc<double>((size_t)N * N);
    double* res = arena.alloc<double>(64); double* cwork = arena.alloc<double>((size_t)10 * N * N);
    // state: a smooth path (as tests/tri_common.py), small SPD covariance
    for (int i = 0; i < N; i++) m[i] = 0.0;
    for (int k = 0; k <= trail; k++) {
        const int ob = k == 0 ? 0 : 20 + 7 * (k - 1);
        m[ob] = 0.08 * k + 0.005 * nrand(); m[ob + 1] = 0.02 * std::sin(0.7 * k) + 0.005 * nrand(); m[ob + 2] = 0.01 * k + 0.005 * nrand();
        double q[4] = {1.0, 0.01 * k + 0.0015 * nrand(), -0.0075 * k + 0.0015 * nrand(), 0.005 * std::sin((double)k)};
        const double qn = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
        for (int r = 0; r < 4; r++) m[(k == 0 ? 6 : ob + 3) + r] = q[r] / qn;
    }
    for (int r = 0; r < 3; r++) m[16 + r] = 1.0;
    {
        std::vector<double> Bm((size_t)N * N);
        for (auto& x : Bm) x = urand() - 0.5;
        for (int i = 0; i < N; i++) for (int j = 0; j < N; j++) { double s = 0; for (int k = 0; k < N; k++) s += Bm[i + (size_t)k * N] * Bm[j + (size_t)k * N]; P[i + (size_t)j * N] = 1e-4 * s / N + (i == j ? 1e-4 : 0.0); }
    }
    orc_ekf_upload(o, m, P);
    double T1[16] = {0}, T2[16];
    { const double qc[4] = {0.9998, 0.01, -0.012, 0.008}; double R[9]; tm_quat_mat(qc, -1, R); for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) T1[4 * c + r] = R[3 * r + c]; }
    T1[12] = 0.01; T1[13] = -0.02; T1[14] = 0.005; T1[15] = 1.0;
    memcpy(T2, T1, sizeof(T1)); T2[12] -= 0.11;
    // packed batch (the layout of TmArgs)
    int* npose = arena.alloc<int>(ntracks); int* idx = arena.alloc<int>(ntracks * TM_MAXPOSE);
    double* ip = arena.alloc<double>(ntracks * TM_MAXOBS * 2); double* vel = arena.alloc<double>(ntracks * TM_MAXOBS * 2);
    int* status = arena.alloc<int>(4 * ntracks); double* pf = arena.alloc<double>(4 * ntracks);
    const size_t Hs = (size_t)2 * TM_MAXOBS * TM_MAXN;
    double* H = arena.alloc<double>(ntracks * Hs); double* f = arena.alloc<double>(ntracks * 2 * TM_MAXOBS);
    int* counter = arena.alloc<int>(4); double* slots = arena.alloc<double>(8 * ntracks);
    counter[0] = 0;
    auto camOf = [&](int i, const double* T, double* pc, double* R) {
        const int ob = i == 0 ? 0 : 20 + 7 * (i - 1);
        double Rq[9]; tm_quat_mat(&m[i == 0 ? 6 : ob + 3], -1, Rq);
        for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) { double v = 0; for (int k = 0; k < 3; k++) v += T[4 * k + r] * Rq[3 * k + c]; R[3 * r + c] = v; }
        for (int r = 0; r < 3; r++) pc[r] = m[ob + r] - (R[r] * T[12] + R[3 + r] * T[13] + R[6 + r] * T[14]);
    };
    for (int t = 0; t < ntracks; t++) {
        const int np = 4 + (t * 5) % 7;
        npose[t] = np;
        std::vector<int> pool; for (int k = 1; k <= trail; k++) pool.push_back(k);
        for (int k = 0; k < np - 1; k++) std::swap(pool[k], pool[k + rand() % (int)(pool.size() - k)]);
        std::sort(pool.begin(), pool.begin() + np - 1);
        idx[t * TM_MAXPOSE] = 0; for (int k = 0; k < np - 1; k++) idx[t * TM_MAXPOSE + 1 + k] = pool[k];
        double p0[3], R0[9]; camOf(0, T1, p0, R0);
        const double depth = 3.0 + t % 4, loc[3] = {(urand() * 0.6 - 0.3) * depth, (urand() * 0.4 - 0.2) * depth, depth};
        double X[3]; for (int r = 0; r < 3; r++) X[r] = p0[r] + R0[r] * loc[0] + R0[3 + r] * loc[1] + R0[6 + r] * loc[2];
        int ob = 0;
        for (int c = 0; c < 2; c++) for (int k = 0; k < np; k++, ob++) {
            double pc[3], R[9], d[3], x[3]; camOf(idx[t * TM_MAXPOSE + k], c ? T2 : T1, pc, R);
            for (int r = 0; r < 3; r++) d[r] = X[r] - pc[r];
            tm_mv(R, d, x);
            double u = x[0] / x[2] + 2e-3 * nrand(), v = x[1] / x[2] + 2e-3 * nrand();
            if (t % 4 == 1 && ob == 1) { u += 0.08; v -= 0.06; }          // gross outlier -> chi2
            if (t % 5 == 3) { u = -u; v = -v; }                           // behind the cameras -> no model
            ip[(t * TM_MAXOBS + ob) * 2] = u; ip[(t * TM_MAXOBS + ob) * 2 + 1] = v;
            vel[(t * TM_MAXOBS + ob) * 2] = 0.05 * nrand(); vel[(t * TM_MAXOBS + ob) * 2 + 1] = 0.05 * nrand();
        }
    }
    // ---- oracle loop
    std::vector<int> eTri(ntracks, -1), eOut(ntracks, 1), eUpd(ntracks, 0);
    int succ = 0;
    {
        std::vector<double> om(N), oP((size_t)N * N), oH((size_t)2 * TM_MAXOBS * N), of(2 * TM_MAXOBS), odpf(3 * (7 * TM_MAXPOSE + 1));
        for (int t = 0; t < ntracks; t++) {
            if (succ >= maxSucc) continue;
            orc_ekf_download(o, om.data(), oP.data());
            int tri, vu, rows, cols; double opf[3], depth;
            orc_track_model(om.data(), trail, stereo, idx + t * TM_MAXPOSE, npose[t], T1, T2, ip + t * TM_MAXOBS * 2, vel + t * TM_MAXOBS * 2, 1, &tri, opf, odpf.data(), &depth, &vu,
                            &rows, &cols, oH.data(), of.data());
            eTri[t] = tri;
            if (tri == 0 && vu == 0) {
                double chi2 = 0;
                eOut[t] = orc_ekf_visual_check(o, oH.data(), rows, cols, of.data(), ip + t * TM_MAXOBS * 2, chiR, -1.0, &chi2);
                if (eOut[t] == 0) { orc_ekf_visual_update(o, oH.data(), rows, cols, of.data(), ip + t * TM_MAXOBS * 2, visR); eUpd[t] = 1; succ++; }
            }
        }
    }
    // ---- the chain on the emulator
    TmArgs ta; memset(&ta, 0, sizeof(ta));
    ta.m = m; ta.N = N; ta.stereo = stereo; ta.timeShift = 1; ta.ntracks = 1;
    for (int c = 0; c < 2; c++) { const double* T = c ? T2 : T1; for (int r = 0; r < 3; r++) { for (int k = 0; k < 3; k++) ta.Rc[c][3 * r + k] = T[4 * k + r]; ta.base[c][r] = T[12 + r]; } }
    ta.gnIterations = 10; ta.convThreshold = 1e-2; ta.convR = 11.0; ta.rcondThreshold = 1e-8; ta.minDist = 0; ta.maxDist = 1e300;
    ta.npose = npose; ta.idx = idx; ta.ip = ip; ta.vel = vel; ta.status = status; ta.pf = pf; ta.dpf = nullptr; ta.H = H; ta.f = f; ta.Hstride = Hs;
    ta.counter = counter; ta.counterMax = maxSucc;
    std::vector<double> tmDyn(tm_smem_bytes() / 8, std::nan(""));
    int fails = 0;

    for (int t = 0; t < ntracks; t++) {
        TmArgs a1 = ta; a1.trackOffset = t;
        gridDim.x = 1;
        emu::launch_cta(TM_NT, 0, [&] { tm_body(a1, tmDyn.data()); });
        const int n = 2 * npose[t] * 2;
        int l = 0; for (int k = 0; k < npose[t]; k++) { const int x = idx[t * TM_MAXPOSE + k]; l = std::max(l, x == 0 ? 10 : 20 + 7 * (x - 1) + 7); }
        EkfUpdateArgs c; memset(&c, 0, sizeof(c));
        c.b.m = m; c.b.P = P; c.b.res = res; c.b.cwork = cwork; c.b.N = N; c.b.trail = trail;
        c.op = EKF_OP_DENSE; c.n = n; c.l = l; c.mode = EKF_MODE_CHECK; c.noiseScale = noiseScale; c.rmseThr = -1.0; c.normalizeAll = 1;
        c.H = H + t * Hs; c.f = f + t * 2 * TM_MAXOBS; c.y = ip + t * TM_MAXOBS * 2;
        c.Rdiag = chiR * chiR * noiseScale; c.chi2Thr = orc_chi2inv95(n);
        c.gateI = status + 4 * t + 1; c.gateIExpect = 0; c.counter = counter; c.counterMax = maxSucc; c.slot = slots + 8 * t; c.lateH = 1;
        const size_t smem = ek2_smem_bytes(n, l, N, false);
        if (fused) { c.mode = EKF_MODE_CHECK_UPDATE; c.Rdiag2 = visR * visR * noiseScale; c.bump = counter; }
        int bad = EMU_LAUNCH_CLUSTER(arena, EK2_C, EK2_NT, smem, emu_chain_update_body, &c);
        if (!fused) {
            EkfUpdateArgs u = c;
            u.mode = EKF_MODE_UPDATE; u.Rdiag = visR * visR * noiseScale; u.chi2Thr = 0.0;
            u.gateI = nullptr; u.counter = nullptr; u.gateD = slots + 8 * t; u.gateDExpect = 0.0; u.bump = counter; u.slot = slots + 8 * t + 4;
            bad += EMU_LAUNCH_CLUSTER(arena, EK2_C, EK2_NT, smem, emu_chain_update_body, &u);
        } else {
            slots[8 * t + 4] = (slots[8 * t] == 0.0 && slots[8 * t + 2] == 0.0) ? 0.0 : 1.0;      // "updated" as the host derives it in fused mode
        }
        const int gTri = status[4 * t], gOut = (int)slots[8 * t], gUpd = slots[8 * t + 4] == 0.0 ? 1 : 0;
        const bool ok = bad == 0 && gTri == eTri[t] && gOut == eOut[t] && gUpd == eUpd[t];
        printf("track %d (n=%2d l=%3d): model %2d/%2d  check %d/%d  updated %d/%d  counter %d  %s\n", t, n, l, gTri, eTri[t], gOut, eOut[t], gUpd, eUpd[t], counter[0], ok ? "ok" : "FAIL");
        fflush(stdout);
        fails += !ok;
    }
    std::vector<double> om(N), oP((size_t)N * N);
    orc_ekf_download(o, om.data(), oP.data());
    double em = 0, eP = 0, pmax = 0;
    for (int i = 0; i < N; i++) em = std::fmax(em, std::fabs(om[i] - m[i]));
    for (size_t i = 0; i < oP.size(); i++) { eP = std::fmax(eP, std::fabs(oP[i] - P[i])); pmax = std::fmax(pmax, std::fabs(oP[i])); }
    const bool ok = counter[0] == succ && succ == maxSucc && em < 1e-9 && eP / pmax < 1e-9;
    printf("chain%s: %d updates (oracle %d)  max|dm| %.2e  max|dP|/max|P| %.2e  %s\n", fused ? " (fused check+update)" : "", counter[0], succ, em, eP / pmax, ok ? "ok" : "FAIL");
    fails += !ok;
    orc_ekf_destroy(o);
    return fails;
}
#endif  // EMU_AS_LIB
