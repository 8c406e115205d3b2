// tests/emu/emu_group_tracks.cpp -- runs the body of the group model kernel (tm_group_body, hybvio_b200/csrc/track_model.cuh) on the
// host emulator: three CTAs of one launch, each on its own argument block (the layout hv_ekf_group_visual_tracks gives a chain step:
// one track of each filter's packed batch) -- different state means, a mono filter and two stereo ones, different tracks, the third
// filter gated off by its success counter -- and compares every output bit for bit with the per-filter body (tm_body, CTA 0 of a
// one-track launch at the same track offset): statuses, pf and depth, d pf, H, f; the other tracks' outputs stay untouched.
//   g++ -std=c++20 -O1 -pthread -Itests/emu/stubs -Itests/emu -Ihybvio_b200/csrc tests/emu/emu_group_tracks.cpp -o build/emu_group_tracks
#include <algorithm>
#include "cuda_emu.h"
#include "track_model.cuh"

static double urand() { return rand() / (double)RAND_MAX; }
static double nrand() { double s = 0; for (int i = 0; i < 12; i++) s += urand(); return s - 6.0; }

static const int TRAIL = 6, N = 20 + 7 * TRAIL, T = 3, TRK = 1;      // N = 62 (config 4); the step issues track 1 of each batch
static const size_t HS = (size_t)2 * TM_MAXOBS * TM_MAXN, DPS = 3 * (7 * TM_MAXPOSE + 1);

// One filter: its state mean, rig, a batch of T tracks and the output buffers of the batch
struct Filter {
    std::vector<double> m, ip, vel, pf, dpf, H, f;
    std::vector<int> npose, idx, st;
    double T1[16], T2[16];
    int stereo, counter;
};

// the construction of tests/tri_common.py: a smooth path, a rig, per track one point projected into every observing camera pose
static void make_filter(Filter& F, int seed, int stereo, int counter)
{
    srand(500 + seed);
    F.stereo = stereo; F.counter = counter;
    F.m.assign(N, 0.0);
    for (int k = 0; k <= TRAIL; k++) {
        double ang[3] = {0.02 * k + 0.003 * nrand(), -0.015 * k + 0.003 * nrand(), 0.01 * std::sin((double)k) + 0.003 * nrand()};
        double q[4] = {1.0, 0.5 * ang[0], 0.5 * ang[1], 0.5 * ang[2]};
        const double qn = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
        const int o = k == 0 ? 0 : 20 + 7 * (k - 1);
        F.m[o] = 0.08 * k + 0.005 * nrand(); F.m[o + 1] = 0.02 * std::sin(0.7 * k) + 0.005 * nrand(); F.m[o + 2] = 0.01 * k + 0.005 * nrand();
        for (int r = 0; r < 4; r++) F.m[(k == 0 ? 6 : o + 3) + r] = q[r] / qn;
    }
    for (int r = 0; r < 3; r++) { F.m[3 + r] = 0.1 * nrand(); F.m[16 + r] = 1.0; }
    double qc[4] = {1.0, 0.01 * nrand(), 0.01 * nrand(), 0.01 * nrand()};
    const double qn = std::sqrt(qc[0] * qc[0] + qc[1] * qc[1] + qc[2] * qc[2] + qc[3] * qc[3]);
    for (double& x : qc) x /= qn;
    double Rc[9]; tm_quat_mat(qc, -1, Rc);
    memset(F.T1, 0, sizeof(F.T1));
    for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) F.T1[4 * c + r] = Rc[3 * r + c];
    F.T1[12] = 0.01; F.T1[13] = -0.02; F.T1[14] = 0.005; F.T1[15] = 1.0;
    memcpy(F.T2, F.T1, sizeof(F.T1)); F.T2[12] -= 0.11;
    F.npose.assign(T, 0); F.idx.assign(T * TM_MAXPOSE, 0);
    F.ip.assign(T * TM_MAXOBS * 2, 0.0); F.vel.assign(T * TM_MAXOBS * 2, 0.0);
    auto cam = [&](int i, const double* Tm, double* pc, double* R) {
        const int o = i == 0 ? 0 : 20 + 7 * (i - 1);
        double Rq[9]; tm_quat_mat(&F.m[i == 0 ? 6 : o + 3], -1, Rq);
        for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) { double v = 0; for (int k = 0; k < 3; k++) v += Tm[4 * k + r] * Rq[3 * k + c]; R[3 * r + c] = v; }
        for (int r = 0; r < 3; r++) pc[r] = F.m[o + r] - (R[r] * Tm[12] + R[3 + r] * Tm[13] + R[6 + r] * Tm[14]);
    };
    for (int t = 0; t < T; t++) {
        const int np = 3 + (seed + 2 * t) % (TRAIL - 1);                  // 3..7 poses: 0 and np - 1 distinct trail slots
        std::vector<int> pool; for (int k = 1; k <= TRAIL; k++) pool.push_back(k);
        for (int k = 0; k < np - 1; k++) std::swap(pool[k], pool[k + rand() % (int)(pool.size() - k)]);
        std::sort(pool.begin(), pool.begin() + np - 1);
        F.npose[t] = np; F.idx[t * TM_MAXPOSE] = 0;
        for (int k = 1; k < np; k++) F.idx[t * TM_MAXPOSE + k] = pool[k - 1];
        double p0[3], R0[9]; cam(0, F.T1, p0, R0);
        const double depth = 3.0 + 4.0 * urand(), local[3] = {(urand() * 0.6 - 0.3) * depth, (urand() * 0.4 - 0.2) * depth, depth};
        double pf[3]; for (int r = 0; r < 3; r++) pf[r] = p0[r] + R0[r] * local[0] + R0[3 + r] * local[1] + R0[6 + r] * local[2];
        int o = 0;
        for (int c = 0; c < (stereo ? 2 : 1); c++) for (int k = 0; k < np; k++) {
            double pc[3], R[9], d[3], x[3]; cam(F.idx[t * TM_MAXPOSE + k], c ? F.T2 : F.T1, pc, R);
            for (int r = 0; r < 3; r++) d[r] = pf[r] - pc[r];
            tm_mv(R, d, x);
            F.ip[t * TM_MAXOBS * 2 + 2 * o] = x[0] / x[2] + 2e-3 * nrand(); F.ip[t * TM_MAXOBS * 2 + 2 * o + 1] = x[1] / x[2] + 2e-3 * nrand();
            F.vel[t * TM_MAXOBS * 2 + 2 * o] = 0.05 * nrand(); F.vel[t * TM_MAXOBS * 2 + 2 * o + 1] = 0.05 * nrand();
            o++;
        }
    }
}

static void reset_outputs(Filter& F)
{
    F.st.assign(4 * T, -7); F.pf.assign(4 * T, 7.0); F.dpf.assign(T * DPS, 7.0); F.H.assign(T * HS, 7.0); F.f.assign(T * 2 * TM_MAXOBS, 7.0);
}

static TmArgs args_of(Filter& F)
{
    TmArgs a; memset(&a, 0, sizeof(a));
    a.m = F.m.data(); a.N = N; a.stereo = F.stereo; a.timeShift = 1; a.ntracks = 1;
    for (int c = 0; c < 2; c++) { const double* Tm = c ? F.T2 : F.T1; for (int r = 0; r < 3; r++) { for (int k = 0; k < 3; k++) a.Rc[c][3 * r + k] = Tm[4 * k + r]; a.base[c][r] = Tm[12 + r]; } }
    a.gnIterations = 10; a.convThreshold = 1e-2; a.convR = 11.0; a.rcondThreshold = 1e-8; a.minDist = 0; a.maxDist = 1e300;
    a.npose = F.npose.data(); a.idx = F.idx.data(); a.ip = F.ip.data(); a.vel = F.vel.data();
    a.status = F.st.data(); a.pf = F.pf.data(); a.dpf = F.dpf.data(); a.H = F.H.data(); a.f = F.f.data(); a.Hstride = HS;
    a.trackOffset = TRK; a.counter = &F.counter; a.counterMax = 5; a.pdl = 1;
    return a;
}

template <class V> static bool same(const V& a, const V& b) { return a.size() == b.size() && memcmp(a.data(), b.data(), a.size() * sizeof(a[0])) == 0; }

int main()
{
    Filter F[3];
    make_filter(F[0], 1, 0, 2);                      // mono
    make_filter(F[1], 2, 1, 0);                      // stereo
    make_filter(F[2], 3, 1, 5);                      // stereo, its chain already has its 5 successful updates
    std::vector<double> dyn(tm_smem_bytes() / 8, std::nan(""));      // shared memory is not zero on the device
    gridDim.x = 1;
    // per filter: CTA 0 of a one-track launch at the step's track offset (what hv_ekf_visual_tracks issues)
    std::vector<Filter> ref(F, F + 3);
    for (Filter& R : ref) {
        reset_outputs(R);
        TmArgs a = args_of(R);
        std::fill(dyn.begin(), dyn.end(), std::nan(""));
        emu::launch_cta(TM_NT, 0, [&] { tm_body(a, dyn.data()); });
    }
    // the group launch: CTA i on args[i]
    TmArgs args[3];
    for (int i = 0; i < 3; i++) { reset_outputs(F[i]); args[i] = args_of(F[i]); }
    gridDim.x = 3;
    for (int inst = 2; inst >= 0; inst--) {          // (any order: the CTAs share nothing)
        std::fill(dyn.begin(), dyn.end(), std::nan(""));
        emu::launch_cta(TM_NT, inst, [&] { tm_group_body(args, blockIdx.x, dyn.data()); });
    }
    int fails = 0;
    for (int i = 0; i < 3; i++) {
        const Filter &G = F[i], &R = ref[i];
        const int* st = &G.st[4 * TRK];
        const bool untouched = G.st[0] == -7 && G.st[8] == -7 && G.H[0] == 7.0 && G.H[2 * HS] == 7.0 && G.pf[0] == 7.0 && G.pf[8] == 7.0;
        bool ok = same(G.st, R.st) && same(G.pf, R.pf) && same(G.dpf, R.dpf) && same(G.H, R.H) && same(G.f, R.f) && untouched;
        if (i == 2) ok = ok && st[0] == TM_SKIPPED && st[1] == TM_VU_NOT_RUN && G.H[TRK * HS] == 7.0;
        else ok = ok && st[0] == TM_OK && st[1] == TM_VU_OK && st[2] == 2 * G.npose[TRK] * (G.stereo ? 2 : 1) && G.H[TRK * HS] != 7.0;
        printf("instance %d (%s, npose %d, counter %d): status %d/%d H %dx%d  %s\n", i, G.stereo ? "stereo" : "mono", G.npose[TRK], G.counter,
               st[0], st[1], st[2], st[3], ok ? "ok" : "FAIL");
        fails += !ok;
    }
    return fails;
}
