// tests/emu/emu_pnp.cpp -- the REAL absolute-pose RANSAC kernel (hybvio_b200/csrc/pnp.cu) on the host emulator against the oracle
// (oracle/hv_oracle_pnp.c), bit for bit: rvec, tvec, mask, inliers and ok. Every job alone (the per-call launch: one CTA) and all jobs
// in one batch (one CTA per job, each reading its own slot of the argument block). The jobs come from a file the test writes: njobs,
// then per job n, fx, fy, cx, cy, has_status, xyz (3n float), xy (2n float), status (n bytes if any); then iterations, reproj_error
// (float), confidence. "pnp_device.inc" is cut out of pnp.cu by the test that builds this file (the `extern __shared__` array becomes a
// pointer).
#include "cuda_emu.h"
#define __constant__
#define __noinline__
inline long long __double_as_longlong(double x) { long long b; memcpy(&b, &x, 8); return b; }
inline double __longlong_as_double(long long b) { double x; memcpy(&x, &b, 8); return x; }
inline int __double2int_rn(double x) { return (int)std::nearbyint(x); }
inline int __shfl_up_sync(unsigned, int v, int delta)
{
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double* slot = emu::cta->xch.data() + (size_t)w * 32;
    slot[lane] = (double)v;
    emu::cta->wbar[w]->arrive_and_wait();
    const int r = lane >= delta ? (int)slot[lane - delta] : v;
    emu::cta->wbar[w]->arrive_and_wait();
    return r;
}
#include "pnp_device.inc"

extern "C" int orc_solve_pnp_ransac(const float* xyz, const float* xy, const uint8_t* status, int n, double fx, double fy, double cx,
                                    double cy, int iterations, float reproj_error, double confidence, double* rvec, double* tvec,
                                    uint8_t* mask, int* inliers, int* ok);

struct Job {
    int n, hasStatus;
    double fx, fy, cx, cy;
    std::vector<float> xyz, xy;
    std::vector<uint8_t> status;
    // outputs (mask with one sentinel byte past n)
    double rvec[3], tvec[3];
    std::vector<uint8_t> mask;
    int inliers, ok;
    std::vector<float> P;
    std::vector<float2> Q;
    std::vector<int> idx;
    std::vector<double> pws, us, al, pcs;
};

static void arm(Job& J, PnpArgs& a)
{
    const size_t n = (size_t)(J.n > 0 ? J.n : 1);
    for (int k = 0; k < 3; k++) { J.rvec[k] = 12345.0; J.tvec[k] = 12345.0; }
    J.mask.assign((size_t)J.n + 1, 0xAB);
    J.inliers = J.ok = -7;
    J.P.assign(3 * n, -1.0f); J.Q.assign(n, float2{-1.0f, -1.0f}); J.idx.assign(n, -1);
    J.pws.assign(3 * n, -1.0); J.us.assign(2 * n, -1.0); J.al.assign(4 * n, -1.0); J.pcs.assign(3 * n, -1.0);
    memset(&a, 0, sizeof(a));
    a.xyz = J.xyz.data(); a.xy = (const float2*)J.xy.data(); a.status = J.hasStatus ? J.status.data() : nullptr;
    a.n = J.n; a.fx = J.fx; a.fy = J.fy; a.cx = J.cx; a.cy = J.cy;
    a.rvec = J.rvec; a.tvec = J.tvec; a.mask = J.mask.data(); a.inliers = &J.inliers; a.ok = &J.ok;
    a.P = J.P.data(); a.Q = J.Q.data(); a.idx = J.idx.data();
    a.pws = J.pws.data(); a.us = J.us.data(); a.al = J.al.data(); a.pcs = J.pcs.data();
}

static bool check(const Job& J, int it, float thr, double conf, const char* what, int j)
{
    double r[3], t[3];
    std::vector<uint8_t> mask((size_t)J.n + 1, 0);
    int inl = -1, ok = -1;
    orc_solve_pnp_ransac(J.xyz.data(), J.xy.data(), J.hasStatus ? J.status.data() : nullptr, J.n, J.fx, J.fy, J.cx, J.cy, it, thr, conf, r, t,
                         mask.data(), &inl, &ok);
    const bool same = ok == J.ok && inl == J.inliers && memcmp(r, J.rvec, sizeof(r)) == 0 && memcmp(t, J.tvec, sizeof(t)) == 0 &&
                      memcmp(mask.data(), J.mask.data(), (size_t)J.n) == 0 && J.mask[(size_t)J.n] == 0xAB;
    printf("%s job %d (n %d): ok %d/%d inliers %d/%d  %s\n", what, j, J.n, J.ok, ok, J.inliers, inl, same ? "ok" : "FAIL");
    return same;
}

int main(int argc, char** argv)
{
    FILE* f = fopen(argc > 1 ? argv[1] : "jobs.bin", "rb");
    if (!f) { printf("no input\n"); return 2; }
    int njobs = 0;
    if (fread(&njobs, 4, 1, f) != 1 || njobs < 1 || njobs > HV_ESSENTIAL_BATCH_MAX) return 2;
    std::vector<Job> jobs((size_t)njobs);
    for (Job& J : jobs) {
        double k[4];
        if (fread(&J.n, 4, 1, f) != 1 || fread(k, 8, 4, f) != 4 || fread(&J.hasStatus, 4, 1, f) != 1) return 2;
        J.fx = k[0]; J.fy = k[1]; J.cx = k[2]; J.cy = k[3];
        J.xyz.resize(3 * (size_t)J.n + 3); J.xy.resize(2 * (size_t)J.n + 2);
        if (fread(J.xyz.data(), 4, 3 * (size_t)J.n, f) != 3 * (size_t)J.n || fread(J.xy.data(), 4, 2 * (size_t)J.n, f) != 2 * (size_t)J.n) return 2;
        if (J.hasStatus) {
            J.status.resize((size_t)J.n + 1);
            if (fread(J.status.data(), 1, (size_t)J.n, f) != (size_t)J.n) return 2;
        }
    }
    int it = 0;
    float thr = 0;
    double conf = 0;
    if (fread(&it, 4, 1, f) != 1 || fread(&thr, 4, 1, f) != 1 || fread(&conf, 8, 1, f) != 1) return 2;
    fclose(f);
    bool all = true;
    static PnpBatchArgs b;
    static PnpShared smem;                             // one CTA at a time
    emu_dynamic_smem = reinterpret_cast<unsigned char*>(&smem);
    for (int j = 0; j < njobs; j++) {                  // the per-call launch: one job, one CTA
        memset(&b, 0, sizeof(b));
        arm(jobs[j], b.job[0]);
        b.iterations = it; b.reprojError = thr; b.confidence = conf;
        emu::launch_cta(PNP_THREADS, 0u, [&] { hv_pnp_kernel(b); });
        all &= check(jobs[j], it, thr, conf, "call ", j);
    }
    memset(&b, 0, sizeof(b));                          // the batch: CTA j runs job j
    for (int j = 0; j < njobs; j++) arm(jobs[j], b.job[j]);
    b.iterations = it; b.reprojError = thr; b.confidence = conf;
    for (int j = njobs - 1; j >= 0; j--) emu::launch_cta(PNP_THREADS, (unsigned)j, [&] { hv_pnp_kernel(b); });
    for (int j = 0; j < njobs; j++) all &= check(jobs[j], it, thr, conf, "batch", j);
    printf(all ? "all ok\n" : "FAIL\n");
    return all ? 0 : 1;
}
