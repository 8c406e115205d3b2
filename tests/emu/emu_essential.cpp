// tests/emu/emu_essential.cpp -- the REAL essential-matrix RANSAC kernel (hybvio_b200/csrc/essential.cu) on the host emulator against
// the oracle (oracle/hv_oracle_essential.c), bit for bit: E (all 10 slots), nsol, mask and inliers. Every job alone (the per-call
// launch: one CTA) and all jobs in one batch (one CTA per job, each reading its own slot of the argument block). The jobs come from a
// file the test writes: njobs, then per job n, fx, fy, cx, cy, has_status, xy1 (2n float), xy2 (2n float), status (n bytes if any);
// then prob, threshold, max_iters. "essential_device.inc" is cut out of essential.cu by the test that builds this file (the
// `extern __shared__` array becomes a pointer).
#include "cuda_emu.h"
#include "cuda_emu_ballot.h"
#define __constant__
#define __noinline__
inline int __popc(unsigned x) { return __builtin_popcount(x); }
struct __attribute__((aligned(16))) double4 { double x, y, z, w; };
inline double4 make_double4(double x, double y, double z, double w) { return double4{x, y, z, w}; }
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
#include "essential_device.inc"

extern "C" int orc_find_essential(const float* xy1, const float* xy2, const uint8_t* status, int n, double fx, double fy, double cx,
                                  double cy, double prob, double threshold, int max_iters, double* E, int* nsol, uint8_t* mask, int* inliers);

struct Job {
    int n, hasStatus;
    double fx, fy, cx, cy;
    std::vector<float> xy1, xy2;
    std::vector<uint8_t> status;
    // outputs (mask with one sentinel byte past n)
    std::vector<double> E;
    std::vector<uint8_t> mask;
    int nsol, inliers;
    std::vector<double4> q;
    std::vector<int> idx;
};

static void arm(Job& J, EssentialArgs& a)
{
    J.E.assign(90, 12345.0);
    J.mask.assign((size_t)J.n + 1, 0xAB);
    J.nsol = J.inliers = -7;
    J.q.assign((size_t)(J.n > 0 ? J.n : 1), double4{0, 0, 0, 0});
    J.idx.assign((size_t)(J.n > 0 ? J.n : 1), -1);
    memset(&a, 0, sizeof(a));
    a.xy1 = (const float2*)J.xy1.data(); a.xy2 = (const float2*)J.xy2.data(); a.status = J.hasStatus ? J.status.data() : nullptr;
    a.n = J.n; a.fx = J.fx; a.fy = J.fy; a.cx = J.cx; a.cy = J.cy;
    a.E = J.E.data(); a.nsol = &J.nsol; a.mask = J.mask.data(); a.inliers = &J.inliers;
    a.q = &J.q.data()->x; a.idx = J.idx.data();
}

static bool check(const Job& J, double prob, double thr, int mi, const char* what, int j)
{
    std::vector<double> E(90);
    std::vector<uint8_t> mask((size_t)J.n + 1, 0);
    int nsol = -1, inl = -1;
    orc_find_essential(J.xy1.data(), J.xy2.data(), J.hasStatus ? J.status.data() : nullptr, J.n, J.fx, J.fy, J.cx, J.cy, prob, thr, mi,
                       E.data(), &nsol, mask.data(), &inl);
    const bool ok = nsol == J.nsol && inl == J.inliers && memcmp(E.data(), J.E.data(), 90 * sizeof(double)) == 0 &&
                    memcmp(mask.data(), J.mask.data(), (size_t)J.n) == 0 && J.mask[(size_t)J.n] == 0xAB;
    printf("%s job %d (n %d): nsol %d/%d inliers %d/%d  %s\n", what, j, J.n, J.nsol, nsol, J.inliers, inl, ok ? "ok" : "FAIL");
    return ok;
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
        J.xy1.resize(2 * (size_t)J.n + 2); J.xy2.resize(2 * (size_t)J.n + 2);
        if (fread(J.xy1.data(), 4, 2 * (size_t)J.n, f) != 2 * (size_t)J.n || fread(J.xy2.data(), 4, 2 * (size_t)J.n, f) != 2 * (size_t)J.n) return 2;
        if (J.hasStatus) {
            J.status.resize((size_t)J.n + 1);
            if (fread(J.status.data(), 1, (size_t)J.n, f) != (size_t)J.n) return 2;
        }
    }
    double prob = 0, thr = 0;
    int mi = 0;
    if (fread(&prob, 8, 1, f) != 1 || fread(&thr, 8, 1, f) != 1 || fread(&mi, 4, 1, f) != 1) return 2;
    fclose(f);
    bool all = true;
    static EssentialBatchArgs b;
    static EssShared smem;                             // one CTA at a time
    emu_dynamic_smem = reinterpret_cast<unsigned char*>(&smem);
    for (int j = 0; j < njobs; j++) {                  // the per-call launch: one job, one CTA
        memset(&b, 0, sizeof(b));
        arm(jobs[j], b.job[0]);
        b.prob = prob; b.threshold = thr; b.maxIters = mi;
        emu::launch_cta(ESS_THREADS, 0u, [&] { hv_essential_kernel(b); });
        all &= check(jobs[j], prob, thr, mi, "call ", j);
    }
    memset(&b, 0, sizeof(b));                          // the batch: CTA j runs job j
    for (int j = 0; j < njobs; j++) arm(jobs[j], b.job[j]);
    b.prob = prob; b.threshold = thr; b.maxIters = mi;
    for (int j = njobs - 1; j >= 0; j--) emu::launch_cta(ESS_THREADS, (unsigned)j, [&] { hv_essential_kernel(b); });
    for (int j = 0; j < njobs; j++) all &= check(jobs[j], prob, thr, mi, "batch", j);
    printf(all ? "all ok\n" : "FAIL\n");
    return all ? 0 : 1;
}
