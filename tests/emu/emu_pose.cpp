// tests/emu/emu_pose.cpp -- the REAL relative-pose kernel (hybvio_b200/csrc/pose.cu) on the host emulator against the oracle
// (oracle/hv_oracle_pose.c), bit for bit: R, t, mask and good. Every job alone (the per-call launch: one CTA) and all jobs in one batch
// (one CTA per job, each reading its own slot of the argument block). The jobs come from a file the test writes: njobs, then per job
// n, fx, fy, cx, cy, nsol (-1: no count, the NULL pointer), has_mask, in_place, E (9 doubles, column-major), xy1 (2n float),
// xy2 (2n float), mask (n bytes if any); then distance_thresh. "pose_device.inc" is cut out of pose.cu by the test that builds this file.
#include "cuda_emu.h"
#define __noinline__
#include "pose_device.inc"

extern "C" int orc_recover_pose(const double* E, int nsol, const float* xy1, const float* xy2, const uint8_t* mask_in, int n, double fx,
                                double fy, double cx, double cy, double dist, double* R, double* t, uint8_t* mask_out, int* good);

struct Job {
    int n, nsol, hasMask, inPlace;
    double fx, fy, cx, cy;
    std::vector<double> E;
    std::vector<float> xy1, xy2;
    std::vector<uint8_t> mask;
    // outputs (mask with one sentinel byte past n)
    std::vector<double> R, t;
    std::vector<uint8_t> out;
    int good;
};

static void arm(Job& J, PoseArgs& a)
{
    J.R.assign(9, 12345.0);
    J.t.assign(3, 12345.0);
    J.out.assign((size_t)J.n + 1, 0xAB);
    if (J.inPlace) memcpy(J.out.data(), J.mask.data(), (size_t)J.n);
    J.good = -7;
    memset(&a, 0, sizeof(a));
    a.E = J.E.data(); a.nsol = J.nsol >= 0 ? &J.nsol : nullptr;
    a.xy1 = (const float2*)J.xy1.data(); a.xy2 = (const float2*)J.xy2.data();
    a.maskIn = !J.hasMask ? nullptr : (J.inPlace ? J.out.data() : J.mask.data());
    a.n = J.n; a.fx = J.fx; a.fy = J.fy; a.cx = J.cx; a.cy = J.cy;
    a.R = J.R.data(); a.t = J.t.data(); a.maskOut = J.out.data(); a.good = &J.good;
}

static bool check(const Job& J, double dist, const char* what, int j)
{
    std::vector<double> R(9), t(3);
    std::vector<uint8_t> out((size_t)J.n + 1, 0);
    int good = -1;
    orc_recover_pose(J.E.data(), J.nsol >= 0 ? J.nsol : 1, J.xy1.data(), J.xy2.data(), J.hasMask ? J.mask.data() : nullptr, J.n, J.fx, J.fy,
                     J.cx, J.cy, dist, R.data(), t.data(), out.data(), &good);
    const bool ok = good == J.good && memcmp(R.data(), J.R.data(), 9 * sizeof(double)) == 0 && memcmp(t.data(), J.t.data(), 3 * sizeof(double)) == 0 &&
                    memcmp(out.data(), J.out.data(), (size_t)J.n) == 0 && J.out[(size_t)J.n] == 0xAB;
    printf("%s job %d (n %d nsol %d mask %d in place %d): good %d/%d  %s\n", what, j, J.n, J.nsol, J.hasMask, J.inPlace, J.good, good,
           ok ? "ok" : "FAIL");
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
        int h[4];
        if (fread(&J.n, 4, 1, f) != 1 || fread(k, 8, 4, f) != 4 || fread(h, 4, 3, f) != 3) return 2;
        J.fx = k[0]; J.fy = k[1]; J.cx = k[2]; J.cy = k[3];
        J.nsol = h[0]; J.hasMask = h[1]; J.inPlace = h[2];
        J.E.resize(9);
        if (fread(J.E.data(), 8, 9, f) != 9) return 2;
        J.xy1.resize(2 * (size_t)J.n + 2); J.xy2.resize(2 * (size_t)J.n + 2);
        if (fread(J.xy1.data(), 4, 2 * (size_t)J.n, f) != 2 * (size_t)J.n || fread(J.xy2.data(), 4, 2 * (size_t)J.n, f) != 2 * (size_t)J.n) return 2;
        J.mask.assign((size_t)J.n + 1, 0);
        if (J.hasMask && fread(J.mask.data(), 1, (size_t)J.n, f) != (size_t)J.n) return 2;
    }
    double dist = 0;
    if (fread(&dist, 8, 1, f) != 1) return 2;
    fclose(f);
    bool all = true;
    static PoseBatchArgs b;
    for (int j = 0; j < njobs; j++) {                  // the per-call launch: one job, one CTA
        memset(&b, 0, sizeof(b));
        arm(jobs[j], b.job[0]);
        b.dist = dist;
        emu::launch_cta(POSE_THREADS, 0u, [&] { hv_pose_kernel(b); });
        all &= check(jobs[j], dist, "call ", j);
    }
    memset(&b, 0, sizeof(b));                          // the batch: CTA j runs job j
    for (int j = 0; j < njobs; j++) arm(jobs[j], b.job[j]);
    b.dist = dist;
    for (int j = njobs - 1; j >= 0; j--) emu::launch_cta(POSE_THREADS, (unsigned)j, [&] { hv_pose_kernel(b); });
    for (int j = 0; j < njobs; j++) all &= check(jobs[j], dist, "batch", j);
    printf(all ? "all ok\n" : "FAIL\n");
    return all ? 0 : 1;
}
