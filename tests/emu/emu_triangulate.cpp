// tests/emu/emu_triangulate.cpp -- the REAL triangulation kernel (hybvio_b200/csrc/triangulate.cu) on the host emulator against the
// oracle (oracle/hv_oracle_triangulate.c), bit for bit: X4, xyz and used. Every job alone (the per-call launch: grid (points, 1)) and all
// jobs in one batch (grid (points of the largest job, jobs)). The jobs come from a file the test writes: njobs, then per job n, has_status,
// has_status2, alias (0: used is its own buffer, 1: used is status, 2: used is status2), want_X4, want_xyz, want_used, P1 and P2 (12
// doubles each, row-major), xy1 (2n float), xy2 (2n float), status (n bytes if any), status2 (n bytes if any).
// "triangulate_device.inc" is cut out of triangulate.cu by the test that builds this file.
#include "cuda_emu.h"
#include "triangulate_device.inc"

extern "C" void orc_triangulate_points(const double* P1, const double* P2, const float* xy1, const float* xy2, const uint8_t* status,
                                       const uint8_t* status2, int n, float* X4, float* xyz, uint8_t* used);

struct Job {
    int n, hasS1, hasS2, alias, wantX4, wantXyz, wantUsed;
    double P1[12], P2[12];
    std::vector<float> xy1, xy2;
    std::vector<uint8_t> s1, s2;
    // outputs, one sentinel element past the end; st1 / st2 the statuses as the kernel sees them (used may overwrite one)
    std::vector<float> X4, xyz;
    std::vector<uint8_t> used, st1, st2;
};

static void arm(Job& J, TriArgs& a)
{
    const size_t n = (size_t)J.n;
    J.X4.assign(4 * n + 1, 1234.5f);
    J.xyz.assign(3 * n + 1, 1234.5f);
    J.used.assign(n + 1, 0xAB);
    J.st1 = J.s1; J.st2 = J.s2;
    memset(&a, 0, sizeof(a));
    memcpy(a.P1, J.P1, sizeof(a.P1));
    memcpy(a.P2, J.P2, sizeof(a.P2));
    a.xy1 = (const float2*)J.xy1.data(); a.xy2 = (const float2*)J.xy2.data();
    a.status = J.hasS1 ? J.st1.data() : nullptr; a.status2 = J.hasS2 ? J.st2.data() : nullptr;
    a.n = J.n;
    a.X4 = J.wantX4 ? J.X4.data() : nullptr;
    a.xyz = J.wantXyz ? J.xyz.data() : nullptr;
    a.used = J.alias == 1 ? J.st1.data() : (J.alias == 2 ? J.st2.data() : (J.wantUsed ? J.used.data() : nullptr));
}

static bool check(const Job& J, const char* what, int j)
{
    const size_t n = (size_t)J.n;
    std::vector<float> X4(4 * n + 1, 0.0f), xyz(3 * n + 1, 0.0f);
    std::vector<uint8_t> used(n + 1, 0);
    orc_triangulate_points(J.P1, J.P2, J.xy1.data(), J.xy2.data(), J.hasS1 ? J.s1.data() : nullptr, J.hasS2 ? J.s2.data() : nullptr, J.n,
                           X4.data(), xyz.data(), used.data());
    bool ok = true;
    if (J.wantX4) ok &= memcmp(X4.data(), J.X4.data(), 16 * n) == 0;
    else ok &= J.X4[0] == 1234.5f;
    if (J.wantXyz) ok &= memcmp(xyz.data(), J.xyz.data(), 12 * n) == 0;
    else ok &= J.xyz[0] == 1234.5f;
    ok &= J.X4[4 * n] == 1234.5f && J.xyz[3 * n] == 1234.5f && J.used[n] == 0xAB;
    const uint8_t* got = J.alias == 1 ? J.st1.data() : (J.alias == 2 ? J.st2.data() : (J.wantUsed ? J.used.data() : nullptr));
    if (got) ok &= memcmp(used.data(), got, n) == 0;
    else ok &= n == 0 || J.used[0] == 0xAB;
    int nu = 0;
    for (size_t i = 0; i < n; i++) nu += used[i];
    printf("%s job %d (n %d status %d/%d alias %d outputs %d%d%d): %d used  %s\n", what, j, J.n, J.hasS1, J.hasS2, J.alias, J.wantX4,
           J.wantXyz, J.wantUsed, nu, ok ? "ok" : "FAIL");
    return ok;
}

static void run(TriBatchArgs& b, int njobs, int maxn)
{
    const unsigned gx = (unsigned)(((maxn > 0 ? maxn : 1) + TRI_THREADS - 1) / TRI_THREADS);
    for (int y = 0; y < njobs; y++) {
        emu::block_y = (unsigned)y;
        for (unsigned x = 0; x < gx; x++) emu::launch_cta(TRI_THREADS, x, [&] { hv_triangulate_kernel(b); });
    }
    emu::block_y = 0;
}

int main(int argc, char** argv)
{
    FILE* f = fopen(argc > 1 ? argv[1] : "jobs.bin", "rb");
    if (!f) { printf("no input\n"); return 2; }
    int njobs = 0;
    if (fread(&njobs, 4, 1, f) != 1 || njobs < 1 || njobs > HV_ESSENTIAL_BATCH_MAX) return 2;
    std::vector<Job> jobs((size_t)njobs);
    for (Job& J : jobs) {
        int h[7];
        if (fread(h, 4, 7, f) != 7) return 2;
        J.n = h[0]; J.hasS1 = h[1]; J.hasS2 = h[2]; J.alias = h[3]; J.wantX4 = h[4]; J.wantXyz = h[5]; J.wantUsed = h[6];
        const size_t n = (size_t)J.n;
        if (fread(J.P1, 8, 12, f) != 12 || fread(J.P2, 8, 12, f) != 12) return 2;
        J.xy1.resize(2 * n + 2); J.xy2.resize(2 * n + 2);
        if (fread(J.xy1.data(), 4, 2 * n, f) != 2 * n || fread(J.xy2.data(), 4, 2 * n, f) != 2 * n) return 2;
        J.s1.assign(n + 1, 0); J.s2.assign(n + 1, 0);
        if (J.hasS1 && fread(J.s1.data(), 1, n, f) != n) return 2;
        if (J.hasS2 && fread(J.s2.data(), 1, n, f) != n) return 2;
    }
    fclose(f);
    bool all = true;
    static TriBatchArgs b;
    for (int j = 0; j < njobs; j++) {                  // the per-call launch: one job
        memset(&b, 0, sizeof(b));
        arm(jobs[j], b.job[0]);
        run(b, 1, jobs[j].n);
        all &= check(jobs[j], "call ", j);
    }
    memset(&b, 0, sizeof(b));                          // the batch: grid row y runs job y
    int maxn = 0;
    for (int j = 0; j < njobs; j++) {
        arm(jobs[j], b.job[j]);
        if (jobs[j].n > maxn) maxn = jobs[j].n;
    }
    run(b, njobs, maxn);
    for (int j = 0; j < njobs; j++) all &= check(jobs[j], "batch", j);
    printf(all ? "all ok\n" : "FAIL\n");
    return all ? 0 : 1;
}
