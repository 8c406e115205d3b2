// tests/emu/emu_gftt_select_batch.cpp -- the REAL hv_gftt_select_batch_kernel (hybvio_b200/csrc/gftt_select.cu: CTA j runs the list body
// of hv_gftt_select_kernel on job j) on the host emulator: every case of the file in ONE emulated launch, one job per case, with
// different nkp, sort widths, radii, max_tracks and spare capacity, and the shared memory sized for the largest sort. Each job's list,
// count and padding against orc_gftt_corners (oracle/hv_oracle_gftt.c) bit for bit. "gftt_select_device.inc" is cut out of
// gftt_select.cu by the test that builds this file; the case file is the one emu_gftt_select.cpp reads (at most 64 cases).
#include "cuda_emu.h"
#include "cuda_emu_ballot.h"
inline float2 make_float2(float x, float y) { return float2{x, y}; }
#include "gftt_select_device.inc"

extern "C" int orc_gftt_corners(const float* kp_xyr, int nkp, const float* prev_xy, int nprev, int mask_radius, int max_tracks, float* corners_xy);

int main(int argc, char** argv)
{
    if (argc < 2) return 2;
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 2;
    int ncases = 0, fails = 0;
    if (fread(&ncases, 4, 1, f) != 1 || ncases < 1 || ncases > HV_CORNER_BATCH_MAX) return 2;
    std::vector<std::vector<float>> kp(ncases), prev(ncases), out(ncases), want(ncases);
    std::vector<int> count(ncases, -7), wantN(ncases), cap(ncases);
    static GfttSelectBatchArgs b;
    memset(&b, 0, sizeof(b));
    int maxPow2 = 2;
    for (int j = 0; j < ncases; j++) {
        int hdr[4];
        if (fread(hdr, 4, 4, f) != 4) return 2;
        const int nkp = hdr[0], nprev = hdr[1], r = hdr[2], maxTracks = hdr[3];
        kp[j].resize(3 * (size_t)nkp + 1); prev[j].resize(2 * (size_t)nprev + 1);
        if (fread(kp[j].data(), 4, 3 * (size_t)nkp, f) != 3 * (size_t)nkp || fread(prev[j].data(), 4, 2 * (size_t)nprev, f) != 2 * (size_t)nprev) return 2;
        want[j].resize(4 * (size_t)nkp + 2);
        wantN[j] = orc_gftt_corners(kp[j].data(), nkp, prev[j].data(), nprev, r, maxTracks, want[j].data());
        const int all = 2 * nkp, need = r > 0 ? (maxTracks < all ? maxTracks : all) : all;
        cap[j] = need + j % 4;                                        // spare slots differ from job to job
        out[j].assign(2 * (size_t)cap[j] + 1, 12345.f);
        GfttSelectArgs& a = b.job[j];
        a.kp = kp[j].data(); a.nkp = nkp; a.prev = prev[j].data(); a.nprev = nprev; a.maskRadius = r; a.maxTracks = maxTracks;
        a.r2 = r > 0 ? (float)(r * r) : 0.f;
        a.pow2 = 2; while (a.pow2 < nkp) a.pow2 *= 2;
        a.out = out[j].data(); a.capacity = cap[j]; a.count = &count[j];
        if (a.pow2 > maxPow2) maxPow2 = a.pow2;
    }
    fclose(f);
    // one shared-memory block of the launch's size, left as the previous CTA wrote it (a CTA must not rely on a fresh one)
    std::vector<unsigned long long> smem((size_t)maxPow2 + 2, 0x5A5A5A5A5A5A5A5Aull);
    emu_dynamic_smem = (unsigned char*)smem.data();
    gridDim.x = ncases; gridDim.y = gridDim.z = 1;
    for (int j = ncases - 1; j >= 0; j--) emu::launch_cta(1024, (unsigned)j, [&] { hv_gftt_select_batch_kernel(b); });
    for (int j = 0; j < ncases; j++) {
        int bad = count[j] != wantN[j];
        for (int i = 0; i < 2 * wantN[j] && !bad; i++) bad = memcmp(&out[j][i], &want[j][i], 4) != 0;
        for (int i = 2 * wantN[j]; i < 2 * cap[j] && !bad; i++) bad = out[j][i] != -1.0e6f;
        bad |= out[j][2 * cap[j]] != 12345.f;                         // nothing written beyond the capacity
        printf("job %d: nkp %d pow2 %d nprev %d r %d max %d cap %d: count %d (oracle %d)  %s\n", j, b.job[j].nkp, b.job[j].pow2, b.job[j].nprev,
               b.job[j].maskRadius, b.job[j].maxTracks, cap[j], count[j], wantN[j], bad ? "FAIL" : "ok");
        fails += bad;
    }
    printf("%s\n", fails ? "FAIL" : "all ok");
    return fails ? 1 : 0;
}
