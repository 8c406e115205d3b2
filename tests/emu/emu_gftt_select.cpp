// tests/emu/emu_gftt_select.cpp -- the REAL body of hv_gftt_select_kernel (device part of hybvio_b200/csrc/gftt_select.cu: bitonic sort of
// the keys, the quirk points, the chunked greedy filter with its ballot loop) on the host emulator against orc_gftt_corners
// (oracle/hv_oracle_gftt.c): list, count and padding bit for bit. "gftt_select_device.inc" is cut out of gftt_select.cu by the test that
// builds this file (the `extern __shared__` array becomes a pointer). The cases come from a file the test writes:
//   int32 ncases; per case int32 nkp, nprev, mask_radius, max_tracks, float32 kp[3 nkp], float32 prev[2 nprev].
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
    if (fread(&ncases, 4, 1, f) != 1) return 2;
    for (int cs = 0; cs < ncases; cs++) {
        int hdr[4];
        if (fread(hdr, 4, 4, f) != 4) return 2;
        const int nkp = hdr[0], nprev = hdr[1], r = hdr[2], maxTracks = hdr[3];
        std::vector<float> kp(3 * (size_t)nkp + 1), prev(2 * (size_t)nprev + 1);
        if (fread(kp.data(), 4, 3 * (size_t)nkp, f) != 3 * (size_t)nkp || fread(prev.data(), 4, 2 * (size_t)nprev, f) != 2 * (size_t)nprev) return 2;
        std::vector<float> want(4 * (size_t)nkp + 2);
        const int wantN = orc_gftt_corners(kp.data(), nkp, prev.data(), nprev, r, maxTracks, want.data());
        const int all = 2 * nkp, need = r > 0 ? (maxTracks < all ? maxTracks : all) : all, cap = need + 3;
        std::vector<float> out(2 * (size_t)cap, 12345.f);
        int count = -7;
        GfttSelectArgs a; memset(&a, 0, sizeof(a));
        a.kp = kp.data(); a.nkp = nkp; a.prev = prev.data(); a.nprev = nprev; a.maskRadius = r; a.maxTracks = maxTracks;
        a.r2 = r > 0 ? (float)(r * r) : 0.f;
        a.pow2 = 2; while (a.pow2 < nkp) a.pow2 *= 2;
        a.out = out.data(); a.capacity = cap; a.count = &count;
        unsigned done = 0, flag = 0;
        a.done = HvDoneSignal{&done, 1, 9, &flag};
        std::vector<unsigned long long> smem((size_t)a.pow2 + 2, 0x5A5A5A5A5A5A5A5Aull);
        emu_dynamic_smem = (unsigned char*)smem.data();
        gridDim.x = gridDim.y = gridDim.z = 1;
        emu::launch_cta(1024, 0, [&] { hv_gftt_select_kernel(a); });
        int bad = count != wantN;
        for (int i = 0; i < 2 * wantN && !bad; i++) bad = memcmp(&out[i], &want[i], 4) != 0;
        for (int i = 2 * wantN; i < 2 * cap && !bad; i++) bad = out[i] != -1.0e6f;
        const bool ok = !bad && flag == 9 && done == 1;
        printf("case %d: nkp %d nprev %d r %d max %d: count %d (oracle %d)  %s\n", cs, nkp, nprev, r, maxTracks, count, wantN, ok ? "ok" : "FAIL");
        fails += !ok;
    }
    fclose(f);
    printf("%s\n", fails ? "FAIL" : "all ok");
    return fails ? 1 : 0;
}
