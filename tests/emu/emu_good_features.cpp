// tests/emu/emu_good_features.cpp -- the REAL Shi-Tomasi kernels (hybvio_b200/csrc/good_features.cu) on the host emulator against the
// cv::goodFeaturesToTrack oracle (oracle/hv_oracle_good_features.c), bit for bit: the response map, count, (x, y), response, the
// HV_CORNER_NONE / 0 padding up to the capacity and an untouched float past it.
// Per frame (the three kernels of hv_launch_good_features) and batched (the three batch kernels over all jobs at once), on blurred noise,
// raw noise, a periodic pattern (many equal responses), a ramp (responses of rounding noise only) and a flat image, with no mask, a
// half-frame mask and a mask that hides the global maximum, at min_distance 0 / 0.5 / 1 / 2.5 / 10 and max_corners 1 / 150 / above the
// candidate count. The test builds this file with a small HV_GF_CHUNK so that the select's radix-select rounds run on small images.
// "good_features_device.inc" is cut out of good_features.cu by the test (the `extern __shared__` array becomes a pointer).
#include "cuda_emu.h"
#include "cuda_emu_ballot.h"
#include "cuda_emu_atomics.h"
#include <cmath>
#include "good_features_device.inc"

extern "C" int orc_gf_eig(const uint8_t* img, int step, int w, int h, float* eig);
extern "C" int orc_gf_detect(const uint8_t* img, int step, int w, int h, int maxCorners, double q, double minDistance, const uint8_t* mask,
                             int mstride, float* out, int capacity);

static unsigned hash2(int x, int y) { unsigned h = (unsigned)x * 374761393u + (unsigned)y * 668265263u; h = (h ^ (h >> 13)) * 1274126177u; return h ^ (h >> 16); }

// kind 0: blurred noise, 1: raw noise, 2: periodic squares, 3: ramp, 4: flat, 5: dark noise (0..5) under bright bars (dy of rounding noise
// below bright rows: boxFilter's running column sum differs from the exact 9-term sum there)
static std::vector<uint8_t> make_image(int w, int h, int kind, int seed)
{
    std::vector<uint8_t> img((size_t)w * h);
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            int p;
            if (kind == 0) {
                int s = 0;
                for (int d = 0; d < 4; d++) s += hash2(x / 3 + d % 2 + 1000 * seed, y / 3 + d / 2) & 0xff;
                p = s / 4 + (int)(hash2(x, y + seed) & 7);
            } else if (kind == 1) {
                p = hash2(x + 1000 * seed, y) & 0xff;
            } else if (kind == 2) {
                p = ((x / 4) + (y / 4)) & 1 ? 200 : 50;
            } else if (kind == 3) {
                p = (x + 2 * y) & 0xff;
            } else if (kind == 5) {
                const bool bar = (y % 23 < 4 && (x + 3 * seed) % 41 < 25) || (x % 29 < 3 && y % 31 > 12);
                p = bar ? 180 + (int)(hash2(x / 7, y / 5 + seed) % 70) : (int)(hash2(x + 1000 * seed, y) % 6);
            } else {
                p = 90;
            }
            img[(size_t)y * w + x] = (uint8_t)(p > 255 ? 255 : p);
        }
    return img;
}

struct Case { int w, h, kind, maskKind, maxCorners; double q, md; };

struct Job {
    Case cs;
    int pitch, mpitch;
    std::vector<uint8_t> img, dev, mask;
    std::vector<float> wantEig, ref;          // oracle map; (x, y, response) x n
    int n;
    std::vector<float> eig;
    std::vector<unsigned long long> keys;
    std::vector<int> grid;
    unsigned words[2];
    std::vector<float> xy, resp;             // capacity + 1 slots (the last is a sentinel)
    int cap, count;
};

// as gf_args in capi.cu
static void setup(Job& J, const Case& cs, int seed, int capExtra, GoodFeaturesArgs& a)
{
    J.cs = cs;
    const int w = cs.w, h = cs.h;
    J.img = make_image(w, h, cs.kind, seed);
    J.pitch = seed & 1 ? w : (w + 3) / 4 * 4 + 4 * (seed % 3);
    J.dev.assign((size_t)J.pitch * h, 0xEE);
    for (int y = 0; y < h; y++) memcpy(J.dev.data() + (size_t)y * J.pitch, J.img.data() + (size_t)y * w, w);
    J.wantEig.assign((size_t)w * h, 0.f);
    orc_gf_eig(J.img.data(), w, w, h, J.wantEig.data());
    J.mpitch = w + 5;
    J.mask.clear();
    if (cs.maskKind == 1) {                                              // the left half
        J.mask.assign((size_t)J.mpitch * h, 0);
        for (int y = 0; y < h; y++) for (int x = 0; x < w / 2; x++) J.mask[(size_t)y * J.mpitch + x] = 255;
    } else if (cs.maskKind == 2) {                                       // everything but a 9 x 9 block around the global maximum
        int best = 0;
        for (int i = 1; i < w * h; i++) if (J.wantEig[i] > J.wantEig[best]) best = i;
        const int bx = best % w, by = best / w;
        J.mask.assign((size_t)J.mpitch * h, 1);
        for (int y = by - 4; y <= by + 4; y++) for (int x = bx - 4; x <= bx + 4; x++)
            if (x >= 0 && x < w && y >= 0 && y < h) J.mask[(size_t)y * J.mpitch + x] = 0;
    }
    const uint8_t* m = J.mask.empty() ? nullptr : J.mask.data();
    J.n = orc_gf_detect(J.img.data(), w, w, h, cs.maxCorners, cs.q, cs.md, m, J.mpitch, nullptr, 0);
    J.ref.assign(3 * (size_t)J.n + 3, 0.f);
    orc_gf_detect(J.img.data(), w, w, h, cs.maxCorners, cs.q, cs.md, m, J.mpitch, J.ref.data(), J.n);
    J.cap = cs.maxCorners + capExtra;
    J.eig.assign((size_t)w * h, -5.f);
    J.keys.assign(w > 2 && h > 2 ? (size_t)(w - 2) * (h - 2) : 1, 0x5A5A5A5A5A5A5A5Aull);
    J.words[0] = J.words[1] = 0u;
    J.xy.assign(2 * (size_t)J.cap + 2, 777.f);
    J.resp.assign((size_t)J.cap + 1, 777.f);
    J.count = -1;
    memset(&a, 0, sizeof(a));
    a.gray = J.dev.data(); a.pitch = J.pitch; a.w = w; a.h = h;
    a.mask = m; a.maskPitch = J.mpitch;
    a.tilesX = (w + 31) / 32; a.tilesY = (h + 7) / 8;
    a.maxCorners = cs.maxCorners; a.quality = cs.q;
    a.useGrid = cs.md >= 1.0;
    if (a.useGrid) {
        a.md2 = cs.md * cs.md;
        long long s = (long long)(cs.md / 1.4142135623730951);
        if (s > 2897) s = 2897;
        if (s < 1) s = 1;
        while (s > 1 && 2.0 * (double)(s - 1) * (double)(s - 1) >= a.md2) s--;
        while (s < 2897 && 2.0 * (double)s * (double)s < a.md2) s++;
        a.cell = (int)s;
        const int big = w > h ? w : h;
        const double r = std::ceil(cs.md) - 1.0;
        a.reach = r > (double)big ? big : (int)r;
        a.gridW = (w + a.cell - 1) / a.cell; a.gridH = (h + a.cell - 1) / a.cell;
        J.grid.assign((size_t)a.gridW * a.gridH, 0x7777);
    }
    a.maxCand = (int)J.keys.size();
    a.eig = J.eig.data(); a.keys = J.keys.data(); a.grid = a.useGrid ? J.grid.data() : nullptr;
    a.maxWord = &J.words[0]; a.nCand = (int*)&J.words[1];
    a.xy = (float2*)J.xy.data(); a.response = seed % 4 == 3 ? nullptr : J.resp.data(); a.capacity = J.cap; a.count = &J.count;
}

static int check(const char* what, Job& J, bool withResp)
{
    const Case& c = J.cs;
    int bad = J.count != J.n;
    bad += memcmp(J.eig.data(), J.wantEig.data(), J.eig.size() * sizeof(float)) != 0;
    for (int i = 0; i < J.cap; i++) {
        const float ex = i < J.n ? J.ref[3 * i] : HV_CORNER_NONE_F, ey = i < J.n ? J.ref[3 * i + 1] : HV_CORNER_NONE_F;
        const float er = i < J.n ? J.ref[3 * i + 2] : 0.f;
        if (memcmp(&J.xy[2 * i], &ex, 4) || memcmp(&J.xy[2 * i + 1], &ey, 4) || (withResp ? memcmp(&J.resp[i], &er, 4) != 0 : J.resp[i] != 777.f)) {
            if (bad < 3) printf("  slot %d: (%g, %g, %g) vs oracle (%g, %g, %g)\n", i, J.xy[2 * i], J.xy[2 * i + 1], J.resp[i], ex, ey, er);
            bad++;
        }
    }
    bad += J.xy[2 * J.cap] != 777.f || J.xy[2 * J.cap + 1] != 777.f || J.resp[J.cap] != 777.f;
    printf("%s %dx%d kind %d mask %d max %d q %g md %g: count %d (oracle %d), capacity %d: %d differ  %s\n", what, c.w, c.h, c.kind, c.maskKind,
           c.maxCorners, c.q, c.md, J.count, J.n, J.cap, bad, bad ? "FAIL" : "ok");
    return bad != 0;
}

static void run_select(const GoodFeaturesArgs& a, std::vector<unsigned long long>& smem)
{
    emu_dynamic_smem = (unsigned char*)smem.data();
    gridDim.x = 1; gridDim.y = 1;
    emu::launch_cta(GF_SEL_NT, 0u, [&] { hv_gf_select_kernel(a); });
}

static const Case CASES[] = {
    {61, 45, 0, 0, 150, 0.01, 10.0}, {61, 45, 0, 1, 150, 0.01, 2.5}, {61, 45, 0, 2, 100000, 0.01, 1.0}, {70, 37, 1, 0, 100000, 1e-4, 0.0},
    {70, 37, 1, 2, 1, 1e-4, 30.0}, {64, 48, 2, 0, 100000, 0.01, 0.5}, {64, 48, 2, 1, 150, 0.01, 2.5}, {57, 33, 3, 0, 100000, 0.01, 1.0},
    {57, 33, 3, 2, 150, 0.01, 10.0}, {40, 20, 4, 0, 150, 0.01, 10.0}, {2, 9, 1, 0, 5, 0.01, 1.0}, {3, 3, 1, 0, 5, 0.01, 0.0},
    {33, 9, 1, 1, 100000, 1e-4, 2.5}, {97, 70, 5, 0, 100000, 1e-4, 0.0}, {97, 70, 5, 2, 150, 0.01, 10.0}, {333, 241, 5, 1, 1000, 1e-4, 2.5},
};
static const int NCASES = sizeof(CASES) / sizeof(CASES[0]);

int main()
{
    int fails = 0;
    std::vector<unsigned long long> smem(HV_GF_CHUNK + 2, 0x5A5A5A5A5A5A5A5Aull);
    std::vector<Job> jobs(NCASES);
    int multiRound = 0;
    for (int j = 0; j < NCASES; j++) {
        GoodFeaturesArgs a;
        setup(jobs[j], CASES[j], j, j % 3 == 0 ? 0 : 5 + j, a);
        const int strips = (a.w + 31) / 32;
        gridDim.x = strips; gridDim.y = 1; gridDim.z = 1;
        for (int c = 0; c < strips; c++) emu::launch_cta(32, (unsigned)c, [&] { hv_gf_response_kernel(a); });
        gridDim.x = a.tilesX; gridDim.y = a.tilesY;
        for (int ty = 0; ty < a.tilesY; ty++) {
            emu::block_y = ty;
            for (int tx = 0; tx < a.tilesX; tx++) emu::launch_cta(GF_NT, (unsigned)tx, [&] { hv_gf_candidate_kernel(a); });
        }
        emu::block_y = 0;
        multiRound += jobs[j].words[1] > (unsigned)HV_GF_CHUNK;
        run_select(a, smem);
        fails += check("frame", jobs[j], a.response != nullptr);
    }
    static GoodFeaturesBatchArgs b;
    memset(&b, 0, sizeof(b));
    int tiles = 0, strips = 0;
    for (int j = 0; j < NCASES; j++) {
        setup(jobs[j], CASES[j], j, j % 3 == 1 ? 0 : 3, b.job[j]);
        b.firstTile[j] = tiles; b.firstStrip[j] = strips;
        tiles += b.job[j].tilesX * b.job[j].tilesY;
        strips += (b.job[j].w + 31) / 32;
    }
    for (int j = NCASES; j <= HV_CORNER_BATCH_MAX; j++) { b.firstTile[j] = tiles; b.firstStrip[j] = strips; }
    gridDim.x = strips; gridDim.y = 1;
    for (int c = 0; c < strips; c++) emu::launch_cta(32, (unsigned)c, [&] { hv_gf_response_batch_kernel(b); });
    gridDim.x = tiles;
    for (int c = 0; c < tiles; c++) emu::launch_cta(GF_NT, (unsigned)c, [&] { hv_gf_candidate_batch_kernel(b); });
    emu_dynamic_smem = (unsigned char*)smem.data();
    gridDim.x = NCASES;
    for (int c = 0; c < NCASES; c++) emu::launch_cta(GF_SEL_NT, (unsigned)c, [&] { hv_gf_select_batch_kernel(b); });
    for (int j = 0; j < NCASES; j++) fails += check("batch", jobs[j], b.job[j].response != nullptr);
    printf("cases with more candidates than one round holds: %d\n", multiRound);
    printf("%s\n", fails ? "FAIL" : "all ok");
    return fails ? 1 : 0;
}
