// tests/emu/emu_lk.cpp -- the REAL bodies of the Lucas-Kanade kernels (hybvio_b200/csrc/lk.cu: CTA-per-feature hv_lk_cta_kernel<WIN> and
// warp-per-feature hv_lk_kernel<WIN>, WIN = 11, 15, 21, 31) on the host emulator against the C oracle in the kernels' own accumulation order
// (oracle/hv_oracle_lk.c, accum_mode 1: bit-exact end points and statuses). "lk_device.inc" is the device part of lk.cu (everything
// before the host launcher), cut out by the test that builds this file. Test infrastructure; also run under ThreadSanitizer.
#include <algorithm>
#include "cuda_emu.h"
#include "lk_device.inc"

extern "C" {
struct orc_pyramid;
orc_pyramid* orc_pyr_create(const uint8_t* img, int w, int h, int stride, int win, int maxLevel);
int orc_pyr_levels(const orc_pyramid* p);
void orc_pyr_level_size(const orc_pyramid* p, int level, int* w, int* h);
void orc_pyr_get_level_padded(const orc_pyramid* p, int level, uint8_t* gray, int16_t* deriv);
void orc_pyr_free(orc_pyramid* p);
int orc_lk(const orc_pyramid* prev, const orc_pyramid* next, const float* prevPts, float* nextPts, uint8_t* status, int n, int maxLevel, int maxIter, double eps,
           int useInitial, double minEig, int accum_mode);
}

static unsigned hash2(int x, int y, unsigned seed) { unsigned h = (unsigned)x * 374761393u + (unsigned)y * 668265263u + seed * 2246822519u; h = (h ^ (h >> 13)) * 1274126177u; return h ^ (h >> 16); }
// smooth value noise (3 octaves), sampled at a sub-pixel offset: the second image is the first one shifted
static double tex(double u, double v)
{
    double s = 128.0;
    const int cell[3] = {6, 17, 48}; const double amp[3] = {70, 50, 35};
    for (int o = 0; o < 3; o++) {
        const double x = u / cell[o], y = v / cell[o]; const int xi = (int)std::floor(x), yi = (int)std::floor(y); const double fx = x - xi, fy = y - yi;
        auto val = [&](int a, int b) { return (hash2(a, b, 42 + o) & 0xffff) / 65535.0 - 0.5; };
        const double top = val(xi, yi) * (1 - fx) + val(xi + 1, yi) * fx, bot = val(xi, yi + 1) * (1 - fx) + val(xi + 1, yi + 1) * fx;
        s += amp[o] * (top * (1 - fy) + bot * fy);
    }
    return s < 0 ? 0 : s > 255 ? 255 : s;
}

struct DevPyr { std::vector<std::vector<uint8_t>> gray; std::vector<std::vector<short2>> deriv; HvPyrDesc desc; };

static void to_device_layout(const orc_pyramid* p, int win, DevPyr& d)
{
    memset(&d.desc, 0, sizeof(d.desc));
    d.desc.nlevels = orc_pyr_levels(p); d.desc.win = win;
    d.gray.resize(d.desc.nlevels); d.deriv.resize(d.desc.nlevels);
    for (int lv = 0; lv < d.desc.nlevels; lv++) {
        int w, h; orc_pyr_level_size(p, lv, &w, &h);
        const int pw = w + 2 * win, ph = h + 2 * win;
        std::vector<uint8_t> g((size_t)pw * ph); std::vector<int16_t> dd((size_t)pw * ph * 2);
        orc_pyr_get_level_padded(p, lv, g.data(), dd.data());
        const int gp = lv == 0 && w % 4 == 0 ? w : (w + 127) & ~127, dp = (w + 31) & ~31;
        d.gray[lv].assign((size_t)gp * h + 16, 0); d.deriv[lv].assign((size_t)dp * h + 16, short2{0, 0});
        for (int y = 0; y < h; y++) for (int x = 0; x < w; x++) {
            d.gray[lv][(size_t)y * gp + x] = g[(size_t)(y + win) * pw + x + win];
            d.deriv[lv][(size_t)y * dp + x] = short2{dd[((size_t)(y + win) * pw + x + win) * 2], dd[((size_t)(y + win) * pw + x + win) * 2 + 1]};
        }
        HvLevel& L = d.desc.lv[lv];
        L.gray = d.gray[lv].data(); L.deriv = d.deriv[lv].data(); L.w = w; L.h = h; L.gpitch = gp; L.dpitch = dp;
    }
}

template <int WIN>
static int run_window(const std::vector<uint8_t>& a, const std::vector<uint8_t>& b, int W, int H, const std::vector<float>& prev,
                      const std::vector<float>& init, int N)
{
    const int MAXL = 3;
    orc_pyramid* pa = orc_pyr_create(a.data(), W, H, W, WIN, MAXL);
    orc_pyramid* pb = orc_pyr_create(b.data(), W, H, W, WIN, MAXL);
    DevPyr da, db; to_device_layout(pa, WIN, da); to_device_layout(pb, WIN, db);
    HvPyrDesc table[2] = {da.desc, db.desc};
    int fails = 0;
    for (int useInitial = 0; useInitial < 2; useInitial++) for (int variant = 0; variant < 3; variant++) {
        if (variant == 2 && WIN != 31) continue;
        std::vector<float> onext = init, knext = init; std::vector<uint8_t> ost(N), kst(N, 7); std::vector<int32_t> kts(N, -1);
        orc_lk(pa, pb, prev.data(), onext.data(), ost.data(), N, MAXL, 20, 0.03, useInitial, 1e-3, 1);
        LkLaunch L; memset(&L, 0, sizeof(L));
        L.table = table; L.njobs = 1; L.prefetch = 1; L.maxLevel = MAXL; L.maxIter = 20; L.eps2 = 0.03 * 0.03; L.minEig = 1e-3f;
        L.jobs[0].prevIdx = 0; L.jobs[0].nextIdx = 1; L.jobs[0].n = N; L.jobs[0].useInitial = useInitial;
        L.jobs[0].prevPts = (const float2*)prev.data(); L.jobs[0].nextPts = (float2*)knext.data(); L.jobs[0].status = kst.data(); L.jobs[0].trackStatus = kts.data();
        if (variant == 0) {
            gridDim.x = N; gridDim.y = 1;
            for (int f = 0; f < N; f++) emu::launch_cta(LKC_NW * 32, (unsigned)f, [&] { hv_lk_cta_kernel<WIN>(L); });
        } else if (variant == 2) {                                    // 8 warps per feature (HV_LK_CTA_WARPS=8): 4 window rows per warp, the last warp owns 3
            gridDim.x = N; gridDim.y = 1;
            for (int f = 0; f < N; f++) emu::launch_cta(8 * 32, (unsigned)f, [&] { hv_lk_cta_kernel<WIN, 8>(L); });
        } else {
            const int ctas = (N + LK_WARPS_PER_CTA - 1) / LK_WARPS_PER_CTA;
            gridDim.x = ctas; gridDim.y = 1;
            for (int c = 0; c < ctas; c++) emu::launch_cta(LK_WARPS_PER_CTA * 32, (unsigned)c, [&] { hv_lk_kernel<WIN>(L); });
        }
        int bad = 0, tracked = 0;
        for (int i = 0; i < N; i++) {
            tracked += ost[i];
            const bool same = kst[i] == ost[i] && memcmp(&knext[2 * i], &onext[2 * i], 8) == 0;
            if (!same) { bad++; if (bad < 4) printf("  feature %d: kernel (%g, %g) st %d, oracle (%g, %g) st %d\n", i, knext[2 * i], knext[2 * i + 1], kst[i], onext[2 * i], onext[2 * i + 1], ost[i]); }
        }
        printf("%s<%d%s>, useInitial=%d: %d features, %d tracked, %d differ from the oracle (bit-exact end points + status)  %s\n",
               variant == 1 ? "hv_lk_kernel" : "hv_lk_cta_kernel", WIN, variant == 2 ? ", 8" : "", useInitial, N, tracked, bad, bad == 0 ? "ok" : "FAIL");
        fails += bad != 0;
    }
    orc_pyr_free(pa); orc_pyr_free(pb);
    return fails;
}

int main()
{
    const int W = 320, H = 240, N = 40;
    std::vector<uint8_t> a((size_t)W * H), b((size_t)W * H);
    for (int y = 0; y < H; y++) for (int x = 0; x < W; x++) {
        a[(size_t)y * W + x] = (uint8_t)std::lrint(tex(x, y));
        b[(size_t)y * W + x] = (uint8_t)std::lrint(tex(x - 2.3, y + 1.7));          // content moves by (+2.3, -1.7) px
    }
    for (int y = 100; y < 150; y++) for (int x = 200; x < 260; x++) a[(size_t)y * W + x] = b[(size_t)y * W + x] = 90;     // flat patch: minEig rejection
    srand(7);
    std::vector<float> prev(2 * N), init(2 * N);
    for (int i = 0; i < N; i++) {
        prev[2 * i] = (float)(-5 + (rand() / (double)RAND_MAX) * (W + 10)); prev[2 * i + 1] = (float)(-5 + (rand() / (double)RAND_MAX) * (H + 10));     // incl. points outside the image
        if (i % 8 == 5) { prev[2 * i] = 230.5f; prev[2 * i + 1] = 125.25f; }                                                                          // on the flat patch
        init[2 * i] = prev[2 * i] + 2.3f + (float)((rand() / (double)RAND_MAX) * 6 - 3); init[2 * i + 1] = prev[2 * i + 1] - 1.7f + (float)((rand() / (double)RAND_MAX) * 6 - 3);
    }
    // every window size the launcher dispatches (hv_launch_lk: 11, 15, 21, 31)
    return run_window<31>(a, b, W, H, prev, init, N) + run_window<21>(a, b, W, H, prev, init, N) + run_window<15>(a, b, W, H, prev, init, N) +
           run_window<11>(a, b, W, H, prev, init, N);
}
