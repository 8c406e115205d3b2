// tests/emu/emu_subpix_batch.cpp -- the REAL hv_subpix_batch_kernel (hybvio_b200/csrc/subpix.cu: a flattened grid over the (job, point)
// pairs, CTA g finds its job from the prefix sum `first` and runs the corner body of hv_subpix_kernel on that job's image) on the host
// emulator: jobs on images of different sizes and pitches, with 0 .. 40 points each (empty jobs first, in the middle and last), in ONE
// emulated launch per window. Every refined corner against the cv::cornerSubPix oracle (oracle/hv_oracle_subpix.c) bit for bit; the
// padding points (HV_CORNER_NONE) stay as they are. "subpix_device.inc" is cut out of subpix.cu by the test that builds this file.
#include "cuda_emu.h"
inline float2 make_float2(float x, float y) { return float2{x, y}; }
#include "subpix_device.inc"

extern "C" {
void orc_subpix_mask(int hw, int hh, int zw, int zh, float* mask);
int orc_subpix_refine(const uint8_t* img, int step, int w, int h, float* xy, int n, int hw, int hh, int zw, int zh, int criteria_type,
                      int max_count, double epsilon, int faults);
}

static unsigned hash2(int x, int y) { unsigned h = (unsigned)x * 374761393u + (unsigned)y * 668265263u; h = (h ^ (h >> 13)) * 1274126177u; return h ^ (h >> 16); }

// smooth random blocks plus per-pixel noise (corners and edges for the refinement to find)
static std::vector<uint8_t> make_image(int w, int h, int seed)
{
    std::vector<float> a((size_t)w * h), b((size_t)w * h);
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) a[(size_t)y * w + x] = (float)(hash2(x / 7 + seed, y / 7) & 0xff);
    for (int pass = 0; pass < 2; pass++) {
        for (int y = 0; y < h; y++)
            for (int x = 0; x < w; x++) {
                float s = 0; int c = 0;
                for (int dy = -1; dy <= 1; dy++) for (int dx = -1; dx <= 1; dx++) {
                    const int xx = x + dx, yy = y + dy;
                    if (xx >= 0 && xx < w && yy >= 0 && yy < h) { s += a[(size_t)yy * w + xx]; c++; }
                }
                b[(size_t)y * w + x] = s / c;
            }
        a.swap(b);
    }
    std::vector<uint8_t> img((size_t)w * h);
    for (int i = 0; i < w * h; i++) img[i] = (uint8_t)(a[i] * 0.9f + (float)(hash2(i, seed) & 15) + 0.5f);
    return img;
}

static int run(int hw, int hh, int zw, int zh, int ctype, int maxCount, double eps)
{
    const int sizes[][3] = {{97, 61, 0}, {64, 48, 10}, {40, 37, 0}, {96, 80, 5}, {120, 70, 40}, {33, 35, 12}, {80, 80, 1}, {51, 49, 0}};
    const int njobs = 8;
    std::vector<std::vector<uint8_t>> img(njobs), dev(njobs);
    std::vector<std::vector<float>> xy(njobs), ref(njobs);
    static SubpixBatchArgs b;
    memset(&b, 0, sizeof(b));
    int total = 0;
    for (int j = 0; j < njobs; j++) {
        const int w = sizes[j][0], h = sizes[j][1], n = sizes[j][2];
        img[j] = make_image(w, h, 3 * j + hw);
        const int pitch = j & 1 ? w : (w + 127) & ~127;              // pitches differ from job to job
        dev[j].assign((size_t)pitch * (h + 1), 0xEE);
        for (int y = 0; y < h; y++) memcpy(dev[j].data() + (size_t)y * pitch, img[j].data() + (size_t)y * w, w);
        for (int i = 0; i < n; i++) {
            float x = (hash2(i, 10 + j) % 100000) * 1e-5f * w, y = (hash2(i, 20 + j) % 100000) * 1e-5f * h;
            if (i % 5 == 1) x = (hash2(i, 30 + j) % 1000) * 1e-3f * (float)(hw + 1);            // near the left border
            if (i % 5 == 2) y = h - 1e-4f - (hash2(i, 40 + j) % 1000) * 1e-3f * (float)(hh + 1);  // near the bottom
            xy[j].push_back(x); xy[j].push_back(y);
        }
        ref[j] = xy[j];
        if (n > 0 && orc_subpix_refine(img[j].data(), w, w, h, ref[j].data(), n, hw, hh, zw, zh, ctype, maxCount, eps, 0) != 0) {
            printf("job %d: oracle refused  FAIL\n", j);
            return 1;
        }
        if (n > 0)
            for (int k = 0; k < 3; k++) { xy[j].push_back(-1.0e6f); xy[j].push_back(-1.0e6f); ref[j].push_back(-1.0e6f); ref[j].push_back(-1.0e6f); }
        xy[j].push_back(777.f);                                       // one float past the job's points: never written
        b.job[j] = SubpixJob{dev[j].data(), pitch, w, h, (float2*)xy[j].data(), (int)(xy[j].size() / 2)};
        b.first[j] = total;
        total += b.job[j].n;
    }
    for (int j = njobs; j <= HV_CORNER_BATCH_MAX; j++) b.first[j] = total;
    SubpixArgs& s = b.s;
    s.hw = hw; s.hh = hh;
    s.maxIters = 100;
    if (ctype & 1) s.maxIters = maxCount < 1 ? 1 : (maxCount > 100 ? 100 : maxCount);
    const double e = (ctype & 2) ? (eps < 0 ? 0 : eps) : 0;
    s.eps2 = e * e;
    orc_subpix_mask(hw, hh, zw, zh, s.mask);
    std::vector<unsigned char> smem(hv_subpix_smem_bytes(hw, hh) + 64, 0x5A);
    emu_dynamic_smem = (unsigned char*)(((uintptr_t)smem.data() + 15) & ~(uintptr_t)15);
    gridDim.x = total; gridDim.y = gridDim.z = 1;
    for (int g = 0; g < total; g++) emu::launch_cta(32, (unsigned)g, [&] { hv_subpix_batch_kernel(b); });
    int fails = 0;
    for (int j = 0; j < njobs; j++) {
        int bad = 0;
        for (size_t i = 0; i < ref[j].size(); i++)
            if (memcmp(&xy[j][i], &ref[j][i], 4) != 0) { if (bad < 3) printf("  job %d coordinate %zu: %.9g vs oracle %.9g\n", j, i, xy[j][i], ref[j][i]); bad++; }
        bad += xy[j].back() != 777.f;
        printf("win %dx%d job %d: %dx%d, %d points from CTA %d: %d differ  %s\n", hw, hh, j, b.job[j].w, b.job[j].h, b.job[j].n, b.first[j], bad,
               bad ? "FAIL" : "ok");
        fails += bad != 0;
    }
    return fails;
}

int main()
{
    int fails = 0;
    fails += run(5, 5, -1, -1, 3, 30, 0.01);
    fails += run(3, 2, 1, 0, 1, 10, 0.0);
    printf("%s\n", fails ? "FAIL" : "all ok");
    return fails ? 1 : 0;
}
