// tests/emu/emu_subpix.cpp -- the REAL body of hv_subpix_kernel (device part of hybvio_b200/csrc/subpix.cu: one warp per corner, patch and
// per-tap terms elementwise, five ordered sums in lanes 0..4) on the host emulator against the C oracle (oracle/hv_oracle_subpix.c, which
// restates cv::cornerSubPix): every refined corner bit-identical, over windows 1..15, zero zones, criteria, border and out-of-image
// starts. "subpix_device.inc" is cut out of subpix.cu by the test that builds this file (the `extern __shared__` array becomes a pointer).
#include "cuda_emu.h"
inline float2 make_float2(float x, float y) { return float2{x, y}; }
#include "subpix_device.inc"

extern "C" {
void orc_subpix_mask(int hw, int hh, int zw, int zh, float* mask);
int orc_subpix_refine(const uint8_t* img, int step, int w, int h, float* xy, int n, int hw, int hh, int zw, int zh, int criteria_type,
                      int max_count, double epsilon, int faults);
}

static unsigned hash2(int x, int y) { unsigned h = (unsigned)x * 374761393u + (unsigned)y * 668265263u; h = (h ^ (h >> 13)) * 1274126177u; return h ^ (h >> 16); }

// 8 x 8 blocks of random gray, box-blurred twice (smooth corners and edges), or a blurred checkerboard with 9-pixel squares
static std::vector<uint8_t> make_image(int w, int h, int kind)
{
    std::vector<float> a((size_t)w * h), b((size_t)w * h);
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++)
            a[(size_t)y * w + x] = kind == 0 ? (float)(hash2(x / 8, y / 8) & 0xff) : (((x / 9) + (y / 9)) & 1 ? 220.f : 30.f);
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
    // plus per-pixel noise, so that no two neighbouring rows or columns are equal (a patch row or column taken from the wrong source shows)
    std::vector<uint8_t> img((size_t)w * h);
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) img[(size_t)y * w + x] = (uint8_t)(a[(size_t)y * w + x] * 0.9f + (float)(hash2(x + 7, y + 11) & 15) + 0.5f);
    return img;
}

static int run(const char* name, int w, int h, int kind, int hw, int hh, int zw, int zh, int ctype, int maxCount, double eps, bool outside)
{
    std::vector<uint8_t> img = make_image(w, h, kind);
    // pitch wider than the width, as pyramid level 0 may have: bytes beyond the width must never be read into the result
    const int pitch = (w + 127) & ~127;
    std::vector<uint8_t> dev((size_t)pitch * (h + 1), 0xEE);
    for (int y = 0; y < h; y++) memcpy(dev.data() + (size_t)y * pitch, img.data() + (size_t)y * w, w);
    std::vector<float> xy;
    for (int i = 0; i < 24; i++) {                              // anywhere
        xy.push_back((hash2(i, 1) % 100000) * 1e-5f * w); xy.push_back((hash2(i, 2) % 100000) * 1e-5f * h);
    }
    for (int i = 0; i < 12; i++) {                              // within win + 1 of a border: the border patch path
        const float d = (hash2(i, 3) % 1000) * 1e-3f * (float)((i & 1 ? hw : hh) + 1);
        float x = (hash2(i, 4) % 100000) * 1e-5f * w, y = (hash2(i, 5) % 100000) * 1e-5f * h;
        switch (i & 3) { case 0: x = d; break; case 1: x = w - 1e-4f - d; break; case 2: y = d; break; default: y = h - 1e-4f - d; }
        xy.push_back(x); xy.push_back(y);
    }
    const float special[][2] = {{0.f, 0.f}, {(float)w - 1e-4f, (float)h - 1e-4f}, {9.f, 9.f}, {9.5f, 18.5f}, {18.f, 27.5f}, {(float)w - 1e-4f, 5.5f}};
    for (auto& s : special) { xy.push_back(s[0]); xy.push_back(s[1]); }
    const int nIn = (int)xy.size() / 2;
    std::vector<float> ref = xy;
    if (orc_subpix_refine(img.data(), w, w, h, ref.data(), nIn, hw, hh, zw, zh, ctype, maxCount, eps, 0) != 0) { printf("%s: oracle refused  FAIL\n", name); return 1; }
    if (outside) {                                             // the device entry point leaves corners outside the image unchanged
        const float o[][2] = {{-0.5f, 3.f}, {(float)w, 3.f}, {3.f, (float)h}, {3.f, -1e-6f}, {NAN, 5.f}};
        for (auto& p : o) { xy.push_back(p[0]); xy.push_back(p[1]); ref.push_back(p[0]); ref.push_back(p[1]); }
    }
    const int n = (int)xy.size() / 2;
    SubpixArgs a; memset(&a, 0, sizeof(a));
    a.gray = dev.data(); a.pitch = pitch; a.w = w; a.h = h; a.xy = (float2*)xy.data(); a.n = n; a.hw = hw; a.hh = hh;
    a.maxIters = 100;
    if (ctype & 1) a.maxIters = maxCount < 1 ? 1 : (maxCount > 100 ? 100 : maxCount);
    const double e = (ctype & 2) ? (eps < 0 ? 0 : eps) : 0;
    a.eps2 = e * e;
    orc_subpix_mask(hw, hh, zw, zh, a.mask);
    unsigned done = 0, flag = 0;
    a.done = HvDoneSignal{&done, (unsigned)n, 7, &flag};
    std::vector<unsigned char> smem(hv_subpix_smem_bytes(hw, hh) + 64, 0x5A);
    emu_dynamic_smem = (unsigned char*)(((uintptr_t)smem.data() + 15) & ~(uintptr_t)15);
    gridDim.x = n; gridDim.y = gridDim.z = 1;
    for (int p = 0; p < n; p++) emu::launch_cta(32, (unsigned)p, [&] { hv_subpix_kernel(a); });
    int bad = 0;
    for (int i = 0; i < 2 * n; i++) {
        if (memcmp(&xy[i], &ref[i], 4) != 0) { if (bad < 3) printf("  %s: coordinate %d: %.9g vs oracle %.9g\n", name, i, xy[i], ref[i]); bad++; }
    }
    const bool flagged = flag == 7 && done == (unsigned)n;
    printf("%s: %dx%d win %dx%d zero %dx%d crit %d/%d/%g: %d corners, %d differ, flag %s  %s\n", name, w, h, hw, hh, zw, zh, ctype, maxCount, eps, n, bad,
           flagged ? "raised" : "missing", bad == 0 && flagged ? "ok" : "FAIL");
    return bad == 0 && flagged ? 0 : 1;
}

int main()
{
    int fails = 0;
    fails += run("texture", 97, 61, 0, 5, 5, -1, -1, 3, 30, 0.01, true);
    fails += run("texture", 97, 61, 0, 1, 1, 0, 0, 1, 100, 0.0, false);
    fails += run("texture", 97, 61, 0, 2, 3, 1, 2, 2, 0, 0.0, false);
    fails += run("texture", 97, 61, 0, 7, 7, 7, 7, 1, 1, 0.0, false);
    fails += run("texture", 64, 48, 0, 11, 11, -1, -1, 3, 150, 1e-3, true);
    fails += run("texture", 40, 37, 0, 15, 15, 2, 1, 3, 20, 0.0, false);
    fails += run("checker", 96, 80, 1, 4, 4, -1, -1, 3, 40, 0.001, false);
    fails += run("checker", 96, 80, 1, 15, 13, 0, 0, 1, 0, 0.0, true);
    printf("%s\n", fails ? "FAIL" : "all ok");
    return fails ? 1 : 0;
}
