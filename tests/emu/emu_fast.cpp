// tests/emu/emu_fast.cpp -- the REAL FAST kernels (hybvio_b200/csrc/fast.cu) on the host emulator against the cv::FAST oracle
// (oracle/hv_oracle_fast.c), bit for bit: count, (x, y), response, the HV_CORNER_NONE / 0 padding up to the capacity and an untouched
// float past it. Per frame (hv_fast_mark_kernel + hv_fast_scatter_kernel on a 2-D / 1-D grid) and batched (the two batch kernels over one
// flattened grid of all jobs) on images of different sizes and pitches -- widths that are no multiple of 4 or 32, images smaller than
// 7 x 7 -- with capacities above, below and at 0 of the count. "fast_device.inc" is cut out of fast.cu by the test that builds this file.
#include "cuda_emu.h"
#include "cuda_emu_ballot.h"
#define __constant__
inline int __popc(unsigned x) { return __builtin_popcount(x); }
inline float2 make_float2(float x, float y) { return float2{x, y}; }
#include "fast_device.inc"

extern "C" int orc_fast_detect(const uint8_t* img, int step, int w, int h, int threshold, int nonmax, float* out, int capacity);

static unsigned hash2(int x, int y) { unsigned h = (unsigned)x * 374761393u + (unsigned)y * 668265263u; h = (h ^ (h >> 13)) * 1274126177u; return h ^ (h >> 16); }

// kind 0: blurred noise, 1: raw noise, 2: checkerboard with noise, 3: flat
static std::vector<uint8_t> make_image(int w, int h, int kind, int seed)
{
    std::vector<uint8_t> img((size_t)w * h);
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            unsigned v = hash2(x + 1000 * seed, y);
            int p;
            if (kind == 0) {
                int s = 0;
                for (int d = 0; d < 4; d++) s += hash2(x / 3 + d % 2 + 1000 * seed, y / 3 + d / 2) & 0xff;
                p = s / 4 + (int)(v & 7);
            } else if (kind == 1) {
                p = v & 0xff;
            } else if (kind == 2) {
                p = (((x / 5) + (y / 5)) & 1 ? 200 : 40) + (int)(v % 9);
            } else {
                p = 90;
            }
            img[(size_t)y * w + x] = (uint8_t)(p > 255 ? 255 : p);
        }
    return img;
}

struct Job {
    int w, h, pitch;
    std::vector<uint8_t> dev;
    std::vector<float> ref;                 // oracle (x, y, response) x n
    int n;
    std::vector<unsigned> mask; std::vector<int> tileCount;
    std::vector<float> xy, resp;            // capacity + 1 slots (the last is a sentinel)
    int cap, count;
};

static void setup(Job& J, int w, int h, int kind, int seed, int threshold, int nonmax, int capMode, FastArgs& a)
{
    J.w = w; J.h = h;
    J.pitch = seed & 1 ? w : (w + 3) / 4 * 4 + 4 * (seed % 3);          // pitches differ from the width and from job to job
    const std::vector<uint8_t> img = make_image(w, h, kind, seed);
    J.dev.assign((size_t)J.pitch * h, 0xEE);
    for (int y = 0; y < h; y++) memcpy(J.dev.data() + (size_t)y * J.pitch, img.data() + (size_t)y * w, w);
    J.n = orc_fast_detect(img.data(), w, w, h, threshold, nonmax, nullptr, 0);
    J.ref.assign(3 * (size_t)J.n + 3, 0.f);
    orc_fast_detect(img.data(), w, w, h, threshold, nonmax, J.ref.data(), J.n);
    J.cap = capMode == 0 ? J.n + 7 : capMode == 1 ? J.n / 2 : 0;
    const int tx = (w + 31) / 32, ty = (h + 7) / 8;
    J.mask.assign((size_t)tx * ty * 8, 0xDEADBEEFu);
    J.tileCount.assign((size_t)tx * ty, -7);
    J.xy.assign(2 * (size_t)J.cap + 2, 777.f);
    J.resp.assign((size_t)J.cap + 1, 777.f);
    J.count = -1;
    memset(&a, 0, sizeof(a));
    a.gray = J.dev.data(); a.pitch = J.pitch; a.w = w; a.h = h;
    a.threshold = threshold < 0 ? 0 : (threshold > 255 ? 255 : threshold); a.nonmax = nonmax;
    a.tilesX = tx; a.tilesY = ty;
    a.mask = J.mask.data(); a.tileCount = J.tileCount.data();
    a.xy = (float2*)J.xy.data(); a.response = seed % 4 == 3 ? nullptr : J.resp.data(); a.capacity = J.cap; a.count = &J.count;
}

static int check(const char* what, Job& J, bool withResp)
{
    int bad = J.count != J.n;
    const int m = J.n < J.cap ? J.n : J.cap;
    for (int i = 0; i < J.cap; i++) {
        const float ex = i < m ? J.ref[3 * i] : HV_CORNER_NONE_F, ey = i < m ? J.ref[3 * i + 1] : HV_CORNER_NONE_F;
        const float er = i < m ? J.ref[3 * i + 2] : 0.f;
        if (memcmp(&J.xy[2 * i], &ex, 4) || memcmp(&J.xy[2 * i + 1], &ey, 4) || (withResp ? memcmp(&J.resp[i], &er, 4) != 0 : J.resp[i] != 777.f)) {
            if (bad < 3) printf("  slot %d: (%g, %g, %g) vs oracle (%g, %g, %g)\n", i, J.xy[2 * i], J.xy[2 * i + 1], J.resp[i], ex, ey, er);
            bad++;
        }
    }
    bad += J.xy[2 * J.cap] != 777.f || J.xy[2 * J.cap + 1] != 777.f || J.resp[J.cap] != 777.f;
    printf("%s %dx%d pitch %d: count %d (oracle %d), capacity %d: %d differ  %s\n", what, J.w, J.h, J.pitch, J.count, J.n, J.cap, bad, bad ? "FAIL" : "ok");
    return bad != 0;
}

static const int SIZES[][3] = {{97, 61, 0}, {64, 48, 1}, {6, 6, 1}, {7, 7, 1}, {130, 37, 2}, {33, 9, 0}, {45, 40, 3}, {8, 23, 1}, {161, 70, 0}};
static const int NJOBS = sizeof(SIZES) / sizeof(SIZES[0]);

static int run(int threshold, int nonmax)
{
    int fails = 0;
    std::vector<Job> jobs(NJOBS);
    // per frame: the two kernels of hv_launch_fast
    for (int j = 0; j < NJOBS; j++) {
        FastArgs a;
        setup(jobs[j], SIZES[j][0], SIZES[j][1], SIZES[j][2], j, threshold, nonmax, j % 3, a);
        gridDim.x = a.tilesX; gridDim.y = a.tilesY; gridDim.z = 1;
        for (int ty = 0; ty < a.tilesY; ty++) {
            emu::block_y = ty;
            for (int tx = 0; tx < a.tilesX; tx++) emu::launch_cta(FAST_NT, (unsigned)tx, [&] { hv_fast_mark_kernel(a); });
        }
        emu::block_y = 0;
        gridDim.x = a.tilesY; gridDim.y = 1;
        for (int b = 0; b < a.tilesY; b++) emu::launch_cta(FAST_NT, (unsigned)b, [&] { hv_fast_scatter_kernel(a); });
        char what[64];
        snprintf(what, sizeof(what), "frame t %d nonmax %d", threshold, nonmax);
        fails += check(what, jobs[j], a.response != nullptr);
    }
    // batched: every job in one flattened grid per kernel
    static FastBatchArgs b;
    memset(&b, 0, sizeof(b));
    int tiles = 0, bands = 0;
    for (int j = 0; j < NJOBS; j++) {
        setup(jobs[j], SIZES[j][0], SIZES[j][1], SIZES[j][2], j, threshold, nonmax, (j + 1) % 3, b.job[j]);
        b.firstTile[j] = tiles; b.firstBand[j] = bands;
        tiles += b.job[j].tilesX * b.job[j].tilesY; bands += b.job[j].tilesY;
    }
    for (int j = NJOBS; j <= HV_CORNER_BATCH_MAX; j++) { b.firstTile[j] = tiles; b.firstBand[j] = bands; }
    gridDim.x = tiles; gridDim.y = 1;
    for (int c = 0; c < tiles; c++) emu::launch_cta(FAST_NT, (unsigned)c, [&] { hv_fast_mark_batch_kernel(b); });
    gridDim.x = bands;
    for (int c = 0; c < bands; c++) emu::launch_cta(FAST_NT, (unsigned)c, [&] { hv_fast_scatter_batch_kernel(b); });
    for (int j = 0; j < NJOBS; j++) {
        char what[64];
        snprintf(what, sizeof(what), "batch job %d t %d nonmax %d", j, threshold, nonmax);
        fails += check(what, jobs[j], b.job[j].response != nullptr);
    }
    return fails;
}

int main()
{
    int fails = 0;
    fails += run(10, 1);
    fails += run(0, 1);
    fails += run(20, 0);
    fails += run(300, 1);
    printf("%s\n", fails ? "FAIL" : "all ok");
    return fails ? 1 : 0;
}
