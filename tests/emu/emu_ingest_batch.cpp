// tests/emu/emu_ingest_batch.cpp -- the REAL hv_ingest_batch_kernel (hybvio_b200/csrc/ingest.cu: a flattened grid over the (job, row,
// 256-pixel block) triples, CTA b finds its job from the prefix sum `first` and runs colour only, remap only or colour + remap fused) on the
// host emulator: HV_CORNER_BATCH_MAX jobs of mixed modes, sizes, source strides, channel counts and coefficients in ONE emulated launch,
// the last of them the job with the most CTAs. Every level-0 image against the frame-ingest oracle (oracle/hv_oracle_gftt.c) bit for bit:
// orc_gray, orc_remap, and orc_remap(orc_gray(rgb), table) on the contiguous gray image for the fused mode; the destination's row padding
// stays as it was. "ingest_device.inc" is cut out of ingest.cu by the test that builds this file.
#include "cuda_emu.h"
#include "ingest_device.inc"

extern "C" {
void orc_gray(const uint8_t* src, int stride, int channels, int w, int h, const float* coeff, uint8_t* dst);
void orc_remap(const uint8_t* src, int stride, int w, int h, const HvRemapEntry* table, uint8_t* dst);
}

static unsigned hash2(int x, int y) { unsigned h = (unsigned)x * 374761393u + (unsigned)y * 668265263u; h = (h ^ (h >> 13)) * 1274126177u; return h ^ (h >> 16); }
static float frac(int i, int seed) { return (float)(hash2(i, seed) % 1000003u) / 1000003.0f; }

struct Case { int w, h, channels, table, pad, coeff; };   // pad: extra bytes per source row; coeff: 0 default, 1 sum above 1, 2 negative

// random table: taps anywhere, about 1 in 12 on the last column, the last row or the last pixel (non-zero fractions), 1 in 15 without a source
static std::vector<HvRemapEntry> make_table(int w, int h, int seed)
{
    std::vector<HvRemapEntry> t((size_t)w * h);
    for (int i = 0; i < w * h; i++) {
        HvRemapEntry& e = t[i];
        e.x0 = (short)(hash2(i, seed) % (unsigned)w); e.y0 = (short)(hash2(i, seed + 1) % (unsigned)h);
        e.xfrac = frac(i, seed + 2); e.yfrac = frac(i, seed + 3);
        switch (hash2(i, seed + 4) % 12) {
        case 0: e.x0 = (short)(w - 1); break;
        case 1: e.y0 = (short)(h - 1); break;
        case 2: e.x0 = (short)(w - 1); e.y0 = (short)(h - 1); break;
        default: break;
        }
        if (e.x0 == w - 1 || e.y0 == h - 1) { e.xfrac = 0.05f + 0.9f * e.xfrac; e.yfrac = 0.05f + 0.9f * e.yfrac; }
        if (hash2(i, seed + 5) % 15 == 0) e.x0 = HV_REMAP_INVALID;
    }
    return t;
}

int main()
{
    // crafted jobs: widths below, at and across 256 with every w % 4, all three modes, padded and dense strides, 1 .. 4 channels
    std::vector<Case> cases = {
        {1, 5, 3, 0, 0, 0},   {6, 4, 1, 1, 3, 0},   {255, 3, 4, 1, 0, 1}, {256, 2, 2, 0, 5, 2},  {257, 3, 1, 1, 0, 0},
        {258, 2, 3, 1, 7, 0}, {7, 9, 4, 0, 2, 1},   {13, 11, 2, 1, 0, 2}, {2, 6, 1, 1, 0, 0},    {300, 2, 4, 1, 1, 0},
        {513, 2, 1, 1, 9, 0}, {3, 3, 3, 1, 0, 1},   {1, 1, 1, 1, 0, 0},   {1, 4, 2, 1, 0, 0},    {514, 1, 3, 0, 0, 2},
    };
    // small filler jobs of random modes up to a full batch, then the job with the most CTAs last
    for (int j = (int)cases.size(); j < HV_CORNER_BATCH_MAX - 1; j++) {
        const unsigned r = hash2(j, 77);
        const int channels = 1 + (int)(r % 4), table = channels == 1 ? 1 : (int)((r >> 4) & 1);
        cases.push_back({1 + (int)(hash2(j, 78) % 40), 1 + (int)(hash2(j, 79) % 4), channels, table, (int)((r >> 8) % 4), (int)((r >> 12) % 3)});
    }
    cases.push_back({520, 40, 3, 1, 4, 0});
    const int njobs = (int)cases.size();
    if (njobs != HV_CORNER_BATCH_MAX) { printf("%d jobs  FAIL\n", njobs); return 1; }

    static IngestBatchArgs b;
    memset(&b, 0, sizeof(b));
    std::vector<std::vector<uint8_t>> src(njobs), dst(njobs), want(njobs);
    std::vector<std::vector<HvRemapEntry>> table(njobs);
    const float coeffs[3][4] = {{0.299f, 0.587f, 0.114f, 0.0f}, {0.9f, 0.8f, 0.7f, 0.6f}, {-0.35f, 1.3f, 0.45f, -0.2f}};
    int total = 0, maxCtas = 0;
    for (int j = 0; j < njobs; j++) {
        const Case& k = cases[j];
        const int w = k.w, h = k.h, c = k.channels;
        const int pitch = w * c + k.pad, dpitch = w % 4 == 0 ? w : (w + 127) / 128 * 128;     // level 0 of hv_pyr_create
        src[j].resize((size_t)pitch * (h - 1) + (size_t)w * c);                                // up to the last pixel, as staged
        for (size_t i = 0; i < src[j].size(); i++) src[j][i] = (uint8_t)(hash2((int)i, 1000 + j) & 0xff);
        dst[j].assign((size_t)dpitch * h, 0xEE);
        IngestJob& J = b.job[j];
        J.src = src[j].data(); J.srcPitch = pitch; J.channels = c;
        float cf[4];
        for (int i = 0; i < 4; i++) cf[i] = k.coeff == 0 || i < c ? coeffs[k.coeff][i] : 0.0f;   // as hv_ingest_frame resolves them
        memcpy(J.coeff, cf, sizeof(cf));
        if (k.table) table[j] = make_table(w, h, 31 * j);
        J.table = k.table ? table[j].data() : nullptr;
        J.dst = dst[j].data(); J.dstPitch = dpitch; J.w = w; J.h = h;
        b.first[j] = total;
        const int ctas = (w + 255) / 256 * h;
        total += ctas;
        if (j < njobs - 1 && ctas > maxCtas) maxCtas = ctas;
        // the oracle: gray of the frame, then the remap of that contiguous image (or of the gray frame at its own stride)
        std::vector<uint8_t> gray((size_t)w * h);
        if (c > 1) orc_gray(src[j].data(), pitch, c, w, h, cf, gray.data());
        want[j].resize((size_t)w * h);
        if (!k.table) want[j] = gray;
        else if (c > 1) orc_remap(gray.data(), w, w, h, table[j].data(), want[j].data());
        else orc_remap(src[j].data(), pitch, w, h, table[j].data(), want[j].data());
    }
    for (int j = njobs; j <= HV_CORNER_BATCH_MAX; j++) b.first[j] = total;
    if ((cases.back().w + 255) / 256 * cases.back().h <= maxCtas) { printf("the last job is not the largest  FAIL\n"); return 1; }

    gridDim.x = total; gridDim.y = gridDim.z = 1;
    for (int g = 0; g < total; g++) emu::launch_cta(256, (unsigned)g, [&] { hv_ingest_batch_kernel(b); });

    int fails = 0;
    for (int j = 0; j < njobs; j++) {
        const Case& k = cases[j];
        const int w = k.w, h = k.h, dpitch = b.job[j].dstPitch;
        int bad = 0, pad = 0;
        for (int y = 0; y < h; y++) {
            for (int x = 0; x < w; x++)
                if (dst[j][(size_t)y * dpitch + x] != want[j][(size_t)y * w + x]) {
                    if (bad < 3) printf("  job %d (%d, %d): %d vs oracle %d\n", j, x, y, dst[j][(size_t)y * dpitch + x], want[j][(size_t)y * w + x]);
                    bad++;
                }
            for (int x = w; x < dpitch; x++) pad += dst[j][(size_t)y * dpitch + x] != 0xEE;
        }
        const char* mode = k.table ? (k.channels > 1 ? "colour + remap" : "remap") : "colour";
        printf("job %d: %dx%d, %d channels, stride %d, %s, CTAs from %d: %d differ, %d padding bytes written  %s\n", j, w, h, k.channels,
               b.job[j].srcPitch, mode, b.first[j], bad, pad, bad || pad ? "FAIL" : "ok");
        fails += bad || pad;
    }
    printf("%s\n", fails ? "FAIL" : "all ok");
    return fails ? 1 : 0;
}
