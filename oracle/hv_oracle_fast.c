/* oracle/hv_oracle_fast.c -- TEST INFRASTRUCTURE: plain-C restatement of cv::FAST with FastFeatureDetector::TYPE_9_16 on an 8-bit
 * single-channel image (OCV/features2d/src/fast.cpp: FAST_t<16> and makeOffsets; OCV/features2d/src/fast_score.cpp: the scalar
 * cornerScore<16>), in OpenCV's order: the rows top to bottom, the columns left to right.
 *   - threshold clamped to [0, 255] (FAST_t: std::min(std::max(threshold, 0), 255)). FAST_t's vector loop loads its threshold as
 *     (char)threshold BEFORE that clamp, so cv2 outside [0, 255] tests most columns at threshold & 255 and the last few (where the
 *     vector loop ends, which depends on the build's SIMD width) at the clamped value; this restatement clamps everywhere;
 *   - candidates on [3, w - 3) x [3, h - 3): a pixel is a corner iff 9 contiguous pixels of its 16-pixel Bresenham circle of radius 3
 *     are all darker than v - threshold or all brighter than v + threshold (the prefilter of FAST_t is a necessary condition only);
 *   - nonmax: the score (cornerScore<16>) of every corner, 0 elsewhere and outside the candidate rectangle (FAST_t's zeroed row
 *     buffers), and a corner is kept iff its score is STRICTLY greater than each of its 8 neighbours'; the response is that score.
 *     Without suppression every corner is kept with response 0.
 * Output (x, y, response) as KeyPoint((float)j, (float)(i - 1), 7.f, -1, (float)score).
 */
#include <stdint.h>
#include <stdlib.h>

/* makeOffsets(pixel, step, 16): the circle as (dx, dy), starting below the centre and turning towards +x */
static const int OFFS16[16][2] = {{0, 3}, {1, 3}, {2, 2}, {3, 1}, {3, 0}, {3, -1}, {2, -2}, {1, -3},
                                  {0, -3}, {-1, -3}, {-2, -2}, {-3, -1}, {-3, 0}, {-3, 1}, {-2, 2}, {-1, 3}};

static int mini(int a, int b) { return a < b ? a : b; }
static int maxi(int a, int b) { return a > b ? a : b; }

/* FAST_t<16>'s segment test at (x, y): the k loop over N = 25 circle positions (the first 9 repeated) counting a run of > K = 8 */
static int orc_fast_is_corner(const uint8_t* img, int step, int x, int y, int threshold)
{
    const uint8_t* p = img + (size_t)y * step + x;
    const int v = p[0];
    for (int side = 0; side < 2; side++) {
        int count = 0;
        for (int k = 0; k < 25; k++) {
            const int q = p[OFFS16[k % 16][1] * step + OFFS16[k % 16][0]];
            if (side == 0 ? q < v - threshold : q > v + threshold) {
                if (++count > 8) return 1;
            } else {
                count = 0;
            }
        }
    }
    return 0;
}

/* cornerScore<16> (fast_score.cpp, the scalar branch) */
int orc_fast_score(const uint8_t* img, int step, int x, int y, int threshold)
{
    const uint8_t* p = img + (size_t)y * step + x;
    const int v = p[0];
    int d[25];
    for (int k = 0; k < 25; k++) d[k] = v - p[OFFS16[k % 16][1] * step + OFFS16[k % 16][0]];
    int a0 = threshold;
    for (int k = 0; k < 16; k += 2) {
        int a = mini(d[k + 1], d[k + 2]);
        a = mini(a, d[k + 3]);
        if (a <= a0) continue;
        a = mini(a, d[k + 4]);
        a = mini(a, d[k + 5]);
        a = mini(a, d[k + 6]);
        a = mini(a, d[k + 7]);
        a = mini(a, d[k + 8]);
        a0 = maxi(a0, mini(a, d[k]));
        a0 = maxi(a0, mini(a, d[k + 9]));
    }
    int b0 = -a0;
    for (int k = 0; k < 16; k += 2) {
        int b = maxi(d[k + 1], d[k + 2]);
        b = maxi(b, d[k + 3]);
        b = maxi(b, d[k + 4]);
        b = maxi(b, d[k + 5]);
        if (b >= b0) continue;
        b = maxi(b, d[k + 6]);
        b = maxi(b, d[k + 7]);
        b = maxi(b, d[k + 8]);
        b0 = mini(b0, maxi(b, d[k]));
        b0 = mini(b0, maxi(b, d[k + 9]));
    }
    return -b0 - 1;
}

/* cv::FAST(img, kp, threshold, nonmax, TYPE_9_16): writes the first `capacity` keypoints as (x, y, response) to out and returns the
 * full count, or -1 when the scratch cannot be allocated. step: the row pitch in bytes. */
int orc_fast_detect(const uint8_t* img, int step, int w, int h, int threshold, int nonmax, float* out, int capacity)
{
    threshold = threshold < 0 ? 0 : (threshold > 255 ? 255 : threshold);
    if (w < 7 || h < 7) return 0;
    /* the score of every pixel: 0 off the candidate rectangle and where the segment test fails; a corner's score is >= threshold, so a
     * corner of score 0 (threshold 0) is marked apart from the non-corners */
    int* score = (int*)calloc((size_t)w * h, sizeof(int));
    uint8_t* corner = (uint8_t*)calloc((size_t)w * h, 1);
    if (!score || !corner) { free(score); free(corner); return -1; }
    for (int y = 3; y < h - 3; y++)
        for (int x = 3; x < w - 3; x++)
            if (orc_fast_is_corner(img, step, x, y, threshold)) {
                corner[(size_t)y * w + x] = 1;
                if (nonmax) score[(size_t)y * w + x] = orc_fast_score(img, step, x, y, threshold);
            }
    int n = 0;
    for (int y = 3; y < h - 3; y++)
        for (int x = 3; x < w - 3; x++) {
            if (!corner[(size_t)y * w + x]) continue;
            const int s = score[(size_t)y * w + x];
            int keep = 1;
            if (nonmax)
                for (int dy = -1; dy <= 1 && keep; dy++)
                    for (int dx = -1; dx <= 1; dx++) {
                        if (!dx && !dy) continue;
                        const int t = score[(size_t)(y + dy) * w + x + dx];
                        if (s <= t) { keep = 0; break; }
                    }
            if (!keep) continue;
            if (n < capacity) { out[3 * n] = (float)x; out[3 * n + 1] = (float)y; out[3 * n + 2] = (float)s; }
            n++;
        }
    free(score);
    free(corner);
    return n;
}

