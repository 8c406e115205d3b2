/* oracle/hv_oracle_good_features.c -- TEST INFRASTRUCTURE: plain-C restatement of
 *   cv::goodFeaturesToTrack(img, corners, maxCorners, qualityLevel, minDistance, mask, cornersQuality,
 *                           blockSize = 3, gradientSize = 3, useHarrisDetector = false)
 * on an 8-bit single-channel image (OCV/imgproc/src/featureselect.cpp, CPU path), in OpenCV's operation order:
 *   1. eig = cornerMinEigenVal(img, 3, 3) (OCV/imgproc/src/corner.cpp), BORDER_REFLECT_101 everywhere:
 *      - Sobel 8U -> 32F with scale s = 1 / (4 * 3 * 255) folded into the smoothing kernel ([1 2 1] * s as fp32: k1 = (float)s, k0 = 2 k1).
 *        The row pass goes through RowFilter<uchar, float> (filter.simd.hpp): ((k[0] S0 + k[1] S1) + k[2] S2), each product rounded.
 *        The column pass is SymmColumnSmallFilter<float>: symmetric S1 k0 + (S0 + S2) k1, antisymmetric [-1 0 1] S2 - S0.
 *          dx: row [-1 0 1] (exact), column [s 2s s];  dy: row [s 2s s], column [-1 0 1]
 *      - cov = (dx dx, dx dy, dy dy) in fp32;
 *      - boxFilter(cov, 3 x 3, normalize = false) on CV_32FC3 (box_filter.simd.hpp): RowSum<float, double> with ksize 3 forms
 *        R = ((c[x - 1] + c[x]) + c[x + 1]) in double per row (reflect-101 columns); ColumnSum<double, float> then keeps ONE running
 *        double sum per column, from the top of the image down: SUM = (0 + R[-1]) + R[0], and for y = 0, 1, ...:
 *        s0 = SUM + R[y + 1], out[y] = (float)s0, SUM = s0 - R[y - 1] (rows reflect-101). The sum is not the exact 9-term sum: dy can be
 *        rounding noise far below 1/3060, and the running sum carries the rounding of the rows above;
 *      - calcMinEigenVal: a = c0 / 2, b = c1, c = c2 / 2, (a + c) - sqrt((a - c)^2 + b^2) in fp32.
 *   2. maxVal = max of eig over the mask's non-zero pixels (0 when the mask selects no pixel).
 *   3. threshold TOZERO at (float)(maxVal * qualityLevel): v is kept iff v > thresh in fp32.
 *   4. - 5. candidates: 1 <= x < w - 1, 1 <= y < h - 1, v != 0, v == max of the thresholded 3 x 3 neighbourhood, mask non-zero.
 *   6. sort by greaterThanPtr: response descending, ties by descending pixel address (y w + x).
 *   7. minDistance >= 1: OpenCV's greedy grid filter (cell cvRound(minDistance), +-1 cell, (float)dx^2 + (float)dy^2 < minDistance^2 in
 *      double); otherwise the first maxCorners candidates. Stops at maxCorners (> 0).
 * Built with -ffp-contract=off, so no multiply-add is contracted.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static int refl101(int p, int len)
{
    if (len == 1) return 0;
    while (p < 0 || p >= len) p = p < 0 ? -p : 2 * len - 2 - p;
    return p;
}

/* cv::Sobel(img, CV_32F, 1, 0, 3, s) and cv::Sobel(img, CV_32F, 0, 1, 3, s), s = 1 / 3060 (cornerMinEigenVal's scale) */
void orc_gf_sobel(const uint8_t* img, int step, int w, int h, float* dx, float* dy)
{
    const float k1 = (float)(1.0 / 3060.0), k0 = 2.0f * k1, zero = 0.0f;
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const int xl = refl101(x - 1, w), xr = refl101(x + 1, w);
            const int rows[3] = {refl101(y - 1, h), y, refl101(y + 1, h)};
            float rdx[3], rdy[3];
            for (int r = 0; r < 3; r++) {
                const uint8_t* p = img + (size_t)rows[r] * step;
                const float S0 = p[xl], S1 = p[x], S2 = p[xr];
                float t = -1.0f * S0; t = t + zero * S1; t = t + 1.0f * S2;
                rdx[r] = t;
                float u = k1 * S0; u = u + k0 * S1; u = u + k1 * S2;
                rdy[r] = u;
            }
            const float a = rdx[1] * k0, b = (rdx[0] + rdx[2]) * k1;
            dx[(size_t)y * w + x] = (a + b) + zero;
            dy[(size_t)y * w + x] = (rdy[2] - rdy[0]) + zero;
        }
}

/* cv::boxFilter(cov, out, CV_32F, Size(3, 3), Point(-1, -1), false, BORDER_REFLECT_101) on a w x h CV_32FC3 image (3 floats per pixel,
 * rows of 3 w floats); returns -1 when the scratch cannot be allocated */
int orc_gf_box(const float* cov, int w, int h, float* out)
{
    double* R = (double*)malloc((size_t)3 * w * h * sizeof(double));
    if (!R) return -1;
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const float* r = cov + (size_t)3 * y * w;
            const int xl = refl101(x - 1, w), xr = refl101(x + 1, w);
            for (int k = 0; k < 3; k++)
                R[((size_t)y * w + x) * 3 + k] = ((double)r[3 * xl + k] + (double)r[3 * x + k]) + (double)r[3 * xr + k];
        }
    for (int x = 0; x < w; x++)
        for (int k = 0; k < 3; k++) {
#define ROW(j) R[((size_t)refl101(j, h) * w + x) * 3 + k]
            double sum = 0.0;
            sum += ROW(-1);
            sum += ROW(0);
            for (int y = 0; y < h; y++) {
                const double s0 = sum + ROW(y + 1);
                out[((size_t)y * w + x) * 3 + k] = (float)s0;
                sum = s0 - ROW(y - 1);
            }
#undef ROW
        }
    free(R);
    return 0;
}

/* cv::cornerMinEigenVal(img, eig, 3, 3); returns -1 when the scratch cannot be allocated */
int orc_gf_eig(const uint8_t* img, int step, int w, int h, float* eig)
{
    const size_t n = (size_t)w * h;
    float* dx = (float*)malloc(n * sizeof(float));
    float* dy = (float*)malloc(n * sizeof(float));
    float* cov = (float*)malloc(3 * n * sizeof(float));
    float* box = (float*)malloc(3 * n * sizeof(float));
    if (!dx || !dy || !cov || !box) { free(dx); free(dy); free(cov); free(box); return -1; }
    orc_gf_sobel(img, step, w, h, dx, dy);
    for (size_t i = 0; i < n; i++) {
        cov[3 * i] = dx[i] * dx[i];
        cov[3 * i + 1] = dx[i] * dy[i];
        cov[3 * i + 2] = dy[i] * dy[i];
    }
    if (orc_gf_box(cov, w, h, box) != 0) { free(dx); free(dy); free(cov); free(box); return -1; }
    for (size_t i = 0; i < n; i++) {
        const float a = box[3 * i] * 0.5f, b = box[3 * i + 1], c = box[3 * i + 2] * 0.5f;
        const float t = a - c, tt = t * t, bb = b * b, r = sqrtf(tt + bb);
        eig[i] = (a + c) - r;
    }
    free(dx); free(dy); free(cov); free(box);
    return 0;
}

typedef struct { float v; int idx; } orc_gf_cand;

/* greaterThanPtr: descending value, ties by descending address */
static int cand_cmp(const void* pa, const void* pb)
{
    const orc_gf_cand* a = (const orc_gf_cand*)pa;
    const orc_gf_cand* b = (const orc_gf_cand*)pb;
    if (a->v > b->v) return -1;
    if (a->v < b->v) return 1;
    return a->idx > b->idx ? -1 : (a->idx < b->idx ? 1 : 0);
}

/* cv::goodFeaturesToTrack(img, corners, maxCorners, q, minDistance, mask, cornersQuality, 3, 3, false): writes the first `capacity`
 * corners as (x, y, response) to out and returns the list's length, or -1 when the scratch cannot be allocated. mask: NULL or w x h u8
 * with row stride mstride. maxCorners <= 0: no limit (as OpenCV). */
int orc_gf_detect(const uint8_t* img, int step, int w, int h, int maxCorners, double q, double minDistance, const uint8_t* mask,
                  int mstride, float* out, int capacity)
{
    if (w < 1 || h < 1) return 0;
    const size_t n = (size_t)w * h;
    float* eig = (float*)malloc(n * sizeof(float));
    orc_gf_cand* cand = (orc_gf_cand*)malloc(n * sizeof(orc_gf_cand));
    if (!eig || !cand || orc_gf_eig(img, step, w, h, eig) != 0) { free(eig); free(cand); return -1; }
    float maxVal = 0.f;
    int any = 0;
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++)
            if (!mask || mask[(size_t)y * mstride + x]) {
                const float v = eig[(size_t)y * w + x];
                if (!any || v > maxVal) maxVal = v;
                any = 1;
            }
    const float thresh = (float)((double)maxVal * q);
    for (size_t i = 0; i < n; i++) eig[i] = eig[i] > thresh ? eig[i] : 0.0f;
    size_t total = 0;
    for (int y = 1; y < h - 1; y++)
        for (int x = 1; x < w - 1; x++) {
            const float v = eig[(size_t)y * w + x];
            if (v == 0.0f || (mask && !mask[(size_t)y * mstride + x])) continue;
            float m = v;
            for (int dyy = -1; dyy <= 1; dyy++)
                for (int dxx = -1; dxx <= 1; dxx++) {
                    const float u = eig[(size_t)(y + dyy) * w + x + dxx];
                    if (u > m) m = u;
                }
            if (v == m) { cand[total].v = v; cand[total].idx = y * w + x; total++; }
        }
    qsort(cand, total, sizeof(orc_gf_cand), cand_cmp);
    int ncorners = 0;
    if (minDistance >= 1) {
        const int cell = (int)lrint(minDistance);
        const int gw = (w + cell - 1) / cell, gh = (h + cell - 1) / cell;
        /* the kept corners of each cell as a linked list (head: the latest, next: the one kept before it in that cell) */
        int* head = (int*)malloc((size_t)gw * gh * sizeof(int));
        int* next = (int*)malloc((total ? total : 1) * sizeof(int));
        float* kx = (float*)malloc((total ? total : 1) * sizeof(float));
        float* ky = (float*)malloc((total ? total : 1) * sizeof(float));
        if (!head || !next || !kx || !ky) { free(head); free(next); free(kx); free(ky); free(eig); free(cand); return -1; }
        for (int i = 0; i < gw * gh; i++) head[i] = -1;
        const double md2 = minDistance * minDistance;
        for (size_t i = 0; i < total; i++) {
            const int y = cand[i].idx / w, x = cand[i].idx - y * w;
            const int xc = x / cell, yc = y / cell;
            const int x1 = xc - 1 < 0 ? 0 : xc - 1, y1 = yc - 1 < 0 ? 0 : yc - 1;
            const int x2 = xc + 1 > gw - 1 ? gw - 1 : xc + 1, y2 = yc + 1 > gh - 1 ? gh - 1 : yc + 1;
            int good = 1;
            for (int yy = y1; yy <= y2 && good; yy++)
                for (int xx = x1; xx <= x2 && good; xx++)
                    for (int k = head[yy * gw + xx]; k >= 0; k = next[k]) {
                        const float ddx = (float)x - kx[k], ddy = (float)y - ky[k];
                        if ((double)(ddx * ddx + ddy * ddy) < md2) { good = 0; break; }
                    }
            if (!good) continue;
            kx[ncorners] = (float)x; ky[ncorners] = (float)y;
            next[ncorners] = head[yc * gw + xc]; head[yc * gw + xc] = ncorners;
            if (ncorners < capacity) { out[3 * ncorners] = (float)x; out[3 * ncorners + 1] = (float)y; out[3 * ncorners + 2] = cand[i].v; }
            ncorners++;
            if (maxCorners > 0 && ncorners == maxCorners) break;
        }
        free(head); free(next); free(kx); free(ky);
    } else {
        for (size_t i = 0; i < total; i++) {
            const int y = cand[i].idx / w, x = cand[i].idx - y * w;
            if (ncorners < capacity) { out[3 * ncorners] = (float)x; out[3 * ncorners + 1] = (float)y; out[3 * ncorners + 2] = cand[i].v; }
            ncorners++;
            if (maxCorners > 0 && ncorners == maxCorners) break;
        }
    }
    free(eig); free(cand);
    return ncorners;
}
