/* oracle/hv_oracle_subpix.c -- TEST INFRASTRUCTURE: plain-C restatement of cv::cornerSubPix for 8-bit single-channel images
 * (OCV/imgproc/src/cornersubpix.cpp) and of the cv::getRectSubPix(8U -> 32F) it samples with (OCV/imgproc/src/samplers.cpp:
 * getRectSubPix_8u32f, its border fall-back getRectSubPix_Cn_ and adjustRect), in OpenCV's operation order and types, with IPP off.
 * Built with -ffp-contract=off (Makefile): every float / double operation is rounded where OpenCV's is.
 *
 * `faults` (tests only) injects known mistakes so that the tests can show that their comparison would catch them:
 *   ORC_SUBPIX_FLOAT_ACC  the five sums in float instead of double
 *   ORC_SUBPIX_NO_REVERT  a point that moved more than the window is kept instead of reverted to its start
 *   ORC_SUBPIX_CLAMP      the border patch as a plain clamp-to-edge bilinear sample instead of getRectSubPix_Cn_ */
#include <float.h>
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#define ORC_SUBPIX_FLOAT_ACC 1
#define ORC_SUBPIX_NO_REVERT 2
#define ORC_SUBPIX_CLAMP 4

static int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

/* cv::getRectSubPix(img, Size(pw, ph), Point2f(cx, cy), dst, CV_32F): dst is ph x pw, row-major. */
void orc_rect_subpix(const uint8_t* img, int step, int w, int h, int pw, int ph, float cx, float cy, float* dst, int faults)
{
    float x = cx - (pw - 1) * 0.5f, y = cy - (ph - 1) * 0.5f;
    const int ipx = (int)floorf(x), ipy = (int)floorf(y);
    if (0 <= ipx && ipx + pw < w && 0 <= ipy && ipy + ph < h) {
        /* getRectSubPix_8u32f: the rectangle lies inside the image */
        float a = x - ipx, b = y - ipy;
        a = a < 0.0001f ? 0.0001f : a;
        const float a12 = a * (1.f - b), a22 = a * b, b1 = 1.f - b, b2 = b;
        const double s = (1. - a) / a;
        for (int i = 0; i < ph; i++) {
            const uint8_t* src = img + (size_t)(ipy + i) * step + ipx;
            float prev = (1 - a) * (b1 * (float)src[0] + b2 * (float)src[step]);
            for (int j = 0; j < pw; j++) {
                const float t = a12 * (float)src[j + 1] + a22 * (float)src[j + 1 + step];
                dst[i * pw + j] = prev + t;
                prev = (float)(t * s);
            }
        }
        return;
    }
    /* getRectSubPix_Cn_<uchar, float, float, nop, nop>, called with the original centre (it recomputes ip and the weights) */
    const float a = x - ipx, b = y - ipy;
    const float a11 = (1.f - a) * (1.f - b), a12 = a * (1.f - b), a21 = (1.f - a) * b, a22 = a * b, b1 = 1.f - b, b2 = b;
    if (faults & ORC_SUBPIX_CLAMP) {
        for (int i = 0; i < ph; i++)
            for (int j = 0; j < pw; j++) {
                const int x0 = clampi(ipx + j, 0, w - 1), x1 = clampi(ipx + j + 1, 0, w - 1);
                const int y0 = clampi(ipy + i, 0, h - 1), y1 = clampi(ipy + i + 1, 0, h - 1);
                dst[i * pw + j] = img[(size_t)y0 * step + x0] * a11 + img[(size_t)y0 * step + x1] * a12 + img[(size_t)y1 * step + x0] * a21 +
                                  img[(size_t)y1 * step + x1] * a22;
            }
        return;
    }
    /* adjustRect: r = [rx, rw) x [ry, rh) is the part whose two taps lie inside the image; col0 / row0 the first source column / row */
    int col0 = ipx >= 0 ? ipx : 0, rx = ipx >= 0 ? 0 : (-ipx > pw ? pw : -ipx), rw;
    if (ipx < w - pw) rw = pw;
    else { rw = w - ipx - 1; if (rw < 0) { col0 += rw; rw = 0; } }
    int row = ipy >= 0 ? ipy : 0, ry = ipy >= 0 ? 0 : -ipy, rh;
    if (ipy < h - ph) rh = ph;
    else { rh = h - ipy - 1; if (rh < 0) { row += rh; rh = 0; } }
    const uint8_t* base = img - rx;         /* column k of the rectangle is source column col0 - rx + k */
    for (int i = 0; i < ph; i++) {
        const int row2 = (i < ry || i >= rh) ? row : row + 1;
        const uint8_t* s1 = base + (size_t)row * step + col0;
        const uint8_t* s2 = base + (size_t)row2 * step + col0;
        float* d = dst + i * pw;
        float s0 = s1[rx] * b1 + s2[rx] * b2;
        for (int j = 0; j < rx; j++) d[j] = s0;
        s0 = s1[rw] * b1 + s2[rw] * b2;
        for (int j = rw; j < pw; j++) d[j] = s0;
        for (int j = rx; j < rw; j++) d[j] = s1[j] * a11 + s1[j + 1] * a12 + s2[j] * a21 + s2[j + 1] * a22;
        if (i < rh) row = row2;
    }
}

/* The mask of cornerSubPix: exp(-y^2) exp(-x^2) over the window in float (std::exp(float) = expf), the zero zone cleared when it
 * applies. mask: (2 hh + 1) x (2 hw + 1). */
void orc_subpix_mask(int hw, int hh, int zw, int zh, float* mask)
{
    const int ww = 2 * hw + 1, wh = 2 * hh + 1;
    for (int i = 0; i < wh; i++) {
        const float y = (float)(i - hh) / hh, vy = expf(-y * y);
        for (int j = 0; j < ww; j++) {
            const float x = (float)(j - hw) / hw;
            mask[i * ww + j] = (float)(vy * expf(-x * x));
        }
    }
    if (zw >= 0 && zh >= 0 && zw * 2 + 1 < ww && zh * 2 + 1 < wh)
        for (int i = hh - zh; i <= hh + zh; i++)
            for (int j = hw - zw; j <= hw + zw; j++) mask[i * ww + j] = 0;
}

/* cv::cornerSubPix(img, xy, Size(hw, hh), Size(zw, zh), TermCriteria(criteria_type, max_count, epsilon)); xy in / out (n x 2).
 * Returns -1 where OpenCV asserts (window, image size, a corner outside the image), before any point is changed; 0 otherwise. */
int orc_subpix_refine(const uint8_t* img, int step, int w, int h, float* xy, int n, int hw, int hh, int zw, int zh, int criteria_type,
                      int max_count, double epsilon, int faults)
{
    if (n <= 0) return 0;
    if (hw <= 0 || hh <= 0 || hw > 15 || hh > 15 || w < 2 * hw + 5 || h < 2 * hh + 5) return -1;
    for (int p = 0; p < n; p++)
        if (!(0 <= xy[2 * p] && xy[2 * p] < w && 0 <= xy[2 * p + 1] && xy[2 * p + 1] < h)) return -1;
    const int ww = 2 * hw + 1, wh = 2 * hh + 1, pw = ww + 2, ph = wh + 2;
    int max_iters = 100;
    if (criteria_type & 1) { max_iters = max_count < 1 ? 1 : max_count; max_iters = max_iters > 100 ? 100 : max_iters; }
    double eps = 0;
    if (criteria_type & 2) eps = epsilon < 0. ? 0. : epsilon;
    eps *= eps;
    float mask[31 * 31], patch[33 * 33];
    orc_subpix_mask(hw, hh, zw, zh, mask);
    for (int p = 0; p < n; p++) {
        const float tx = xy[2 * p], ty = xy[2 * p + 1];
        float cx = tx, cy = ty;
        int iter = 0;
        double err = 0;
        do {
            orc_rect_subpix(img, step, w, h, pw, ph, cx, cy, patch, faults);
            double a = 0, b = 0, c = 0, bb1 = 0, bb2 = 0;
            float fa = 0, fb = 0, fc = 0, fbb1 = 0, fbb2 = 0;
            for (int i = 0, k = 0; i < wh; i++) {
                const float* sub = patch + (i + 1) * pw + 1;
                const double py = i - hh;
                for (int j = 0; j < ww; j++, k++) {
                    const double m = mask[k];
                    const double tgx = sub[j + 1] - sub[j - 1];
                    const double tgy = sub[j + pw] - sub[j - pw];
                    const double gxx = tgx * tgx * m, gxy = tgx * tgy * m, gyy = tgy * tgy * m;
                    const double px = j - hw;
                    if (faults & ORC_SUBPIX_FLOAT_ACC) {
                        fa += (float)gxx; fb += (float)gxy; fc += (float)gyy;
                        fbb1 += (float)(gxx * px + gxy * py); fbb2 += (float)(gxy * px + gyy * py);
                    } else {
                        a += gxx; b += gxy; c += gyy;
                        bb1 += gxx * px + gxy * py;
                        bb2 += gxy * px + gyy * py;
                    }
                }
            }
            if (faults & ORC_SUBPIX_FLOAT_ACC) { a = fa; b = fb; c = fc; bb1 = fbb1; bb2 = fbb2; }
            const double det = a * c - b * b;
            if (fabs(det) <= DBL_EPSILON * DBL_EPSILON) break;
            const double scale = 1.0 / det;
            const float nx = (float)(cx + c * scale * bb1 - b * scale * bb2);
            const float ny = (float)(cy - b * scale * bb1 + a * scale * bb2);
            err = (nx - cx) * (nx - cx) + (ny - cy) * (ny - cy);       /* float, as Point2f arithmetic */
            if (nx < 0 || nx >= w || ny < 0 || ny >= h) break;           /* a step out of the image is not taken */
            cx = nx; cy = ny;
        } while (++iter < max_iters && err > eps);
        if (!(faults & ORC_SUBPIX_NO_REVERT) && (fabsf(cx - tx) > hw || fabsf(cy - ty) > hh)) { cx = tx; cy = ty; }
        xy[2 * p] = cx; xy[2 * p + 1] = cy;
    }
    return 0;
}
