/* oracle/hv_oracle_pnp.c -- TEST INFRASTRUCTURE: plain-C restatement of
 *   cv::solvePnPRansac(xyz[used], xy[used], K, noArray(), rvec, tvec, false, iterations, reprojError, confidence, inliers, SOLVEPNP_P3P)
 * (OCV/calib3d/src/solvepnp.cpp, ptsetreg.cpp, p3p.cpp, epnp.cpp) as the device computes it (hybvio_b200/csrc/pnp.cu), operation for
 * operation:
 *   1. the used points (status != 0) in index order, m of them; m < 4: no result;
 *   2. m == 4: the P3P model of the four points (below), every point an inlier, no refinement (OpenCV's model_points == npoints path);
 *   3. m > 4: RANSAC with modelPoints = 4. cv::RNG(~0) draws each subset (rng.uniform(0, m), a repeated index drawn again); its model is
 *      the P3P pose of the subset's first three points that reprojects the fourth closest, stored as (rvec, tvec) and scored through
 *      R = Rodrigues(rvec): a point is an inlier when the float32 squared distance between its image point and the float32 projection
 *      (double R X + t, x * (1 / z), x * fx + cx, rounded to float) is <= (float)(thr * thr), thr the float reprojection error;
 *      a count above max(best, 3) wins and the bound shrinks through RANSACUpdateNumIters(confidence, (m - count) / m, 4, niters);
 *   4. the winner's inliers, in index order, go through one EPnP in double (epnp::compute_pose), whose pose is returned; the returned
 *      inliers are the RANSAC model's.
 * What is this library's own (OpenCV's SVDs, matrix inverse, acos / cos / sin and P3P solver are not restated):
 *   - P3P: Grunert's distances along the three unit rays, eliminated to a quartic in v = s3 / s1 (u = s2 / s1 is the quotient of two
 *     polynomials in v) with double-double coefficients; the real roots v > 0 by recursion on the derivatives (the quartic's own sign
 *     in double-double), then PNP_POLISH Newton steps on the two conics, each bracketed by PNP_BISECT bisection steps on the
 *     ordered bit patterns of doubles (to one ulp: a bounded amount of work whatever the data); solutions with u or v not positive
 *     dropped; the pose from the two triangles' orthonormal frames;
 *   - Rodrigues with an atan2 and a sin / cos of + - * / and sqrt only (a Taylor series of theta / 8 and three angle doublings), so that
 *     the device and this oracle round alike;
 *   - SVDs: one-sided (Hestenes) Jacobi with a fixed number of cyclic sweeps (PNP_SWEEPS3 for the 3 x 3 and 6 x k problems,
 *     PNP_SWEEPS12 for EPnP's 12 x 12 M^T M, whose rotations sum over its rows by a 32-lane butterfly as the device's warp does);
 *     least squares and the pseudo-inverse drop singular values at or below 2 DBL_EPSILON times their sum, as OpenCV's back substitution;
 *   - EPnP's sums over the points in the CTA's fixed order (pnp_reduce).
 * EPnP's PCA is OpenCV's own Jacobi SVD, restated for its sign convention (pnp_ocv_svd3), which decides the pose on noisy points.
 * Built with -ffp-contract=off, so no multiply-add is contracted; the kernel is built with --fmad=false. Only log and pow (the
 * iteration bound) are the C library's, as in the essential oracle.
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define PNP_THREADS 512
#define PNP_BISECT 64
#define PNP_SWEEPS3 8
#define PNP_SWEEPS12 12

/* ------------------------------------------------------------------------------------------------ trigonometry of + - * / sqrt */
/* sin and cos of th in [0, 4]: Taylor series of th / 8 (|x| <= 0.5, terms to x^19 / x^18), then three doublings */
void orc_pnp_sincos(double th, double* ps, double* pc)
{
    const double x = th * 0.125, x2 = x * x;
    double s = -1.0 / 121645100408832000.0;
    s = 1.0 / 355687428096000.0 + x2 * s;
    s = -1.0 / 1307674368000.0 + x2 * s;
    s = 1.0 / 6227020800.0 + x2 * s;
    s = -1.0 / 39916800.0 + x2 * s;
    s = 1.0 / 362880.0 + x2 * s;
    s = -1.0 / 5040.0 + x2 * s;
    s = 1.0 / 120.0 + x2 * s;
    s = -1.0 / 6.0 + x2 * s;
    s = x + x * (x2 * s);
    double c = -1.0 / 6402373705728000.0;
    c = 1.0 / 20922789888000.0 + x2 * c;
    c = -1.0 / 87178291200.0 + x2 * c;
    c = 1.0 / 479001600.0 + x2 * c;
    c = -1.0 / 3628800.0 + x2 * c;
    c = 1.0 / 40320.0 + x2 * c;
    c = -1.0 / 720.0 + x2 * c;
    c = 1.0 / 24.0 + x2 * c;
    c = -0.5 + x2 * c;
    c = 1.0 + x2 * c;
    for (int k = 0; k < 3; k++) {
        const double s2 = 2.0 * (s * c), c2 = (c - s) * (c + s);
        s = s2; c = c2;
    }
    *ps = s; *pc = c;
}

/* atan z for z in [0, 1]: two half-angle reductions (|w| <= tan(pi / 16)), then the series to w^25 */
static double pnp_atan01(double z)
{
    double w = z / (1.0 + sqrt(1.0 + z * z));
    w = w / (1.0 + sqrt(1.0 + w * w));
    const double w2 = w * w;
    double p = 1.0 / 25.0;
    p = -1.0 / 23.0 + w2 * p;
    p = 1.0 / 21.0 + w2 * p;
    p = -1.0 / 19.0 + w2 * p;
    p = 1.0 / 17.0 + w2 * p;
    p = -1.0 / 15.0 + w2 * p;
    p = 1.0 / 13.0 + w2 * p;
    p = -1.0 / 11.0 + w2 * p;
    p = 1.0 / 9.0 + w2 * p;
    p = -1.0 / 7.0 + w2 * p;
    p = 1.0 / 5.0 + w2 * p;
    p = -1.0 / 3.0 + w2 * p;
    return 4.0 * (w + w * (w2 * p));
}

/* atan2(y, x) for y >= 0 */
double orc_pnp_atan2(double y, double x)
{
    const double ax = fabs(x);
    double a;
    if (y == 0.0 && ax == 0.0) a = 0.0;
    else if (y <= ax) a = pnp_atan01(y / ax);
    else a = 1.5707963267948966 - pnp_atan01(ax / y);
    return x < 0.0 ? 3.141592653589793 - a : a;
}

/* cv::Rodrigues, rotation vector -> R (row-major) */
void orc_pnp_rodrigues_v2r(const double* r, double* R)
{
    const double th = sqrt((r[0] * r[0] + r[1] * r[1]) + r[2] * r[2]);
    if (th < DBL_EPSILON) {
        for (int k = 0; k < 9; k++) R[k] = k % 4 == 0 ? 1.0 : 0.0;
        return;
    }
    double s, c;
    orc_pnp_sincos(th, &s, &c);
    const double c1 = 1.0 - c, it = 1.0 / th;
    const double x = r[0] * it, y = r[1] * it, z = r[2] * it;
    const double rr[9] = {x * x, x * y, x * z, x * y, y * y, y * z, x * z, y * z, z * z};
    const double K[9] = {0.0, -z, y, z, 0.0, -x, -y, x, 0.0};
    for (int k = 0; k < 9; k++) R[k] = (c * (k % 4 == 0 ? 1.0 : 0.0) + c1 * rr[k]) + s * K[k];
}

/* cv::Rodrigues, R (row-major, orthonormal to rounding; OpenCV's U V^T projection is not restated) -> rotation vector, with
 * theta = atan2(s, c) for OpenCV's acos(c) */
void orc_pnp_rodrigues_r2v(const double* R, double* r)
{
    double x = R[7] - R[5], y = R[2] - R[6], z = R[3] - R[1];
    const double s = sqrt(((x * x + y * y) + z * z) * 0.25);
    double c = ((R[0] + R[4]) + R[8] - 1.0) * 0.5;
    c = c > 1.0 ? 1.0 : c < -1.0 ? -1.0 : c;
    double th = orc_pnp_atan2(s, c);
    if (s < 1e-5) {
        if (c > 0.0) { x = 0.0; y = 0.0; z = 0.0; }
        else {
            double t = (R[0] + 1.0) * 0.5;
            x = sqrt(t > 0.0 ? t : 0.0);
            t = (R[4] + 1.0) * 0.5;
            y = sqrt(t > 0.0 ? t : 0.0) * (R[1] < 0.0 ? -1.0 : 1.0);
            t = (R[8] + 1.0) * 0.5;
            z = sqrt(t > 0.0 ? t : 0.0) * (R[2] < 0.0 ? -1.0 : 1.0);
            if (fabs(x) < fabs(y) && fabs(x) < fabs(z) && (R[5] > 0.0) != (y * z > 0.0)) z = -z;
            th = th / sqrt((x * x + y * y) + z * z);
            x = x * th; y = y * th; z = z * th;
        }
    } else {
        const double vth = (1.0 / (2.0 * s)) * th;
        x = x * vth; y = y * vth; z = z * vth;
    }
    r[0] = x; r[1] = y; r[2] = z;
}

/* ------------------------------------------------------------------------------------------------ P3P */
static int pnp_sgn(double v) { return (v > 0.0) - (v < 0.0); }

static long long pnp_okey(double x)
{
    long long b;
    memcpy(&b, &x, 8);
    return b >= 0 ? b : -(b & 0x7fffffffffffffffll);
}

static double pnp_ofrom(long long k)
{
    const unsigned long long u = k >= 0 ? (unsigned long long)k : ((unsigned long long)(-k) | 0x8000000000000000ull);
    double x;
    memcpy(&x, &u, 8);
    return x;
}

static double pnp_horner(const double* c, int d, double x)
{
    double s = c[d];
    for (int i = d - 1; i >= 0; i--) s = s * x + c[i];
    return s;
}

/* double-double arithmetic (hi + lo), as in the essential solver: Grunert's quartic loses digits to cancellation in double, enough to
 * turn a close pair of real roots into a complex pair. Products go through an explicit fma, so that the device and this oracle agree. */
static void pnp_dd_fast(double s, double e, double* h, double* l)
{
    const double x = s + e;
    *h = x; *l = e - (x - s);
}

static void pnp_dd_add(const double* a, const double* b, double* r)
{
    const double s = a[0] + b[0], bb = s - a[0];
    const double e = (a[0] - (s - bb)) + (b[0] - bb);
    const double t = a[1] + b[1], tb = t - a[1];
    const double te = (a[1] - (t - tb)) + (b[1] - tb);
    double h, l;
    pnp_dd_fast(s, e + t, &h, &l);
    pnp_dd_fast(h, l + te, r, r + 1);
}

static void pnp_dd_sub(const double* a, const double* b, double* r)
{
    const double nb[2] = {-b[0], -b[1]};
    pnp_dd_add(a, nb, r);
}

static void pnp_dd_mul(const double* a, const double* b, double* r)
{
    const double p = a[0] * b[0];
    pnp_dd_fast(p, fma(a[0], b[0], -p) + (a[0] * b[1] + a[1] * b[0]), r, r + 1);
}

static void pnp_dd_mul_d(const double* a, double x, double* r)
{
    const double p = a[0] * x;
    pnp_dd_fast(p, fma(a[0], x, -p) + a[1] * x, r, r + 1);
}

static void pnp_dd_div(const double* a, const double* b, double* r)
{
    const double q1 = a[0] / b[0], q[2] = {q1, 0.0};
    double m[2], e[2];
    pnp_dd_mul(b, q, m);
    pnp_dd_sub(a, m, e);
    pnp_dd_fast(q1, e[0] / b[0], r, r + 1);
}

/* the sign of the quartic (double-double coefficients P, degree d) at x, by Horner's rule in double-double */
static int pnp_sgn_dd(const double* P, int d, double x)
{
    double s[2] = {P[2 * d], P[2 * d + 1]}, t[2];
    for (int i = d - 1; i >= 0; i--) {
        pnp_dd_mul_d(s, x, t);
        pnp_dd_add(t, P + 2 * i, s);
    }
    return (s[0] > 0.0) - (s[0] < 0.0);
}

/* the root of the degree-d polynomial c in (lo, hi] where it is monotonic: 1 and *root, or 0 */
static int pnp_interval_root(const double* c, int d, double lo, double hi, double* root)
{
    const int slo = pnp_sgn(pnp_horner(c, d, lo)), shi = pnp_sgn(pnp_horner(c, d, hi));
    if (slo != 0 && shi == 0) { *root = hi; return 1; }
    if (slo == 0 || shi == 0 || slo == shi) return 0;
    long long kl = pnp_okey(lo), kh = pnp_okey(hi);
    for (int it = 0; it < PNP_BISECT; it++) {
        const unsigned long long span = (unsigned long long)kh - (unsigned long long)kl;
        if (span <= 1) continue;
        const long long km = kl + (long long)(span >> 1);
        if (pnp_sgn(pnp_horner(c, d, pnp_ofrom(km))) == slo) kl = km; else kh = km;
    }
    *root = pnp_ofrom(kh);
    return 1;
}

/* pnp_interval_root with the sign of the quartic itself (double-double coefficients P) */
static int pnp_interval_root_dd(const double* P, int d, double lo, double hi, double* root)
{
    const int slo = pnp_sgn_dd(P, d, lo), shi = pnp_sgn_dd(P, d, hi);
    if (slo != 0 && shi == 0) { *root = hi; return 1; }
    if (slo == 0 || shi == 0 || slo == shi) return 0;
    long long kl = pnp_okey(lo), kh = pnp_okey(hi);
    for (int it = 0; it < PNP_BISECT; it++) {
        const unsigned long long span = (unsigned long long)kh - (unsigned long long)kl;
        if (span <= 1) continue;
        const long long km = kl + (long long)(span >> 1);
        if (pnp_sgn_dd(P, d, pnp_ofrom(km)) == slo) kl = km; else kh = km;
    }
    *root = pnp_ofrom(kh);
    return 1;
}

/* the real roots in (0, R] (ascending) of the quartic p by recursion on its derivatives (lane 0 of the device's warp) */
int orc_pnp_quartic_roots(const double* P, double* roots)
{
    double p[5];
    for (int k = 0; k < 5; k++) p[k] = P[2 * k];
    int D = 4;
    while (D > 0 && p[D] == 0.0) D--;
    if (D < 1) return 0;
    double mx = 0.0;
    for (int i = 0; i < D; i++) {
        const double a = fabs(p[i]) / fabs(p[D]);
        if (a > mx) mx = a;
    }
    double R = 1.0 + mx;
    if (!(R <= DBL_MAX)) R = DBL_MAX;
    double der[5][5], crit[4];
    for (int i = 0; i <= D; i++) der[D][i] = p[i];
    for (int d = D; d > 1; d--)
        for (int i = 0; i < d; i++) der[d - 1][i] = (double)(i + 1) * der[d][i + 1];
    int ncrit = 0;
    for (int d = 1; d <= D; d++) {
        double nc[4];
        int k = 0;
        for (int l = 0; l <= ncrit; l++) {
            const double lo = l == 0 ? 0.0 : crit[l - 1], hi = l == ncrit ? R : crit[l];
            double root;
            if (d == D ? pnp_interval_root_dd(P, D, lo, hi, &root) : pnp_interval_root(der[d], d, lo, hi, &root)) nc[k++] = root;
        }
        for (int i = 0; i < k; i++) crit[i] = nc[i];
        ncrit = k;
    }
    for (int i = 0; i < ncrit; i++) roots[i] = crit[i];
    return ncrit;
}

static void pnp_cross(const double* a, const double* b, double* c)
{
    c[0] = a[1] * b[2] - a[2] * b[1];
    c[1] = a[2] * b[0] - a[0] * b[2];
    c[2] = a[0] * b[1] - a[1] * b[0];
}

static double pnp_dot(const double* a, const double* b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }

/* the orthonormal frame (columns e1, e2, e3 of F, row-major) of the triangle a, b, c: e1 along b - a, e3 along (b - a) x (c - a) */
static int pnp_frame(const double* a, const double* b, const double* c, double* F)
{
    double u[3] = {b[0] - a[0], b[1] - a[1], b[2] - a[2]}, w[3] = {c[0] - a[0], c[1] - a[1], c[2] - a[2]}, n[3], e2[3];
    pnp_cross(u, w, n);
    const double lu = sqrt(pnp_dot(u, u)), ln = sqrt(pnp_dot(n, n));
    if (!(lu > 0.0) || !(ln > 0.0)) return 0;
    for (int k = 0; k < 3; k++) { u[k] = u[k] / lu; n[k] = n[k] / ln; }
    pnp_cross(n, u, e2);
    for (int k = 0; k < 3; k++) { F[3 * k] = u[k]; F[3 * k + 1] = e2[k]; F[3 * k + 2] = n[k]; }
    return 1;
}

/* the unit ray of pixel (u, v) */
static void pnp_ray(float u, float v, double fx, double fy, double cx, double cy, double* f)
{
    const double x = ((double)u - cx) / fx, y = ((double)v - cy) / fy;
    const double n = sqrt((x * x + y * y) + 1.0);
    f[0] = x / n; f[1] = y / n; f[2] = 1.0 / n;
}

/* the coefficients (ascending) of Grunert's quartic in v = s3 / s1 and of u = N(v) / (d0 + d1 v): K1 = d12^2 / d13^2,
 * K2 = d12^2 / d23^2; the two conics (1 + u^2 - 2 u c12) = K1 (1 + v^2 - 2 v c13) = K2 (u^2 + v^2 - 2 u v c23) */
int orc_pnp_grunert(const double* X, const double* f, double* P, double* Nc, double* Dc)
{
    const double c12 = pnp_dot(f, f + 3), c13 = pnp_dot(f, f + 6), c23 = pnp_dot(f + 3, f + 6);
    double e[3];
    for (int k = 0; k < 3; k++) e[k] = X[k] - X[3 + k];
    const double d12 = pnp_dot(e, e);
    for (int k = 0; k < 3; k++) e[k] = X[k] - X[6 + k];
    const double d13 = pnp_dot(e, e);
    for (int k = 0; k < 3; k++) e[k] = X[3 + k] - X[6 + k];
    const double d23 = pnp_dot(e, e);
    if (!(d13 > 0.0) || !(d23 > 0.0)) return 0;
    double K1[2], K2[2], L[2], LK1[2], t[2];
    const double one[2] = {1.0, 0.0}, D12[2] = {d12, 0.0}, D13[2] = {d13, 0.0}, D23[2] = {d23, 0.0};
    pnp_dd_div(D12, D13, K1);
    pnp_dd_div(D12, D23, K2);
    pnp_dd_sub(one, K2, L);
    pnp_dd_mul(L, K1, LK1);
    double N[3][2], D[2][2], q[3][2];
    pnp_dd_sub(LK1, K2, N[2]);
    pnp_dd_mul_d(LK1, -2.0 * c13, N[1]);
    pnp_dd_add(LK1, K2, N[0]);
    pnp_dd_mul_d(K2, 2.0 * c12, D[0]);
    pnp_dd_mul_d(K2, -2.0 * c23, D[1]);
    q[0][0] = K1[0]; q[0][1] = K1[1]; q[2][0] = K1[0]; q[2][1] = K1[1];
    pnp_dd_mul_d(K1, -2.0 * c13, q[1]);
    double N2[5][2], ND[4][2], D2[3][2], qD2[5][2];
    for (int k = 0; k < 5; k++) { N2[k][0] = N2[k][1] = qD2[k][0] = qD2[k][1] = 0.0; }
    for (int k = 0; k < 4; k++) ND[k][0] = ND[k][1] = 0.0;
    for (int k = 0; k < 3; k++) D2[k][0] = D2[k][1] = 0.0;
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) { pnp_dd_mul(N[i], N[j], t); pnp_dd_add(N2[i + j], t, N2[i + j]); }
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 2; j++) { pnp_dd_mul(N[i], D[j], t); pnp_dd_add(ND[i + j], t, ND[i + j]); }
    for (int i = 0; i < 2; i++)
        for (int j = 0; j < 2; j++) { pnp_dd_mul(D[i], D[j], t); pnp_dd_add(D2[i + j], t, D2[i + j]); }
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) { pnp_dd_mul(q[i], D2[j], t); pnp_dd_add(qD2[i + j], t, qD2[i + j]); }
    for (int k = 0; k < 5; k++) {
        double v[2];
        pnp_dd_sub(N2[k], qD2[k], v);
        if (k < 4) { pnp_dd_mul_d(ND[k], 2.0 * c12, t); pnp_dd_sub(v, t, v); }
        if (k < 3) pnp_dd_add(v, D2[k], v);
        P[2 * k] = v[0]; P[2 * k + 1] = v[1];
    }
    for (int k = 0; k < 3; k++) Nc[k] = N[k][0];
    for (int k = 0; k < 2; k++) Dc[k] = D[k][0];
    return 1;
}

/* PNP_POLISH Newton steps on Grunert's two conics themselves from (u, v): the quartic's expanded coefficients lose digits to
 * cancellation, the conics are as well conditioned as the problem. A step is skipped where the Jacobian is singular. */
#define PNP_POLISH 3
static void pnp_polish(double c12, double c13, double c23, double d12, double d13, double d23, double* pu, double* pv)
{
    double u = *pu, v = *pv;
    for (int it = 0; it < PNP_POLISH; it++) {
        const double g = (1.0 + u * u) - 2.0 * (u * c12);
        const double F1 = d13 * g - d12 * ((1.0 + v * v) - 2.0 * (v * c13));
        const double F2 = d23 * g - d12 * ((u * u + v * v) - 2.0 * (u * (v * c23)));
        const double a = d13 * (2.0 * u - 2.0 * c12), b = -(d12 * (2.0 * v - 2.0 * c13));
        const double c = d23 * (2.0 * u - 2.0 * c12) - d12 * (2.0 * u - 2.0 * (v * c23)), d = -(d12 * (2.0 * v - 2.0 * (u * c23)));
        const double det = a * d - b * c;
        if (!(det != 0.0) || det != det) break;
        const double du = (F1 * d - b * F2) / det, dv = (a * F2 - c * F1) / det;
        if (du != du || dv != dv) break;
        u = u - du; v = v - dv;
    }
    *pu = u; *pv = v;
}

/* every P3P pose (R row-major, t) of the world points X (3 x 3) seen at pixels xy (3 x 2), in ascending order of v; returns their count */
int orc_pnp_p3p(const double* X, const float* xy, double fx, double fy, double cx, double cy, double* Rs, double* ts)
{
    double f[9], Fw[9], P[10], Nc[3], Dc[2], roots[4];
    for (int i = 0; i < 3; i++) pnp_ray(xy[2 * i], xy[2 * i + 1], fx, fy, cx, cy, f + 3 * i);
    if (!pnp_frame(X, X + 3, X + 6, Fw)) return 0;
    if (!orc_pnp_grunert(X, f, P, Nc, Dc)) return 0;
    double e[3];
    for (int k = 0; k < 3; k++) e[k] = X[k] - X[6 + k];
    const double d13 = pnp_dot(e, e), c13 = pnp_dot(f, f + 6), c12 = pnp_dot(f, f + 3), c23 = pnp_dot(f + 3, f + 6);
    for (int k = 0; k < 3; k++) e[k] = X[k] - X[3 + k];
    const double d12 = pnp_dot(e, e);
    for (int k = 0; k < 3; k++) e[k] = X[3 + k] - X[6 + k];
    const double d23 = pnp_dot(e, e);
    const int nr = orc_pnp_quartic_roots(P, roots);
    int ns = 0;
    for (int r = 0; r < nr; r++) {
        double v = roots[r];
        const double num = (Nc[2] * v + Nc[1]) * v + Nc[0], den = Dc[0] + Dc[1] * v;
        if (!(den != 0.0)) continue;
        double u = num / den;
        if (!(u > 0.0)) continue;
        pnp_polish(c12, c13, c23, d12, d13, d23, &u, &v);
        if (!(u > 0.0) || !(v > 0.0)) continue;
        const double s1 = sqrt(d13 / ((v - 2.0 * c13) * v + 1.0)), s2 = u * s1, s3 = v * s1;
        double Y[9], Fc[9];
        for (int k = 0; k < 3; k++) { Y[k] = s1 * f[k]; Y[3 + k] = s2 * f[3 + k]; Y[6 + k] = s3 * f[6 + k]; }
        if (!pnp_frame(Y, Y + 3, Y + 6, Fc)) continue;
        double* R = Rs + 9 * ns;
        double* t = ts + 3 * ns;
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) R[3 * i + j] = (Fc[3 * i] * Fw[3 * j] + Fc[3 * i + 1] * Fw[3 * j + 1]) + Fc[3 * i + 2] * Fw[3 * j + 2];
        for (int i = 0; i < 3; i++) t[i] = Y[i] - pnp_dot(R + 3 * i, X);
        ns++;
    }
    return ns;
}

/* the RANSAC kernel on four points: the P3P pose of the first three that reprojects the fourth closest (the first on a tie), as
 * (rvec, tvec); 0 when P3P has no solution */
int orc_pnp_model4(const double* X4, const float* xy4, double fx, double fy, double cx, double cy, double* model)
{
    double Rs[36], ts[12];
    const int ns = orc_pnp_p3p(X4, xy4, fx, fy, cx, cy, Rs, ts);
    if (ns == 0) return 0;
    int best = 0;
    double be = 0.0;
    for (int k = 0; k < ns; k++) {
        const double* R = Rs + 9 * k;
        const double* t = ts + 3 * k;
        const double xc = pnp_dot(R, X4 + 9) + t[0], yc = pnp_dot(R + 3, X4 + 9) + t[1], zc = pnp_dot(R + 6, X4 + 9) + t[2];
        const double du = (fx * (xc / zc) + cx) - (double)xy4[6], dv = (fy * (yc / zc) + cy) - (double)xy4[7];
        const double err = du * du + dv * dv;
        if (k == 0 || err < be) { best = k; be = err; }
    }
    orc_pnp_rodrigues_r2v(Rs + 9 * best, model);
    for (int i = 0; i < 3; i++) model[3 + i] = ts[3 * best + i];
    return 1;
}

/* projectPoints' float32 image point under (R, t) and the float32 squared distance to (u, v) */
static float pnp_err(const double* R, const double* t, const float* X, const float* x, double fx, double fy, double cx, double cy)
{
    const double a = X[0], b = X[1], c = X[2];
    double px = ((R[0] * a + R[1] * b) + R[2] * c) + t[0];
    double py = ((R[3] * a + R[4] * b) + R[5] * c) + t[1];
    double pz = ((R[6] * a + R[7] * b) + R[8] * c) + t[2];
    pz = pz != 0.0 ? 1.0 / pz : 1.0;
    px = px * pz; py = py * pz;
    const float u = (float)(px * fx + cx), v = (float)(py * fy + cy);
    const float du = x[0] - u, dv = x[1] - v;
    return du * du + dv * dv;
}

static unsigned rng_next(uint64_t* s)
{
    *s = (uint64_t)(unsigned)*s * 4164903690u + (unsigned)(*s >> 32);
    return (unsigned)*s;
}

/* cv::RANSACUpdateNumIters(p, ep, 4, niters) for p in (0, 1), ep in [0, 1] */
int orc_pnp_update_niters(double p, double ep, int niters)
{
    double num = 1.0 - p;
    if (num < DBL_MIN) num = DBL_MIN;
    double denom = 1.0 - pow(1.0 - ep, 4.0);
    if (denom < DBL_MIN) return 0;
    num = log(num);
    denom = log(denom);
    return denom >= 0.0 || -num >= niters * (-denom) ? niters : (int)nearbyint(num / denom);
}

/* the draws of the first `iters` iterations: 4 distinct indices of [0, m) each */
void orc_pnp_subsets(int m, int iters, int* sub)
{
    uint64_t s = ~0ull;
    for (int it = 0; it < iters; it++) {
        int* d = sub + 4 * it;
        for (int i = 0; i < 4; i++) {
            int v;
            for (;;) {
                v = (int)(rng_next(&s) % (unsigned)m);
                int dup = 0;
                for (int k = 0; k < i; k++) dup |= d[k] == v;
                if (!dup) break;
            }
            d[i] = v;
        }
    }
}

/* ------------------------------------------------------------------------------------------------ EPnP */
static void jacobi_rotate(double* A, double* V, int rows, int ncols, int p, int q)
{
    double a = 0.0, b = 0.0, g = 0.0;
    for (int r = 0; r < rows; r++) {
        const double x = A[r * ncols + p], y = A[r * ncols + q];
        a = a + x * x;
        b = b + y * y;
        g = g + x * y;
    }
    if (g == 0.0) return;
    const double zeta = (b - a) / (2.0 * g);
    double t = 1.0 / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
    if (zeta < 0.0) t = -t;
    const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
    for (int r = 0; r < rows; r++) {
        const double x = A[r * ncols + p], y = A[r * ncols + q];
        A[r * ncols + p] = c * x - s * y;
        A[r * ncols + q] = s * x + c * y;
    }
    for (int r = 0; r < ncols; r++) {
        const double x = V[r * ncols + p], y = V[r * ncols + q];
        V[r * ncols + p] = c * x - s * y;
        V[r * ncols + q] = s * x + c * y;
    }
}

/* one-sided Jacobi of A (rows x n, n <= 5): A <- A V, V (n x n) orthogonal; w[j] = |column j of A| */
static void jacobi(double* A, double* V, double* w, int rows, int n)
{
    for (int i = 0; i < n * n; i++) V[i] = i % (n + 1) == 0 ? 1.0 : 0.0;
    for (int s = 0; s < PNP_SWEEPS3; s++)
        for (int p = 0; p < n - 1; p++)
            for (int q = p + 1; q < n; q++) jacobi_rotate(A, V, rows, n, p, q);
    for (int j = 0; j < n; j++) {
        double s = 0.0;
        for (int r = 0; r < rows; r++) s = s + A[r * n + j] * A[r * n + j];
        w[j] = sqrt(s);
    }
}

static double svd_threshold(const double* w, int n)
{
    double s = 0.0;
    for (int j = 0; j < n; j++) s = s + w[j];
    return s * (2.0 * DBL_EPSILON);
}

/* OpenCV's JacobiSVDImpl_ (OCV/core/src/lapack.cpp) on the symmetric 3 x 3 A, restated for its sign convention, which decides EPnP's
 * control points and so its pose on noisy points: one-sided rotations of the rows of A^T until none changes (at most 30 sweeps), the
 * rotation of OpenCV's branch on beta = |row i|^2 - |row j|^2, hypot as sqrt(p^2 + beta^2); w descending (the first of equal norms kept
 * first), u's rows the unit left singular vectors (zero where w <= DBL_MIN) */
static void pnp_ocv_svd3(const double* A, double* w, double* u)
{
    double At[9], W[3];
    for (int i = 0; i < 3; i++)
        for (int k = 0; k < 3; k++) At[3 * i + k] = A[3 * k + i];
    for (int i = 0; i < 3; i++) {
        double sd = 0.0;
        for (int k = 0; k < 3; k++) sd = sd + At[3 * i + k] * At[3 * i + k];
        W[i] = sd;
    }
    for (int it = 0; it < 30; it++) {
        int changed = 0;
        for (int i = 0; i < 2; i++)
            for (int j = i + 1; j < 3; j++) {
                double* Ai = At + 3 * i;
                double* Aj = At + 3 * j;
                double a = W[i], b = W[j], p = 0.0;
                for (int k = 0; k < 3; k++) p = p + Ai[k] * Aj[k];
                if (fabs(p) <= (10.0 * DBL_EPSILON) * sqrt(a * b)) continue;
                p = p * 2.0;
                const double beta = a - b, gamma = sqrt(p * p + beta * beta);
                double c, s;
                if (beta < 0.0) {
                    const double delta = (gamma - beta) * 0.5;
                    s = sqrt(delta / gamma);
                    c = p / (gamma * s * 2.0);
                } else {
                    c = sqrt((gamma + beta) / (gamma * 2.0));
                    s = p / (gamma * c * 2.0);
                }
                a = 0.0; b = 0.0;
                for (int k = 0; k < 3; k++) {
                    const double t0 = c * Ai[k] + s * Aj[k], t1 = -s * Ai[k] + c * Aj[k];
                    Ai[k] = t0; Aj[k] = t1;
                    a = a + t0 * t0; b = b + t1 * t1;
                }
                W[i] = a; W[j] = b;
                changed = 1;
            }
        if (!changed) break;
    }
    for (int i = 0; i < 3; i++) {
        double sd = 0.0;
        for (int k = 0; k < 3; k++) sd = sd + At[3 * i + k] * At[3 * i + k];
        W[i] = sqrt(sd);
    }
    for (int i = 0; i < 2; i++) {
        int j = i;
        for (int k = i + 1; k < 3; k++)
            if (W[j] < W[k]) j = k;
        if (i != j) {
            double t = W[i]; W[i] = W[j]; W[j] = t;
            for (int k = 0; k < 3; k++) { t = At[3 * i + k]; At[3 * i + k] = At[3 * j + k]; At[3 * j + k] = t; }
        }
    }
    for (int i = 0; i < 3; i++) {
        w[i] = W[i];
        const double sc = W[i] > DBL_MIN ? 1.0 / W[i] : 0.0;
        for (int k = 0; k < 3; k++) u[3 * i + k] = At[3 * i + k] * sc;
    }
}

/* cvSolve(A, b, x, CV_SVD): the least-squares solution of the 6 x n system (n <= 5), A overwritten */
static void lsq(double* A, const double* b, double* x, int n)
{
    double V[25], w[5];
    jacobi(A, V, w, 6, n);
    const double thr = svd_threshold(w, n);
    for (int i = 0; i < n; i++) x[i] = 0.0;
    for (int j = 0; j < n; j++) {
        if (!(w[j] > thr)) continue;
        double d = 0.0;
        for (int r = 0; r < 6; r++) d = d + A[r * n + j] * b[r];
        const double f = d / (w[j] * w[j]);
        for (int i = 0; i < n; i++) x[i] = x[i] + V[i * n + j] * f;
    }
}

/* column order of w descending (a stable selection: the lower index first on a tie) */
static void order_desc(const double* w, int n, int* ord)
{
    int used[12] = {0};
    for (int k = 0; k < n; k++) {
        int b = -1;
        for (int j = 0; j < n; j++)
            if (!used[j] && (b < 0 || w[j] > w[b])) b = j;
        used[b] = 1;
        ord[k] = b;
    }
}

/* the CTA's fixed summation order for S sums over the m points: P = PNP_THREADS / S chunks of C = ceil(m / P) consecutive points,
 * each summed in index order from 0, then the P chunk sums in chunk order from 0 (thread e P + k sums chunk k of sum e) */
typedef double (*pnp_term_fn)(const void* ctx, int e, int j);
static void pnp_reduce(int S, int m, pnp_term_fn term, const void* ctx, double* out)
{
    const int P = PNP_THREADS / S, C = (m + P - 1) / P;
    for (int e = 0; e < S; e++) {
        double tot = 0.0;
        for (int k = 0; k < P; k++) {
            double s = 0.0;
            const int j1 = (k + 1) * C < m ? (k + 1) * C : m;
            for (int j = k * C; j < j1; j++) s = s + term(ctx, e, j);
            tot = tot + s;
        }
        out[e] = tot;
    }
}

typedef struct {
    const double* pws; const double* us; const double* al; const double* pcs;
    const double* c0; const double* pc0;
    double fu, fv, uc, vc;
    const double* R; const double* t;
} EpnpCtx;

static const int SYM3[6][2] = {{0, 0}, {0, 1}, {0, 2}, {1, 1}, {1, 2}, {2, 2}};

static double term_pw(const void* p, int e, int j) { return ((const EpnpCtx*)p)->pws[3 * j + e]; }
static double term_pc(const void* p, int e, int j) { return ((const EpnpCtx*)p)->pcs[3 * j + e]; }
static double term_cov(const void* p, int e, int j)
{
    const EpnpCtx* c = (const EpnpCtx*)p;
    const double* w = c->pws + 3 * j;
    return (w[SYM3[e][0]] - c->c0[SYM3[e][0]]) * (w[SYM3[e][1]] - c->c0[SYM3[e][1]]);
}

/* entry (r, k) of EPnP's two rows of M for point j */
static double m_entry(const EpnpCtx* c, int j, int row, int k)
{
    const double a = c->al[4 * j + k / 3];
    const int s = k % 3;
    if (row == 0) return s == 0 ? a * c->fu : s == 1 ? 0.0 : a * (c->uc - c->us[2 * j]);
    return s == 0 ? 0.0 : s == 1 ? a * c->fv : a * (c->vc - c->us[2 * j + 1]);
}

static int MTM_P[78], MTM_Q[78];
static void mtm_pairs(void)
{
    int e = 0;
    for (int p = 0; p < 12; p++)
        for (int q = p; q < 12; q++) { MTM_P[e] = p; MTM_Q[e] = q; e++; }
}

static double term_mtm(const void* p, int e, int j)
{
    const EpnpCtx* c = (const EpnpCtx*)p;
    const int a = MTM_P[e], b = MTM_Q[e];
    return m_entry(c, j, 0, a) * m_entry(c, j, 0, b) + m_entry(c, j, 1, a) * m_entry(c, j, 1, b);
}

static double term_abt(const void* p, int e, int j)
{
    const EpnpCtx* c = (const EpnpCtx*)p;
    const int a = e / 3, b = e % 3;
    return (c->pcs[3 * j + a] - c->pc0[a]) * (c->pws[3 * j + b] - c->c0[b]);
}

static double term_rep(const void* p, int e, int j)
{
    const EpnpCtx* c = (const EpnpCtx*)p;
    (void)e;
    const double* pw = c->pws + 3 * j;
    const double Xc = pnp_dot(c->R, pw) + c->t[0], Yc = pnp_dot(c->R + 3, pw) + c->t[1];
    const double iz = 1.0 / (pnp_dot(c->R + 6, pw) + c->t[2]);
    const double ue = c->uc + (c->fu * Xc) * iz, ve = c->vc + (c->fv * Yc) * iz;
    const double du = c->us[2 * j] - ue, dv = c->us[2 * j + 1] - ve;
    return sqrt(du * du + dv * dv);
}

/* the butterfly sum of a warp's 32 lanes (every lane ends with this value) */
static double bfly(const double* v0)
{
    double v[32], w[32];
    memcpy(v, v0, sizeof(v));
    for (int o = 16; o >= 1; o >>= 1) {
        for (int l = 0; l < 32; l++) w[l] = v[l] + v[l ^ o];
        memcpy(v, w, sizeof(v));
    }
    return v[0];
}

/* one-sided Jacobi of the 12 x 12 M^T M as the device's warp runs it (lane r holds row r; lanes 12-31 hold zeros) */
static void jacobi12(double* A, double* V, double* nrm2)
{
    double col[32];
    for (int i = 0; i < 144; i++) V[i] = i % 13 == 0 ? 1.0 : 0.0;
    for (int s = 0; s < PNP_SWEEPS12; s++)
        for (int p = 0; p < 11; p++)
            for (int q = p + 1; q < 12; q++) {
                double va[32], vb[32], vg[32];
                for (int r = 0; r < 32; r++) {
                    const double x = r < 12 ? A[12 * r + p] : 0.0, y = r < 12 ? A[12 * r + q] : 0.0;
                    va[r] = x * x; vb[r] = y * y; vg[r] = x * y;
                }
                const double a = bfly(va), b = bfly(vb), g = bfly(vg);
                if (g == 0.0) continue;
                const double zeta = (b - a) / (2.0 * g);
                double t = 1.0 / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
                if (zeta < 0.0) t = -t;
                const double c = 1.0 / sqrt(1.0 + t * t), sn = c * t;
                for (int r = 0; r < 12; r++) {
                    double x = A[12 * r + p], y = A[12 * r + q];
                    A[12 * r + p] = c * x - sn * y;
                    A[12 * r + q] = sn * x + c * y;
                    x = V[12 * r + p]; y = V[12 * r + q];
                    V[12 * r + p] = c * x - sn * y;
                    V[12 * r + q] = sn * x + c * y;
                }
            }
    for (int j = 0; j < 12; j++) {
        for (int r = 0; r < 32; r++) col[r] = r < 12 ? A[12 * r + j] * A[12 * r + j] : 0.0;
        nrm2[j] = bfly(col);
    }
}

/* epnp::qr_solve of the 6 x 4 system (A, b overwritten); x is left as it is when A is singular, as OpenCV leaves it */
static void qr_solve(double* A, double* b, double* X)
{
    const int nr = 6, nc = 4;
    double A1[4], A2[4];
    for (int k = 0; k < nc; k++) {
        double eta = fabs(A[k * nc + k]);
        for (int i = k + 1; i < nr; i++) {
            const double elt = fabs(A[(i - 1) * nc + k]);       /* OpenCV compares the row above: ppAik1 moves after the read */
            if (eta < elt) eta = elt;
        }
        if (eta == 0.0) return;
        double sum2 = 0.0;
        const double inv_eta = 1.0 / eta;
        for (int i = k; i < nr; i++) {
            A[i * nc + k] = A[i * nc + k] * inv_eta;
            sum2 = sum2 + A[i * nc + k] * A[i * nc + k];
        }
        double sigma = sqrt(sum2);
        if (A[k * nc + k] < 0.0) sigma = -sigma;
        A[k * nc + k] = A[k * nc + k] + sigma;
        A1[k] = sigma * A[k * nc + k];
        A2[k] = -eta * sigma;
        for (int j = k + 1; j < nc; j++) {
            double sum = 0.0;
            for (int i = k; i < nr; i++) sum = sum + A[i * nc + k] * A[i * nc + j];
            const double tau = sum / A1[k];
            for (int i = k; i < nr; i++) A[i * nc + j] = A[i * nc + j] - tau * A[i * nc + k];
        }
    }
    for (int j = 0; j < nc; j++) {
        double tau = 0.0;
        for (int i = j; i < nr; i++) tau = tau + A[i * nc + j] * b[i];
        tau = tau / A1[j];
        for (int i = j; i < nr; i++) b[i] = b[i] - tau * A[i * nc + j];
    }
    X[nc - 1] = b[nc - 1] / A2[nc - 1];
    for (int i = nc - 2; i >= 0; i--) {
        double sum = 0.0;
        for (int j = i + 1; j < nc; j++) sum = sum + A[i * nc + j] * X[j];
        X[i] = (b[i] - sum) / A2[i];
    }
}

static void gauss_newton(const double* L, const double* rho, double* be)
{
    double x[4] = {0.0, 0.0, 0.0, 0.0};
    for (int it = 0; it < 5; it++) {
        double A[24], b[6];
        for (int i = 0; i < 6; i++) {
            const double* l = L + 10 * i;
            A[4 * i] = ((2.0 * l[0] * be[0] + l[1] * be[1]) + l[3] * be[2]) + l[6] * be[3];
            A[4 * i + 1] = ((l[1] * be[0] + 2.0 * l[2] * be[1]) + l[4] * be[2]) + l[7] * be[3];
            A[4 * i + 2] = ((l[3] * be[0] + l[4] * be[1]) + 2.0 * l[5] * be[2]) + l[8] * be[3];
            A[4 * i + 3] = ((l[6] * be[0] + l[7] * be[1]) + l[8] * be[2]) + 2.0 * l[9] * be[3];
            double s = l[0] * be[0] * be[0];
            s = s + l[1] * be[0] * be[1];
            s = s + l[2] * be[1] * be[1];
            s = s + l[3] * be[0] * be[2];
            s = s + l[4] * be[1] * be[2];
            s = s + l[5] * be[2] * be[2];
            s = s + l[6] * be[0] * be[3];
            s = s + l[7] * be[1] * be[3];
            s = s + l[8] * be[2] * be[3];
            s = s + l[9] * be[3] * be[3];
            b[i] = rho[i] - s;
        }
        qr_solve(A, b, x);
        for (int i = 0; i < 4; i++) be[i] = be[i] + x[i];
    }
}

/* the three beta approximations of epnp::compute_pose: L (6 x 10), rho (6) -> betas[k] (4) */
static void find_betas(const double* L, const double* rho, double (*be)[4])
{
    double A[30], b[5];
    for (int i = 0; i < 6; i++) { A[4 * i] = L[10 * i]; A[4 * i + 1] = L[10 * i + 1]; A[4 * i + 2] = L[10 * i + 3]; A[4 * i + 3] = L[10 * i + 6]; }
    lsq(A, rho, b, 4);
    if (b[0] < 0.0) {
        be[0][0] = sqrt(-b[0]); be[0][1] = -b[1] / be[0][0]; be[0][2] = -b[2] / be[0][0]; be[0][3] = -b[3] / be[0][0];
    } else {
        be[0][0] = sqrt(b[0]); be[0][1] = b[1] / be[0][0]; be[0][2] = b[2] / be[0][0]; be[0][3] = b[3] / be[0][0];
    }
    for (int i = 0; i < 6; i++) for (int k = 0; k < 3; k++) A[3 * i + k] = L[10 * i + k];
    lsq(A, rho, b, 3);
    if (b[0] < 0.0) { be[1][0] = sqrt(-b[0]); be[1][1] = b[2] < 0.0 ? sqrt(-b[2]) : 0.0; }
    else { be[1][0] = sqrt(b[0]); be[1][1] = b[2] > 0.0 ? sqrt(b[2]) : 0.0; }
    if (b[1] < 0.0) be[1][0] = -be[1][0];
    be[1][2] = 0.0; be[1][3] = 0.0;
    for (int i = 0; i < 6; i++) for (int k = 0; k < 5; k++) A[5 * i + k] = L[10 * i + k];
    lsq(A, rho, b, 5);
    if (b[0] < 0.0) { be[2][0] = sqrt(-b[0]); be[2][1] = b[2] < 0.0 ? sqrt(-b[2]) : 0.0; }
    else { be[2][0] = sqrt(b[0]); be[2][1] = b[2] > 0.0 ? sqrt(b[2]) : 0.0; }
    if (b[1] < 0.0) be[2][0] = -be[2][0];
    be[2][2] = b[3] / be[2][0]; be[2][3] = 0.0;
    for (int k = 0; k < 3; k++) gauss_newton(L, rho, be[k]);
}

/* L_6x10 and rho of epnp::compute_L_6x10 / compute_rho from the null vectors v (4 x 12, v[0] the smallest) and control points */
static void l6x10(const double (*v)[12], const double (*cws)[3], double* L, double* rho)
{
    double dv[4][6][3];
    for (int i = 0; i < 4; i++) {
        int a = 0, b = 1;
        for (int j = 0; j < 6; j++) {
            for (int k = 0; k < 3; k++) dv[i][j][k] = v[i][3 * a + k] - v[i][3 * b + k];
            b++;
            if (b > 3) { a++; b = a + 1; }
        }
    }
    for (int i = 0; i < 6; i++) {
        double* r = L + 10 * i;
        r[0] = pnp_dot(dv[0][i], dv[0][i]);
        r[1] = 2.0 * pnp_dot(dv[0][i], dv[1][i]);
        r[2] = pnp_dot(dv[1][i], dv[1][i]);
        r[3] = 2.0 * pnp_dot(dv[0][i], dv[2][i]);
        r[4] = 2.0 * pnp_dot(dv[1][i], dv[2][i]);
        r[5] = pnp_dot(dv[2][i], dv[2][i]);
        r[6] = 2.0 * pnp_dot(dv[0][i], dv[3][i]);
        r[7] = 2.0 * pnp_dot(dv[1][i], dv[3][i]);
        r[8] = 2.0 * pnp_dot(dv[2][i], dv[3][i]);
        r[9] = pnp_dot(dv[3][i], dv[3][i]);
    }
    const int PA[6] = {0, 0, 0, 1, 1, 2}, PB[6] = {1, 2, 3, 2, 3, 3};
    for (int i = 0; i < 6; i++) {
        double d[3];
        for (int k = 0; k < 3; k++) d[k] = cws[PA[i]][k] - cws[PB[i]][k];
        rho[i] = pnp_dot(d, d);
    }
}

/* R = U V^T of the SVD of abt (3 x 3 row-major), OpenCV's last-row flip when det R < 0; u3 = u1 x u2 where sigma3 <= 1e-8 sigma1 */
static void procrustes(const double* abt, double* R)
{
    double A[9], V[9], w[3], U[9];
    int ord[3];
    memcpy(A, abt, sizeof(A));
    jacobi(A, V, w, 3, 3);
    order_desc(w, 3, ord);
    double Vs[9];
    for (int k = 0; k < 3; k++) {
        const int j = ord[k];
        for (int r = 0; r < 3; r++) { U[3 * r + k] = w[j] > 0.0 ? A[3 * r + j] / w[j] : 0.0; Vs[3 * r + k] = V[3 * r + j]; }
    }
    if (!(w[ord[2]] > 1e-8 * w[ord[0]])) {
        const double u1[3] = {U[0], U[3], U[6]}, u2[3] = {U[1], U[4], U[7]};
        double u3[3];
        pnp_cross(u1, u2, u3);
        U[2] = u3[0]; U[5] = u3[1]; U[8] = u3[2];
    }
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) R[3 * i + j] = (U[3 * i] * Vs[3 * j] + U[3 * i + 1] * Vs[3 * j + 1]) + U[3 * i + 2] * Vs[3 * j + 2];
    const double det = ((((R[0] * R[4] * R[8] + R[1] * R[5] * R[6]) + R[2] * R[3] * R[7]) - R[2] * R[4] * R[6]) - R[1] * R[3] * R[8]) -
                       R[0] * R[5] * R[7];
    if (det < 0.0) { R[6] = -R[6]; R[7] = -R[7]; R[8] = -R[8]; }
}

/* epnp::compute_pose of n points (world pws (3 n), image us (2 n), already OpenCV's undistort round trip); R row-major, t */
void orc_pnp_epnp(const double* pws, const double* us, int n, double fu, double fv, double uc, double vc, double* Rout, double* tout)
{
    double* al = (double*)malloc(sizeof(double) * 4 * (size_t)n);
    double* pcs = (double*)malloc(sizeof(double) * 3 * (size_t)n);
    mtm_pairs();
    EpnpCtx c = {pws, us, al, pcs, NULL, NULL, fu, fv, uc, vc, NULL, NULL};
    double c0[3], cov6[6], cws[4][3];
    pnp_reduce(3, n, term_pw, &c, c0);
    for (int k = 0; k < 3; k++) c0[k] = c0[k] / n;
    c.c0 = c0;
    pnp_reduce(6, n, term_cov, &c, cov6);
    {
        double A[9], V[9], w[3];
        for (int e = 0; e < 6; e++) { A[3 * SYM3[e][0] + SYM3[e][1]] = cov6[e]; A[3 * SYM3[e][1] + SYM3[e][0]] = cov6[e]; }
        pnp_ocv_svd3(A, w, V);
        for (int k = 0; k < 3; k++) cws[0][k] = c0[k];
        for (int i = 1; i < 4; i++) {
            const double kk = sqrt(w[i - 1] / n);
            for (int j = 0; j < 3; j++) cws[i][j] = c0[j] + kk * V[3 * (i - 1) + j];
        }
    }
    double ci[9];
    {
        double A[9], V[9], w[3];
        for (int i = 0; i < 3; i++)
            for (int j = 1; j < 4; j++) A[3 * i + j - 1] = cws[j][i] - cws[0][i];
        jacobi(A, V, w, 3, 3);
        const double thr = svd_threshold(w, 3);
        for (int i = 0; i < 9; i++) ci[i] = 0.0;
        for (int j = 0; j < 3; j++) {
            if (!(w[j] > thr)) continue;
            const double w2 = w[j] * w[j];
            for (int r = 0; r < 3; r++)
                for (int q = 0; q < 3; q++) ci[3 * r + q] = ci[3 * r + q] + V[3 * r + j] * (A[3 * q + j] / w2);
        }
    }
    for (int i = 0; i < n; i++) {
        const double* p = pws + 3 * i;
        double* a = al + 4 * i;
        for (int j = 0; j < 3; j++) a[1 + j] = (ci[3 * j] * (p[0] - c0[0]) + ci[3 * j + 1] * (p[1] - c0[1])) + ci[3 * j + 2] * (p[2] - c0[2]);
        a[0] = ((1.0 - a[1]) - a[2]) - a[3];
    }
    double mtm[78], A[144], V[144], nrm2[12], v[4][12];
    pnp_reduce(78, n, term_mtm, &c, mtm);
    for (int e = 0; e < 78; e++) { A[12 * MTM_P[e] + MTM_Q[e]] = mtm[e]; A[12 * MTM_Q[e] + MTM_P[e]] = mtm[e]; }
    jacobi12(A, V, nrm2);
    {
        int ord[12];
        order_desc(nrm2, 12, ord);
        for (int i = 0; i < 4; i++)
            for (int k = 0; k < 12; k++) v[i][k] = V[12 * k + ord[11 - i]];
    }
    double L[60], rho[6], be[3][4], Rs[3][9], ts[3][3], rep[3];
    l6x10((const double (*)[12])v, (const double (*)[3])cws, L, rho);
    find_betas(L, rho, be);
    for (int N = 0; N < 3; N++) {
        double ccs[4][3];
        for (int j = 0; j < 4; j++)
            for (int k = 0; k < 3; k++) {
                double s = 0.0;
                for (int i = 0; i < 4; i++) s = s + be[N][i] * v[i][3 * j + k];
                ccs[j][k] = s;
            }
        const double z0 = ((al[0] * ccs[0][2] + al[1] * ccs[1][2]) + al[2] * ccs[2][2]) + al[3] * ccs[3][2];
        if (z0 < 0.0)
            for (int j = 0; j < 4; j++)
                for (int k = 0; k < 3; k++) ccs[j][k] = -ccs[j][k];
        for (int i = 0; i < n; i++) {
            const double* a = al + 4 * i;
            for (int k = 0; k < 3; k++) pcs[3 * i + k] = ((a[0] * ccs[0][k] + a[1] * ccs[1][k]) + a[2] * ccs[2][k]) + a[3] * ccs[3][k];
        }
        double pc0[3], abt[9];
        pnp_reduce(3, n, term_pc, &c, pc0);
        for (int k = 0; k < 3; k++) pc0[k] = pc0[k] / n;
        c.pc0 = pc0;
        pnp_reduce(9, n, term_abt, &c, abt);
        procrustes(abt, Rs[N]);
        for (int i = 0; i < 3; i++) ts[N][i] = pc0[i] - pnp_dot(Rs[N] + 3 * i, c0);
        c.R = Rs[N]; c.t = ts[N];
        double sum;
        pnp_reduce(1, n, term_rep, &c, &sum);
        rep[N] = sum / n;
    }
    int N = 0;
    if (rep[1] < rep[0]) N = 1;
    if (rep[2] < rep[N]) N = 2;
    memcpy(Rout, Rs[N], sizeof(double) * 9);
    memcpy(tout, ts[N], sizeof(double) * 3);
    free(al); free(pcs);
}

/* ------------------------------------------------------------------------------------------------ the whole call */
/* rvec, tvec: 3 each; mask n; returns 0, or -1 when out of memory */
int orc_solve_pnp_ransac(const float* xyz, const float* xy, const uint8_t* status, int n, double fx, double fy, double cx, double cy,
                         int iterations, float reproj_error, double confidence, double* rvec, double* tvec, uint8_t* mask, int* inliers,
                         int* ok)
{
    const size_t cap = (size_t)(n > 0 ? n : 1);
    float* P = (float*)malloc(sizeof(float) * 3 * cap);
    float* Q = (float*)malloc(sizeof(float) * 2 * cap);
    int* idx = (int*)malloc(sizeof(int) * cap);
    uint8_t* in = (uint8_t*)malloc(cap);
    double* pws = (double*)malloc(sizeof(double) * 3 * cap);
    double* us = (double*)malloc(sizeof(double) * 2 * cap);
    if (!P || !Q || !idx || !in || !pws || !us) { free(P); free(Q); free(idx); free(in); free(pws); free(us); return -1; }
    int m = 0;
    for (int i = 0; i < n; i++) {
        mask[i] = 0;
        if (status && !status[i]) continue;
        memcpy(P + 3 * m, xyz + 3 * i, 3 * sizeof(float));
        memcpy(Q + 2 * m, xy + 2 * i, 2 * sizeof(float));
        idx[m++] = i;
    }
    for (int k = 0; k < 3; k++) { rvec[k] = 0.0; tvec[k] = 0.0; }
    *inliers = 0; *ok = 0;
    const double thr = (double)reproj_error;
    const float t2 = (float)(thr * thr);
    double model[6], best[6];
    if (m == 4) {
        double X4[12];
        for (int k = 0; k < 12; k++) X4[k] = P[k];
        if (orc_pnp_model4(X4, Q, fx, fy, cx, cy, model)) {
            for (int k = 0; k < 3; k++) { rvec[k] = model[k]; tvec[k] = model[3 + k]; }
            for (int j = 0; j < 4; j++) mask[idx[j]] = 1;
            *inliers = 4; *ok = 1;
        }
    } else if (m > 4) {
        int niters = iterations > 1 ? iterations : 1, good = 0;
        uint64_t s = ~0ull;
        for (int it = 0; it < niters; it++) {
            int d[4];
            for (int i = 0; i < 4; i++) {
                int v;
                for (;;) {
                    v = (int)(rng_next(&s) % (unsigned)m);
                    int dup = 0;
                    for (int k = 0; k < i; k++) dup |= d[k] == v;
                    if (!dup) break;
                }
                d[i] = v;
            }
            double X4[12];
            float x4[8];
            for (int i = 0; i < 4; i++) {
                for (int k = 0; k < 3; k++) X4[3 * i + k] = P[3 * d[i] + k];
                x4[2 * i] = Q[2 * d[i]]; x4[2 * i + 1] = Q[2 * d[i] + 1];
            }
            if (!orc_pnp_model4(X4, x4, fx, fy, cx, cy, model)) continue;
            double R[9];
            orc_pnp_rodrigues_v2r(model, R);
            int cnt = 0;
            for (int j = 0; j < m; j++) cnt += pnp_err(R, model + 3, P + 3 * j, Q + 2 * j, fx, fy, cx, cy) <= t2;
            if (cnt > (good > 3 ? good : 3)) {
                good = cnt;
                memcpy(best, model, sizeof(best));
                niters = orc_pnp_update_niters(confidence, (double)(m - cnt) / m, niters);
            }
        }
        if (good > 0) {
            double R[9];
            orc_pnp_rodrigues_v2r(best, R);
            int ni = 0;
            const double ifx = 1.0 / fx, ify = 1.0 / fy;
            for (int j = 0; j < m; j++) {
                in[j] = pnp_err(R, best + 3, P + 3 * j, Q + 2 * j, fx, fy, cx, cy) <= t2;
                mask[idx[j]] = in[j];
                if (!in[j]) continue;
                for (int k = 0; k < 3; k++) pws[3 * ni + k] = P[3 * j + k];
                us[2 * ni] = (((double)Q[2 * j] - cx) * ifx) * fx + cx;
                us[2 * ni + 1] = (((double)Q[2 * j + 1] - cy) * ify) * fy + cy;
                ni++;
            }
            double Re[9];
            orc_pnp_epnp(pws, us, ni, fx, fy, cx, cy, Re, tvec);
            orc_pnp_rodrigues_r2v(Re, rvec);
            *inliers = good; *ok = 1;
        }
    }
    free(P); free(Q); free(idx); free(in); free(pws); free(us);
    return 0;
}
