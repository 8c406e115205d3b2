// hybvio_b200/csrc/pnp.cu -- cv::solvePnPRansac(xyz[used], xy[used], K, noArray(), rvec, tvec, false, iterations, reprojError, confidence,
// inliers, SOLVEPNP_P3P) on the device (OCV/calib3d/src/solvepnp.cpp, ptsetreg.cpp, epnp.cpp): absolute pose from 3-D points and their
// pixels, with outliers rejected, for one frame's tracks or many sessions per launch.
//
// One CTA per job (one launch for one call or a batch of up to HV_ESSENTIAL_BATCH_MAX). Per job:
//   1. the used points (status != 0) are compacted in index order by a block scan into scratch; the mask is zeroed;
//   2. m == 4: thread 0 forms the P3P model of the four points (every point an inlier, no refinement); m < 4: no result;
//   3. m > 4: RANSAC in waves of PNP_WARPS iterations. Thread 0 replays cv::RNG(~0)'s draws for the wave (4 distinct indices); lane 0
//      of warp w forms iteration base + w's model (P3P of the first three points, the solution that reprojects the fourth closest,
//      stored as (rvec, tvec) and turned back into R as OpenCV's model storage does); all 32 lanes score the m points (float32 squared
//      pixel distance <= (float)(thr * thr), counts reduced exactly); thread 0 runs the acceptance scan in iteration order: a count
//      above max(best, 3) wins and niters = RANSACUpdateNumIters(confidence, (m - count) / m, 4, niters). The loop stops once the next
//      wave starts at or past niters, so the result does not depend on the wave size;
//   4. the winner's inliers are compacted in index order (a second block scan) and go through one EPnP in double: the sums over the
//      points run over the CTA in a fixed order (pnp_reduce), the 12 x 12 eigenvectors on warp 0 (lane r holds row r), the small dense
//      steps on thread 0;
//   5. rvec, tvec, the mask (at the original indices), inliers and ok.
// The arithmetic is the oracle's (oracle/hv_oracle_pnp.c, which says what it computes and what is this library's own) operation for
// operation; this file is built with --fmad=false, so both round every product and sum alike. Only log and pow (the iteration bound)
// are CUDA's own, as in essential.cu.
#include "hv_common.cuh"
#include <cfloat>

#define PNP_THREADS 512
#define PNP_WARPS (PNP_THREADS / 32)
#define PNP_BISECT 64                 // bisection steps per root bracket: to one ulp from any interval of doubles
#define PNP_SWEEPS3 8                 // 3 x 3 and 6 x k Jacobi sweeps
#define PNP_SWEEPS12 12               // 12 x 12 (EPnP's M^T M) Jacobi sweeps

// ------------------------------------------------------------------------------------------------ serial steps (the oracle's)
/* sin and cos of th in [0, 4]: Taylor series of th / 8 (|x| <= 0.5, terms to x^19 / x^18), then three doublings */
__device__ static void pnp_sincos(double th, double* ps, double* pc)
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
__device__ static double pnp_atan01(double z)
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
__device__ static double pnp_atan2(double y, double x)
{
    const double ax = fabs(x);
    double a;
    if (y == 0.0 && ax == 0.0) a = 0.0;
    else if (y <= ax) a = pnp_atan01(y / ax);
    else a = 1.5707963267948966 - pnp_atan01(ax / y);
    return x < 0.0 ? 3.141592653589793 - a : a;
}

/* cv::Rodrigues, rotation vector -> R (row-major) */
__device__ static void pnp_rodrigues_v2r(const double* r, double* R)
{
    const double th = sqrt((r[0] * r[0] + r[1] * r[1]) + r[2] * r[2]);
    if (th < DBL_EPSILON) {
        for (int k = 0; k < 9; k++) R[k] = k % 4 == 0 ? 1.0 : 0.0;
        return;
    }
    double s, c;
    pnp_sincos(th, &s, &c);
    const double c1 = 1.0 - c, it = 1.0 / th;
    const double x = r[0] * it, y = r[1] * it, z = r[2] * it;
    const double rr[9] = {x * x, x * y, x * z, x * y, y * y, y * z, x * z, y * z, z * z};
    const double K[9] = {0.0, -z, y, z, 0.0, -x, -y, x, 0.0};
    for (int k = 0; k < 9; k++) R[k] = (c * (k % 4 == 0 ? 1.0 : 0.0) + c1 * rr[k]) + s * K[k];
}

/* cv::Rodrigues, R (row-major, orthonormal to rounding; OpenCV's U V^T projection is not restated) -> rotation vector, with
 * theta = atan2(s, c) for OpenCV's acos(c) */
__device__ static void pnp_rodrigues_r2v(const double* R, double* r)
{
    double x = R[7] - R[5], y = R[2] - R[6], z = R[3] - R[1];
    const double s = sqrt(((x * x + y * y) + z * z) * 0.25);
    double c = ((R[0] + R[4]) + R[8] - 1.0) * 0.5;
    c = c > 1.0 ? 1.0 : c < -1.0 ? -1.0 : c;
    double th = pnp_atan2(s, c);
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


__device__ static int pnp_sgn(double v) { return (v > 0.0) - (v < 0.0); }

__device__ static long long pnp_okey(double x)
{
    const long long b = __double_as_longlong(x);
    return b >= 0 ? b : -(b & 0x7fffffffffffffffll);
}

__device__ static double pnp_ofrom(long long k)
{
    return __longlong_as_double(k >= 0 ? k : (long long)((unsigned long long)(-k) | 0x8000000000000000ull));
}

__device__ static double pnp_horner(const double* c, int d, double x)
{
    double s = c[d];
    for (int i = d - 1; i >= 0; i--) s = s * x + c[i];
    return s;
}

/* double-double arithmetic (hi + lo), as in the essential solver: Grunert's quartic loses digits to cancellation in double, enough to
 * turn a close pair of real roots into a complex pair. Products go through an explicit fma, so that the device and this oracle agree. */
__device__ static void pnp_dd_fast(double s, double e, double* h, double* l)
{
    const double x = s + e;
    *h = x; *l = e - (x - s);
}

__device__ static void pnp_dd_add(const double* a, const double* b, double* r)
{
    const double s = a[0] + b[0], bb = s - a[0];
    const double e = (a[0] - (s - bb)) + (b[0] - bb);
    const double t = a[1] + b[1], tb = t - a[1];
    const double te = (a[1] - (t - tb)) + (b[1] - tb);
    double h, l;
    pnp_dd_fast(s, e + t, &h, &l);
    pnp_dd_fast(h, l + te, r, r + 1);
}

__device__ static void pnp_dd_sub(const double* a, const double* b, double* r)
{
    const double nb[2] = {-b[0], -b[1]};
    pnp_dd_add(a, nb, r);
}

__device__ static void pnp_dd_mul(const double* a, const double* b, double* r)
{
    const double p = a[0] * b[0];
    pnp_dd_fast(p, fma(a[0], b[0], -p) + (a[0] * b[1] + a[1] * b[0]), r, r + 1);
}

__device__ static void pnp_dd_mul_d(const double* a, double x, double* r)
{
    const double p = a[0] * x;
    pnp_dd_fast(p, fma(a[0], x, -p) + a[1] * x, r, r + 1);
}

__device__ static void pnp_dd_div(const double* a, const double* b, double* r)
{
    const double q1 = a[0] / b[0], q[2] = {q1, 0.0};
    double m[2], e[2];
    pnp_dd_mul(b, q, m);
    pnp_dd_sub(a, m, e);
    pnp_dd_fast(q1, e[0] / b[0], r, r + 1);
}

/* the sign of the quartic (double-double coefficients P, degree d) at x, by Horner's rule in double-double */
__device__ static int pnp_sgn_dd(const double* P, int d, double x)
{
    double s[2] = {P[2 * d], P[2 * d + 1]}, t[2];
    for (int i = d - 1; i >= 0; i--) {
        pnp_dd_mul_d(s, x, t);
        pnp_dd_add(t, P + 2 * i, s);
    }
    return (s[0] > 0.0) - (s[0] < 0.0);
}

/* the root of the degree-d polynomial c in (lo, hi] where it is monotonic: 1 and *root, or 0 */
__device__ static int pnp_interval_root(const double* c, int d, double lo, double hi, double* root)
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
__device__ static int pnp_interval_root_dd(const double* P, int d, double lo, double hi, double* root)
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
__device__ static int pnp_quartic_roots(const double* P, double* roots)
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

__device__ static void pnp_cross(const double* a, const double* b, double* c)
{
    c[0] = a[1] * b[2] - a[2] * b[1];
    c[1] = a[2] * b[0] - a[0] * b[2];
    c[2] = a[0] * b[1] - a[1] * b[0];
}

__device__ static double pnp_dot(const double* a, const double* b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }

/* the orthonormal frame (columns e1, e2, e3 of F, row-major) of the triangle a, b, c: e1 along b - a, e3 along (b - a) x (c - a) */
__device__ static int pnp_frame(const double* a, const double* b, const double* c, double* F)
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
__device__ static void pnp_ray(float u, float v, double fx, double fy, double cx, double cy, double* f)
{
    const double x = ((double)u - cx) / fx, y = ((double)v - cy) / fy;
    const double n = sqrt((x * x + y * y) + 1.0);
    f[0] = x / n; f[1] = y / n; f[2] = 1.0 / n;
}

/* the coefficients (ascending) of Grunert's quartic in v = s3 / s1 and of u = N(v) / (d0 + d1 v): K1 = d12^2 / d13^2,
 * K2 = d12^2 / d23^2; the two conics (1 + u^2 - 2 u c12) = K1 (1 + v^2 - 2 v c13) = K2 (u^2 + v^2 - 2 u v c23) */
__device__ static int pnp_grunert(const double* X, const double* f, double* P, double* Nc, double* Dc)
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
__device__ static void pnp_polish(double c12, double c13, double c23, double d12, double d13, double d23, double* pu, double* pv)
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
__device__ static int pnp_p3p(const double* X, const float* xy, double fx, double fy, double cx, double cy, double* Rs, double* ts)
{
    double f[9], Fw[9], P[10], Nc[3], Dc[2], roots[4];
    for (int i = 0; i < 3; i++) pnp_ray(xy[2 * i], xy[2 * i + 1], fx, fy, cx, cy, f + 3 * i);
    if (!pnp_frame(X, X + 3, X + 6, Fw)) return 0;
    if (!pnp_grunert(X, f, P, Nc, Dc)) return 0;
    double e[3];
    for (int k = 0; k < 3; k++) e[k] = X[k] - X[6 + k];
    const double d13 = pnp_dot(e, e), c13 = pnp_dot(f, f + 6), c12 = pnp_dot(f, f + 3), c23 = pnp_dot(f + 3, f + 6);
    for (int k = 0; k < 3; k++) e[k] = X[k] - X[3 + k];
    const double d12 = pnp_dot(e, e);
    for (int k = 0; k < 3; k++) e[k] = X[3 + k] - X[6 + k];
    const double d23 = pnp_dot(e, e);
    const int nr = pnp_quartic_roots(P, roots);
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
__device__ static int pnp_model4(const double* X4, const float* xy4, double fx, double fy, double cx, double cy, double* model)
{
    double Rs[36], ts[12];
    const int ns = pnp_p3p(X4, xy4, fx, fy, cx, cy, Rs, ts);
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
    pnp_rodrigues_r2v(Rs + 9 * best, model);
    for (int i = 0; i < 3; i++) model[3 + i] = ts[3 * best + i];
    return 1;
}


/* projectPoints' float32 image point under (R, t) and the float32 squared distance to (u, v) */
__device__ static float pnp_err(const double* R, const double* t, const float* X, const float* x, double fx, double fy, double cx, double cy)
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


/* cv::RANSACUpdateNumIters(p, ep, 4, niters) for p in (0, 1), ep in [0, 1] */
__device__ static int pnp_update_niters(double p, double ep, int niters)
{
    double num = 1.0 - p;
    if (num < DBL_MIN) num = DBL_MIN;
    double denom = 1.0 - pow(1.0 - ep, 4.0);
    if (denom < DBL_MIN) return 0;
    num = log(num);
    denom = log(denom);
    return denom >= 0.0 || -num >= niters * (-denom) ? niters : __double2int_rn(num / denom);
}


__device__ static void pnp_rotate(double* A, double* V, int rows, int ncols, int p, int q)
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
__device__ static void pnp_jacobi(double* A, double* V, double* w, int rows, int n)
{
    for (int i = 0; i < n * n; i++) V[i] = i % (n + 1) == 0 ? 1.0 : 0.0;
    for (int s = 0; s < PNP_SWEEPS3; s++)
        for (int p = 0; p < n - 1; p++)
            for (int q = p + 1; q < n; q++) pnp_rotate(A, V, rows, n, p, q);
    for (int j = 0; j < n; j++) {
        double s = 0.0;
        for (int r = 0; r < rows; r++) s = s + A[r * n + j] * A[r * n + j];
        w[j] = sqrt(s);
    }
}

__device__ static double pnp_svd_threshold(const double* w, int n)
{
    double s = 0.0;
    for (int j = 0; j < n; j++) s = s + w[j];
    return s * (2.0 * DBL_EPSILON);
}

/* OpenCV's JacobiSVDImpl_ (OCV/core/src/lapack.cpp) on the symmetric 3 x 3 A, restated for its sign convention, which decides EPnP's
 * control points and so its pose on noisy points: one-sided rotations of the rows of A^T until none changes (at most 30 sweeps), the
 * rotation of OpenCV's branch on beta = |row i|^2 - |row j|^2, hypot as sqrt(p^2 + beta^2); w descending (the first of equal norms kept
 * first), u's rows the unit left singular vectors (zero where w <= DBL_MIN) */
__device__ static void pnp_ocv_svd3(const double* A, double* w, double* u)
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
__device__ static void pnp_lsq(double* A, const double* b, double* x, int n)
{
    double V[25], w[5];
    pnp_jacobi(A, V, w, 6, n);
    const double thr = pnp_svd_threshold(w, n);
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
__device__ static void pnp_order_desc(const double* w, int n, int* ord)
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


/* epnp::qr_solve of the 6 x 4 system (A, b overwritten); x is left as it is when A is singular, as OpenCV leaves it */
__device__ static void pnp_qr_solve(double* A, double* b, double* X)
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

__device__ static void pnp_gauss_newton(const double* L, const double* rho, double* be)
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
        pnp_qr_solve(A, b, x);
        for (int i = 0; i < 4; i++) be[i] = be[i] + x[i];
    }
}

/* the three beta approximations of epnp::compute_pose: L (6 x 10), rho (6) -> betas[k] (4) */
__device__ static void pnp_find_betas(const double* L, const double* rho, double (*be)[4])
{
    double A[30], b[5];
    for (int i = 0; i < 6; i++) { A[4 * i] = L[10 * i]; A[4 * i + 1] = L[10 * i + 1]; A[4 * i + 2] = L[10 * i + 3]; A[4 * i + 3] = L[10 * i + 6]; }
    pnp_lsq(A, rho, b, 4);
    if (b[0] < 0.0) {
        be[0][0] = sqrt(-b[0]); be[0][1] = -b[1] / be[0][0]; be[0][2] = -b[2] / be[0][0]; be[0][3] = -b[3] / be[0][0];
    } else {
        be[0][0] = sqrt(b[0]); be[0][1] = b[1] / be[0][0]; be[0][2] = b[2] / be[0][0]; be[0][3] = b[3] / be[0][0];
    }
    for (int i = 0; i < 6; i++) for (int k = 0; k < 3; k++) A[3 * i + k] = L[10 * i + k];
    pnp_lsq(A, rho, b, 3);
    if (b[0] < 0.0) { be[1][0] = sqrt(-b[0]); be[1][1] = b[2] < 0.0 ? sqrt(-b[2]) : 0.0; }
    else { be[1][0] = sqrt(b[0]); be[1][1] = b[2] > 0.0 ? sqrt(b[2]) : 0.0; }
    if (b[1] < 0.0) be[1][0] = -be[1][0];
    be[1][2] = 0.0; be[1][3] = 0.0;
    for (int i = 0; i < 6; i++) for (int k = 0; k < 5; k++) A[5 * i + k] = L[10 * i + k];
    pnp_lsq(A, rho, b, 5);
    if (b[0] < 0.0) { be[2][0] = sqrt(-b[0]); be[2][1] = b[2] < 0.0 ? sqrt(-b[2]) : 0.0; }
    else { be[2][0] = sqrt(b[0]); be[2][1] = b[2] > 0.0 ? sqrt(b[2]) : 0.0; }
    if (b[1] < 0.0) be[2][0] = -be[2][0];
    be[2][2] = b[3] / be[2][0]; be[2][3] = 0.0;
    for (int k = 0; k < 3; k++) pnp_gauss_newton(L, rho, be[k]);
}

/* L_6x10 and rho of epnp::compute_L_6x10 / compute_rho from the null vectors v (4 x 12, v[0] the smallest) and control points */
__device__ static void pnp_l6x10(const double (*v)[12], const double (*cws)[3], double* L, double* rho)
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

/* R = U V^T of the SVD of abt (3 x 3 row-major), OpenCV's last-row flip when det R < 0. Where sigma3 <= 1e-8 sigma1 (points on a
 * plane) u3 is not determined by abt and is taken as det(V) (u1 x u2), so that det R = +1 and R is the nearest rotation: u1 x u2 alone
 * gives det R = det V, and the flip of a reflection's last row is not the nearest rotation. */
__device__ static void pnp_procrustes(const double* abt, double* R)
{
    double A[9], V[9], w[3], U[9];
    int ord[3];
    memcpy(A, abt, sizeof(A));
    pnp_jacobi(A, V, w, 3, 3);
    pnp_order_desc(w, 3, ord);
    double Vs[9];
    for (int k = 0; k < 3; k++) {
        const int j = ord[k];
        for (int r = 0; r < 3; r++) { U[3 * r + k] = w[j] > 0.0 ? A[3 * r + j] / w[j] : 0.0; Vs[3 * r + k] = V[3 * r + j]; }
    }
    if (!(w[ord[2]] > 1e-8 * w[ord[0]])) {
        const double u1[3] = {U[0], U[3], U[6]}, u2[3] = {U[1], U[4], U[7]};
        double u3[3];
        pnp_cross(u1, u2, u3);
        const double dv = ((((Vs[0] * Vs[4] * Vs[8] + Vs[1] * Vs[5] * Vs[6]) + Vs[2] * Vs[3] * Vs[7]) - Vs[2] * Vs[4] * Vs[6]) -
                           Vs[1] * Vs[3] * Vs[8]) - Vs[0] * Vs[5] * Vs[7];
        const double sg = dv < 0.0 ? -1.0 : 1.0;
        U[2] = sg * u3[0]; U[5] = sg * u3[1]; U[8] = sg * u3[2];
    }
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) R[3 * i + j] = (U[3 * i] * Vs[3 * j] + U[3 * i + 1] * Vs[3 * j + 1]) + U[3 * i + 2] * Vs[3 * j + 2];
    const double det = ((((R[0] * R[4] * R[8] + R[1] * R[5] * R[6]) + R[2] * R[3] * R[7]) - R[2] * R[4] * R[6]) - R[1] * R[3] * R[8]) -
                       R[0] * R[5] * R[7];
    if (det < 0.0) { R[6] = -R[6]; R[7] = -R[7]; R[8] = -R[8]; }
}


__device__ __forceinline__ unsigned pnp_rng_next(unsigned long long* s)
{
    *s = (unsigned long long)(unsigned)*s * 4164903690ull + (unsigned)(*s >> 32);
    return (unsigned)*s;
}

// ------------------------------------------------------------------------------------------------ the CTA's steps
// the butterfly sum over the warp's 32 lanes (every lane ends with the same value)
__device__ __forceinline__ double pnp_bfly(double v, int lane)
{
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) v = v + __shfl_sync(0xffffffffu, v, lane ^ o);
    return v;
}

struct PnpShared {
    double model[PNP_WARPS][6];       // (rvec, tvec) of each warp's iteration
    double Rw[PNP_WARPS][9];          // its R = Rodrigues(rvec)
    double best[6], Rb[9];
    int sub[PNP_WARPS][4];
    int has[PNP_WARPS], cnt[PNP_WARPS];
    int warpSum[PNP_WARPS];
    unsigned long long rng;
    int m, niters, good, base, ni, ok;
    // EPnP
    double part[PNP_THREADS];
    double sums[78];
    double c0[3], cws[4][3], ci[9], pc0[3], ccs[4][3];
    double A12[144], V12[144], nrm2[12], v[4][12];
    double L[60], rho[6], be[3][4], Rs[3][9], ts[3][3], rep[3];
};

// the exclusive offset of this thread's `cnt` flagged items among the CTA's (threads in order); *total: the CTA's count
__device__ static int pnp_scan(int cnt, PnpShared& s, int* total)
{
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int incl = cnt;
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    if (lane == 31) s.warpSum[warp] = incl;
    __syncthreads();
    int off = incl - cnt;
    for (int w = 0; w < warp; w++) off += s.warpSum[w];
    if (tid == PNP_THREADS - 1) *total = off + cnt;
    __syncthreads();
    return off;
}

// S sums over m points in the oracle's fixed order (pnp_reduce there): thread e P + k sums chunk k of sum e, thread e the chunks
template <class F>
__device__ static void pnp_reduce(int S, int m, const F& term, PnpShared& s, double* out)
{
    const int tid = threadIdx.x, P = PNP_THREADS / S, C = (m + P - 1) / P;
    if (tid < S * P) {
        const int e = tid / P, k = tid % P, j1 = min(m, (k + 1) * C);
        double acc = 0.0;
        for (int j = k * C; j < j1; j++) acc = acc + term(e, j);
        s.part[tid] = acc;
    }
    __syncthreads();
    if (tid < S) {
        double tot = 0.0;
        for (int k = 0; k < P; k++) tot = tot + s.part[tid * P + k];
        out[tid] = tot;
    }
    __syncthreads();
}

__constant__ signed char PNP_SYM3[6][2] = {{0, 0}, {0, 1}, {0, 2}, {1, 1}, {1, 2}, {2, 2}};

// one-sided Jacobi of the 12 x 12 M^T M in s.A12 on one warp (lane r holds row r of A and V in registers); V to s.V12, the squared
// column norms to s.nrm2
__device__ static void pnp_jacobi12(PnpShared& s, int lane)
{
    double A[12], V[12];
#pragma unroll
    for (int k = 0; k < 12; k++) { A[k] = lane < 12 ? s.A12[12 * lane + k] : 0.0; V[k] = lane == k ? 1.0 : 0.0; }
#pragma unroll 1
    for (int sw = 0; sw < PNP_SWEEPS12; sw++) {
#pragma unroll
        for (int p = 0; p < 11; p++)
#pragma unroll
            for (int q = p + 1; q < 12; q++) {
                const double x = A[p], y = A[q];
                const double a = pnp_bfly(x * x, lane), b = pnp_bfly(y * y, lane), g = pnp_bfly(x * y, lane);
                if (g == 0.0) continue;
                const double zeta = (b - a) / (2.0 * g);
                double t = 1.0 / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
                if (zeta < 0.0) t = -t;
                const double c = 1.0 / sqrt(1.0 + t * t), sn = c * t;
                A[p] = c * x - sn * y;
                A[q] = sn * x + c * y;
                const double vx = V[p], vy = V[q];
                V[p] = c * vx - sn * vy;
                V[q] = sn * vx + c * vy;
            }
    }
#pragma unroll
    for (int j = 0; j < 12; j++) {
        const double nn = pnp_bfly(A[j] * A[j], lane);
        if (lane == 0) s.nrm2[j] = nn;
        if (lane < 12) s.V12[12 * lane + j] = V[j];
    }
}

// epnp::compute_pose of the n compacted inliers (a.pws, a.us); R, t of the chosen beta approximation to s.Rs[N], s.ts[N], N returned
// to thread 0
__device__ static int pnp_epnp(const PnpArgs& a, int n, PnpShared& s)
{
    const int tid = threadIdx.x, lane = tid & 31;
    const double fu = a.fx, fv = a.fy, uc = a.cx, vc = a.cy;
    const double* pws = a.pws;
    const double* us = a.us;
    double* al = a.al;
    double* pcs = a.pcs;
    pnp_reduce(3, n, [&](int e, int j) { return pws[3 * j + e]; }, s, s.c0);
    if (tid < 3) s.c0[tid] = s.c0[tid] / n;
    __syncthreads();
    pnp_reduce(6, n, [&](int e, int j) {
        const double* w = pws + 3 * j;
        const int p = PNP_SYM3[e][0], q = PNP_SYM3[e][1];
        return (w[p] - s.c0[p]) * (w[q] - s.c0[q]);
    }, s, s.sums);
    if (tid == 0) {
        double A[9], V[9], w[3];
        for (int e = 0; e < 6; e++) { A[3 * PNP_SYM3[e][0] + PNP_SYM3[e][1]] = s.sums[e]; A[3 * PNP_SYM3[e][1] + PNP_SYM3[e][0]] = s.sums[e]; }
        pnp_ocv_svd3(A, w, V);
        for (int k = 0; k < 3; k++) s.cws[0][k] = s.c0[k];
        for (int i = 1; i < 4; i++) {
            const double kk = sqrt(w[i - 1] / n);
            for (int j = 0; j < 3; j++) s.cws[i][j] = s.c0[j] + kk * V[3 * (i - 1) + j];
        }
        for (int i = 0; i < 3; i++)
            for (int j = 1; j < 4; j++) A[3 * i + j - 1] = s.cws[j][i] - s.cws[0][i];
        pnp_jacobi(A, V, w, 3, 3);
        const double thr = pnp_svd_threshold(w, 3);
        double ci[9];
        for (int i = 0; i < 9; i++) ci[i] = 0.0;
        for (int j = 0; j < 3; j++) {
            if (!(w[j] > thr)) continue;
            const double w2 = w[j] * w[j];
            for (int r = 0; r < 3; r++)
                for (int q = 0; q < 3; q++) ci[3 * r + q] = ci[3 * r + q] + V[3 * r + j] * (A[3 * q + j] / w2);
        }
        for (int i = 0; i < 9; i++) s.ci[i] = ci[i];
    }
    __syncthreads();
    for (int i = tid; i < n; i += PNP_THREADS) {
        const double* p = pws + 3 * i;
        double* al4 = al + 4 * i;
        double b[3];
        for (int j = 0; j < 3; j++) b[j] = (s.ci[3 * j] * (p[0] - s.c0[0]) + s.ci[3 * j + 1] * (p[1] - s.c0[1])) + s.ci[3 * j + 2] * (p[2] - s.c0[2]);
        al4[1] = b[0]; al4[2] = b[1]; al4[3] = b[2];
        al4[0] = ((1.0 - b[0]) - b[1]) - b[2];
    }
    __syncthreads();
    pnp_reduce(78, n, [&](int e, int j) {
        int p = 0, rem = e;
        while (rem >= 12 - p) { rem -= 12 - p; p++; }
        const int q = p + rem;
        const double ap = al[4 * j + p / 3], aq = al[4 * j + q / 3];
        const double du = uc - us[2 * j], dv = vc - us[2 * j + 1];
        const int sp = p % 3, sq = q % 3;
        const double m1p = sp == 0 ? ap * fu : sp == 1 ? 0.0 : ap * du, m1q = sq == 0 ? aq * fu : sq == 1 ? 0.0 : aq * du;
        const double m2p = sp == 0 ? 0.0 : sp == 1 ? ap * fv : ap * dv, m2q = sq == 0 ? 0.0 : sq == 1 ? aq * fv : aq * dv;
        return m1p * m1q + m2p * m2q;
    }, s, s.sums);
    if (tid < 78) {
        int p = 0, rem = tid;
        while (rem >= 12 - p) { rem -= 12 - p; p++; }
        const int q = p + rem;
        s.A12[12 * p + q] = s.sums[tid];
        s.A12[12 * q + p] = s.sums[tid];
    }
    __syncthreads();
    if (tid < 32) pnp_jacobi12(s, lane);
    __syncthreads();
    if (tid == 0) {
        int ord[12];
        pnp_order_desc(s.nrm2, 12, ord);
        for (int i = 0; i < 4; i++)
            for (int k = 0; k < 12; k++) s.v[i][k] = s.V12[12 * k + ord[11 - i]];
        pnp_l6x10((const double (*)[12])s.v, (const double (*)[3])s.cws, s.L, s.rho);
        pnp_find_betas(s.L, s.rho, s.be);
    }
    __syncthreads();
    for (int N = 0; N < 3; N++) {
        if (tid == 0) {
            double ccs[4][3];
            for (int j = 0; j < 4; j++)
                for (int k = 0; k < 3; k++) {
                    double t = 0.0;
                    for (int i = 0; i < 4; i++) t = t + s.be[N][i] * s.v[i][3 * j + k];
                    ccs[j][k] = t;
                }
            const double z0 = ((al[0] * ccs[0][2] + al[1] * ccs[1][2]) + al[2] * ccs[2][2]) + al[3] * ccs[3][2];
            for (int j = 0; j < 4; j++)
                for (int k = 0; k < 3; k++) s.ccs[j][k] = z0 < 0.0 ? -ccs[j][k] : ccs[j][k];
        }
        __syncthreads();
        for (int i = tid; i < n; i += PNP_THREADS) {
            const double* a4 = al + 4 * i;
            for (int k = 0; k < 3; k++) pcs[3 * i + k] = ((a4[0] * s.ccs[0][k] + a4[1] * s.ccs[1][k]) + a4[2] * s.ccs[2][k]) + a4[3] * s.ccs[3][k];
        }
        __syncthreads();
        pnp_reduce(3, n, [&](int e, int j) { return pcs[3 * j + e]; }, s, s.pc0);
        if (tid < 3) s.pc0[tid] = s.pc0[tid] / n;
        __syncthreads();
        pnp_reduce(9, n, [&](int e, int j) { return (pcs[3 * j + e / 3] - s.pc0[e / 3]) * (pws[3 * j + e % 3] - s.c0[e % 3]); }, s, s.sums);
        if (tid == 0) {
            pnp_procrustes(s.sums, s.Rs[N]);
            for (int i = 0; i < 3; i++) s.ts[N][i] = s.pc0[i] - pnp_dot(s.Rs[N] + 3 * i, s.c0);
        }
        __syncthreads();
        const double* R = s.Rs[N];
        const double* t = s.ts[N];
        pnp_reduce(1, n, [&](int, int j) {
            const double* pw = pws + 3 * j;
            const double Xc = pnp_dot(R, pw) + t[0], Yc = pnp_dot(R + 3, pw) + t[1];
            const double iz = 1.0 / (pnp_dot(R + 6, pw) + t[2]);
            const double ue = uc + (fu * Xc) * iz, ve = vc + (fv * Yc) * iz;
            const double du = us[2 * j] - ue, dv = us[2 * j + 1] - ve;
            return sqrt(du * du + dv * dv);
        }, s, s.rep + N);
        if (tid == 0) s.rep[N] = s.rep[N] / n;
        __syncthreads();
    }
    int N = 0;
    if (s.rep[1] < s.rep[0]) N = 1;
    if (s.rep[2] < s.rep[N]) N = 2;
    return N;
}

__device__ static void pnp_job(const PnpArgs& a, int iterations, float reprojError, double confidence, PnpShared& s)
{
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n = a.n;
    // 1. compaction in index order: thread t scans [t c, (t + 1) c)
    const int chunk = (n + PNP_THREADS - 1) / PNP_THREADS;
    const int i0 = min(n, tid * chunk), i1 = min(n, i0 + chunk);
    int used = 0;
    for (int i = i0; i < i1; i++) used += a.status == nullptr || a.status[i] != 0;
    int off = pnp_scan(used, s, &s.m);
    for (int i = i0; i < i1; i++) {
        a.mask[i] = 0;
        if (a.status != nullptr && a.status[i] == 0) continue;
        a.P[3 * off] = a.xyz[3 * i]; a.P[3 * off + 1] = a.xyz[3 * i + 1]; a.P[3 * off + 2] = a.xyz[3 * i + 2];
        a.Q[off] = a.xy[i];
        a.idx[off] = i;
        off++;
    }
    if (tid == 0) { s.ok = 0; s.good = 0; }
    __syncthreads();
    const int m = s.m;
    const double thr = (double)reprojError;
    const float t2 = (float)(thr * thr);
    const double fx = a.fx, fy = a.fy, cx = a.cx, cy = a.cy;
    int N = -1;
    if (m == 4) {
        if (tid == 0) {
            double X4[12];
            for (int k = 0; k < 12; k++) X4[k] = a.P[k];
            s.ok = pnp_model4(X4, reinterpret_cast<const float*>(a.Q), fx, fy, cx, cy, s.best);
            s.good = s.ok ? 4 : 0;
        }
        __syncthreads();
        if (tid < 4 && s.ok) a.mask[a.idx[tid]] = 1;
    } else if (m > 4) {
        if (tid == 0) { s.niters = iterations > 1 ? iterations : 1; s.rng = ~0ull; s.base = 0; }
        __syncthreads();
        for (;;) {
            const int base = s.base, niters = s.niters;
            if (base >= niters) break;
            if (tid == 0) {
                unsigned long long st = s.rng;
                for (int w = 0; w < PNP_WARPS && base + w < niters; w++)
                    for (int i = 0; i < 4; i++) {
                        int v;
                        for (;;) {
                            v = (int)(pnp_rng_next(&st) % (unsigned)m);
                            int dup = 0;
                            for (int k = 0; k < i; k++) dup |= s.sub[w][k] == v;
                            if (!dup) break;
                        }
                        s.sub[w][i] = v;
                    }
                s.rng = st;
            }
            __syncthreads();
            if (base + warp < niters) {
                if (lane == 0) {
                    double X4[12];
                    float x4[8];
                    for (int i = 0; i < 4; i++) {
                        const int d = s.sub[warp][i];
                        for (int k = 0; k < 3; k++) X4[3 * i + k] = a.P[3 * d + k];
                        x4[2 * i] = a.Q[d].x; x4[2 * i + 1] = a.Q[d].y;
                    }
                    const int h = pnp_model4(X4, x4, fx, fy, cx, cy, s.model[warp]);
                    if (h) pnp_rodrigues_v2r(s.model[warp], s.Rw[warp]);
                    s.has[warp] = h;
                }
                __syncwarp();
                if (s.has[warp]) {
                    double R[9], t[3];
                    for (int k = 0; k < 9; k++) R[k] = s.Rw[warp][k];
                    for (int k = 0; k < 3; k++) t[k] = s.model[warp][3 + k];
                    int c = 0;
                    for (int j = lane; j < m; j += 32) c += pnp_err(R, t, a.P + 3 * j, reinterpret_cast<const float*>(a.Q + j), fx, fy, cx, cy) <= t2;
                    c = __reduce_add_sync(0xffffffffu, c);
                    if (lane == 0) s.cnt[warp] = c;
                }
            }
            __syncthreads();
            if (tid == 0) {
                int nit = niters, g = s.good;
                for (int w = 0; w < PNP_WARPS && base + w < nit; w++) {
                    if (!s.has[w]) continue;
                    const int c = s.cnt[w];
                    if (c > (g > 3 ? g : 3)) {
                        g = c;
                        for (int k = 0; k < 6; k++) s.best[k] = s.model[w][k];
                        nit = pnp_update_niters(confidence, (double)(m - c) / m, nit);
                    }
                }
                s.good = g; s.niters = nit; s.base = base + PNP_WARPS;
            }
            __syncthreads();
        }
        if (s.good > 0) {
            if (tid == 0) { pnp_rodrigues_v2r(s.best, s.Rb); s.ok = 1; }
            __syncthreads();
            // 4. the inliers in index order: thread t scans [t c, (t + 1) c) of the m used points
            const int mc = (m + PNP_THREADS - 1) / PNP_THREADS;
            const int j0 = min(m, tid * mc), j1 = min(m, j0 + mc);
            int cnt = 0;
            for (int j = j0; j < j1; j++) cnt += pnp_err(s.Rb, s.best + 3, a.P + 3 * j, reinterpret_cast<const float*>(a.Q + j), fx, fy, cx, cy) <= t2;
            int o = pnp_scan(cnt, s, &s.ni);
            const double ifx = 1.0 / fx, ify = 1.0 / fy;
            for (int j = j0; j < j1; j++) {
                const int in = pnp_err(s.Rb, s.best + 3, a.P + 3 * j, reinterpret_cast<const float*>(a.Q + j), fx, fy, cx, cy) <= t2;
                a.mask[a.idx[j]] = (uint8_t)in;
                if (!in) continue;
                for (int k = 0; k < 3; k++) a.pws[3 * o + k] = a.P[3 * j + k];
                a.us[2 * o] = (((double)a.Q[j].x - cx) * ifx) * fx + cx;
                a.us[2 * o + 1] = (((double)a.Q[j].y - cy) * ify) * fy + cy;
                o++;
            }
            __syncthreads();
            N = pnp_epnp(a, s.ni, s);
        }
    }
    // 5. outputs
    if (tid == 0) {
        double r[3] = {0.0, 0.0, 0.0}, t[3] = {0.0, 0.0, 0.0};
        if (s.ok && N < 0) { for (int k = 0; k < 3; k++) { r[k] = s.best[k]; t[k] = s.best[3 + k]; } }
        else if (s.ok) { pnp_rodrigues_r2v(s.Rs[N], r); for (int k = 0; k < 3; k++) t[k] = s.ts[N][k]; }
        for (int k = 0; k < 3; k++) { a.rvec[k] = r[k]; a.tvec[k] = t[k]; }
        *a.inliers = s.ok ? s.good : 0;
        *a.ok = s.ok;
    }
}

__global__ void __launch_bounds__(PNP_THREADS, 1) hv_pnp_kernel(const __grid_constant__ PnpBatchArgs b)
{
    extern __shared__ __align__(16) unsigned char pnp_smem[];
    pnp_job(b.job[blockIdx.x], b.iterations, b.reprojError, b.confidence, *reinterpret_cast<PnpShared*>(pnp_smem));
}

cudaError_t hv_launch_pnp(const PnpBatchArgs& b, int njobs, cudaStream_t stream)
{
    static_assert(sizeof(PnpShared) <= 48 * 1024, "pnp workspace exceeds the default dynamic shared memory of a CTA");
    hv_pnp_kernel<<<njobs, PNP_THREADS, sizeof(PnpShared), stream>>>(b);
    return cudaGetLastError();
}
