/* oracle/hv_oracle_essential.c -- TEST INFRASTRUCTURE: plain-C restatement of
 *   cv::findEssentialMat(xy1[used], xy2[used], K, RANSAC, prob, threshold, maxIters, mask)
 * (OCV/calib3d/src/five-point.cpp, ptsetreg.cpp) as the device computes it (hybvio_b200/csrc/essential.cu), operation for operation:
 *   1. used points: status != 0 (every point without a status), compacted in index order; m = their count.
 *   2. normalisation as findEssentialMat's MatExpr does it: x' = x * (1 / fx) + (-cx) * (1 / fx), y' likewise with fy, cy, in double;
 *      threshold' = threshold / ((fx + fy) / 2); an error e (float) is an inlier iff e <= (float)(threshold'^2).
 *   3. m < 5: no solution. m == 5: every solution of the five points, all five in the mask.
 *   4. m > 5: RANSACPointSetRegistrator::run: cv::RNG seeded with ~0; each iteration draws 5 distinct indices with rng.uniform(0, m)
 *      (a repeated index is drawn again); every solution of the subset is scored by its Sampson error
 *      (float)((x2' E x1)^2 / ((Ex1)_0^2 + (Ex1)_1^2 + (E^T x2)_0^2 + (E^T x2)_1^2)); a count above max(best, 4) wins (strict),
 *      and niters = RANSACUpdateNumIters(prob, (m - count) / m, 5, niters), which only shrinks it. maxIters <= 0 runs one iteration.
 * The five-point solver is this project's own (OpenCV's SVD, matrix inverse and Durand-Kerner root finder are iterative and not
 * restated); mathematically it solves the same system, so it returns the same essential matrices up to rounding:
 *   a. Householder QR of the 5 x 9 epipolar matrix Q^T; the last four columns of the orthogonal factor span the null space of Q:
 *      E = x X + y Y + z Z + W;
 *   b. the ten cubic constraints det(E) = 0 and E E^T E - tr(E E^T) E / 2 = 0 in the 20 monomials of x, y, z (Nister's order);
 *   c. Gauss-Jordan elimination with partial pivoting of the 10 x 20 coefficient matrix;
 *   d. the 3 x 3 matrix of polynomials in z (rows <e> - z <f>, <g> - z <h>, <i> - z <j>) and its degree-10 determinant;
 *   e. the real roots of the determinant by recursion on the derivatives: the real roots of p' split the real line into intervals on
 *      which p is monotonic; an interval whose ends differ in sign holds one root, bracketed by 48 bisection steps on the ordered bit
 *      patterns of doubles (within 2^16 ulps at the end, whatever the root's magnitude): a fixed amount of work for any data;
 *   f. per root, ascending: (x, y, 1) from the largest cross product of two rows of the 3 x 3 matrix (skipped when the unit vector's
 *      last entry is below 1e-10, as OpenCV skips it), (x, y, z) polished by Gauss-Newton steps on the ten constraints, E normalised
 *      to unit Frobenius norm.
 * Built with -ffp-contract=off, so no multiply-add is contracted; the kernel is built with --fmad=false.
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ESS_MAX_SOL 10

/* quadratic monomial of (linear variable u) * (linear variable v); variables x, y, z, 1 */
static const int QI[4][4] = {{0, 1, 2, 3}, {1, 4, 5, 6}, {2, 5, 7, 8}, {3, 6, 8, 9}};
/* cubic monomial (Nister's order: x3 y3 x2y xy2 x2z x2 y2z y2 xyz xy | xz2 xz x yz2 yz y z3 z2 z 1) of quadratic q * variable v;
 * quadratic monomials: xx xy xz x yy yz y zz z 1 */
static const int CI[10][4] = {{0, 2, 4, 5}, {2, 3, 8, 9}, {4, 8, 10, 11}, {5, 9, 11, 12}, {3, 1, 6, 7},
                              {8, 6, 13, 14}, {9, 7, 14, 15}, {10, 13, 16, 17}, {11, 14, 17, 18}, {12, 15, 18, 19}};

static void mul_ll(const double* a, const double* b, double* q)
{
    for (int k = 0; k < 10; k++) q[k] = 0.0;
    for (int u = 0; u < 4; u++)
        for (int v = 0; v < 4; v++) q[QI[u][v]] = q[QI[u][v]] + a[u] * b[v];
}

static void mul_ql(const double* q, const double* l, double* c)
{
    for (int k = 0; k < 20; k++) c[k] = 0.0;
    for (int i = 0; i < 10; i++)
        for (int v = 0; v < 4; v++) c[CI[i][v]] = c[CI[i][v]] + q[i] * l[v];
}

/* the linear polynomial of E[i][j] (coefficients of x, y, z, 1) */
static void elin(const double N[4][9], int i, int j, double* l)
{
    for (int b = 0; b < 4; b++) l[b] = N[b][3 * i + j];
}

static void eet(const double N[4][9], int i, int j, double* q)
{
    double a[4], b[4], t[10];
    for (int k = 0; k < 10; k++) q[k] = 0.0;
    for (int k = 0; k < 3; k++) {
        elin(N, i, k, a); elin(N, j, k, b);
        mul_ll(a, b, t);
        for (int s = 0; s < 10; s++) q[s] = q[s] + t[s];
    }
}

/* constraint e (0: det E; 1 + 3 i + j: (E E^T E - tr(E E^T) E / 2)_ij) as 20 cubic coefficients */
static void constraint(const double N[4][9], int e, double* row)
{
    double c[20], l[4];
    if (e == 0) {
        double a[4], b[4], q1[10], q2[10], t[3][10];
        static const int TI[3][8] = {{1, 1, 2, 2, 1, 2, 2, 1}, {1, 0, 2, 2, 1, 2, 2, 0}, {1, 0, 2, 1, 1, 1, 2, 0}};
        for (int s = 0; s < 3; s++) {
            elin(N, TI[s][0], TI[s][1], a); elin(N, TI[s][2], TI[s][3], b); mul_ll(a, b, q1);
            elin(N, TI[s][4], TI[s][5], a); elin(N, TI[s][6], TI[s][7], b); mul_ll(a, b, q2);
            for (int k = 0; k < 10; k++) t[s][k] = q1[k] - q2[k];
        }
        elin(N, 0, 0, l); mul_ql(t[0], l, row);
        elin(N, 0, 1, l); mul_ql(t[1], l, c);
        for (int k = 0; k < 20; k++) row[k] = row[k] - c[k];
        elin(N, 0, 2, l); mul_ql(t[2], l, c);
        for (int k = 0; k < 20; k++) row[k] = row[k] + c[k];
        return;
    }
    const int i = (e - 1) / 3, j = (e - 1) % 3;
    double q[10], tr[10], t[10];
    eet(N, 0, 0, tr);
    eet(N, 1, 1, t);
    for (int k = 0; k < 10; k++) tr[k] = tr[k] + t[k];
    eet(N, 2, 2, t);
    for (int k = 0; k < 10; k++) tr[k] = (tr[k] + t[k]) * 0.5;
    for (int k = 0; k < 20; k++) row[k] = 0.0;
    for (int s = 0; s < 3; s++) {
        eet(N, i, s, q);
        elin(N, s, j, l);
        mul_ql(q, l, c);
        for (int k = 0; k < 20; k++) row[k] = row[k] + c[k];
    }
    elin(N, i, j, l);
    mul_ql(tr, l, c);
    for (int k = 0; k < 20; k++) row[k] = row[k] - c[k];
}

static void pmul(const double* a, int na, const double* b, int nb, double* out)
{
    for (int k = 0; k < na + nb - 1; k++) out[k] = 0.0;
    for (int i = 0; i < na; i++)
        for (int j = 0; j < nb; j++) out[i + j] = out[i + j] + a[i] * b[j];
}

static double horner(const double* c, int d, double x)
{
    double s = c[d];
    for (int i = d - 1; i >= 0; i--) s = s * x + c[i];
    return s;
}

static int sgn(double v) { return (v > 0.0) - (v < 0.0); }

/* order-preserving map of doubles (not NaN) to integers, and back */
static int64_t okey(double x)
{
    int64_t b;
    memcpy(&b, &x, 8);
    return b >= 0 ? b : -(b & INT64_MAX);
}

static double ofrom(int64_t k)
{
    const int64_t b = k >= 0 ? k : ((-k) | INT64_MIN);
    double x;
    memcpy(&x, &b, 8);
    return x;
}

/* the root of the degree-d polynomial c in (lo, hi], where its sign at lo is slo and differs at hi: ESS_BISECT steps leave at most 2^16
 * ulps of the root (about 1.5e-11 of its magnitude), which the Gauss-Newton polish takes to full precision */
#define ESS_BISECT 48
static double bisect(const double* c, int d, double lo, double hi, int slo)
{
    int64_t kl = okey(lo), kh = okey(hi);
    for (int it = 0; it < ESS_BISECT; it++) {
        const uint64_t span = (uint64_t)kh - (uint64_t)kl;
        if (span <= 1) continue;
        const int64_t km = kl + (int64_t)(span >> 1);
        if (sgn(horner(c, d, ofrom(km))) == slo) kl = km; else kh = km;
    }
    return ofrom(kh);
}

/* the real roots of the polynomial p (ascending coefficients, degree <= 10), ascending; returns their number */
static int real_roots(const double* p, double* roots)
{
    int D = 10;
    while (D > 0 && p[D] == 0.0) D--;
    if (D < 1) return 0;
    double mx = 0.0;
    for (int i = 0; i < D; i++) {
        const double a = fabs(p[i]) / fabs(p[D]);
        if (a > mx) mx = a;
    }
    double R = 1.0 + mx;
    if (!(R <= DBL_MAX)) R = DBL_MAX;
    double der[11][11];
    for (int i = 0; i <= D; i++) der[D][i] = p[i];
    for (int d = D; d > 1; d--)
        for (int i = 0; i < d; i++) der[d - 1][i] = (double)(i + 1) * der[d][i + 1];
    double crit[10], cur[10];
    int ncrit = 0, ncur = 0;
    for (int d = 1; d <= D; d++) {
        ncur = 0;
        for (int k = 0; k <= ncrit; k++) {
            const double lo = k == 0 ? -R : crit[k - 1], hi = k == ncrit ? R : crit[k];
            const int slo = sgn(horner(der[d], d, lo)), shi = sgn(horner(der[d], d, hi));
            if (slo != 0 && shi != 0 && slo != shi) cur[ncur++] = bisect(der[d], d, lo, hi, slo);
            else if (slo != 0 && shi == 0) cur[ncur++] = hi;
        }
        for (int k = 0; k < ncur; k++) crit[k] = cur[k];
        ncrit = ncur;
    }
    for (int k = 0; k < ncur; k++) roots[k] = cur[k];
    return ncur;
}

/* the 20 cubic monomials at (x, y, z) (Nister's order) and their derivatives by x, y and z */
static void monomials(double x, double y, double z, double* v, double* dx, double* dy, double* dz)
{
    const double xx = x * x, yy = y * y, zz = z * z, xy = x * y, xz = x * z, yz = y * z;
    const double val[20] = {xx * x, yy * y, xx * y, x * yy, xx * z, xx, yy * z, yy, xy * z, xy, x * zz, xz, x, y * zz, yz, y, zz * z, zz, z, 1.0};
    const double ddx[20] = {3.0 * xx, 0.0, 2.0 * xy, yy, 2.0 * xz, 2.0 * x, 0.0, 0.0, yz, y, zz, z, 1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    const double ddy[20] = {0.0, 3.0 * yy, xx, 2.0 * xy, 0.0, 0.0, 2.0 * yz, 2.0 * y, xz, x, 0.0, 0.0, 0.0, zz, z, 1.0, 0.0, 0.0, 0.0, 0.0};
    const double ddz[20] = {0.0, 0.0, 0.0, 0.0, xx, 0.0, yy, 0.0, xy, 0.0, 2.0 * xz, x, 0.0, 2.0 * yz, y, 0.0, 3.0 * zz, 2.0 * z, 1.0, 0.0};
    for (int c = 0; c < 20; c++) { v[c] = val[c]; dx[c] = ddx[c]; dy[c] = ddy[c]; dz[c] = ddz[c]; }
}

/* ESS_POLISH Gauss-Newton steps on the ten constraints M0 (the coefficient matrix before elimination) from (x, y, z); 0 when the
 * normal equations are singular. The degree-10 determinant loses digits to cancellation (its roots alone leave residuals up to 1e-7 in
 * the constraints); four steps bring every solution of the 2000 configurations of tests/test_oracle_essential.py below 1e-12. */
#define ESS_POLISH 4
static int polish(const double M0[10][20], double* px, double* py, double* pz)
{
    double x = *px, y = *py, z = *pz;
    for (int it = 0; it < ESS_POLISH; it++) {
        double v[20], dx[20], dy[20], dz[20], F[10], J[10][3];
        monomials(x, y, z, v, dx, dy, dz);
        for (int e = 0; e < 10; e++) {
            double f = 0.0, a = 0.0, b = 0.0, c = 0.0;
            for (int k = 0; k < 20; k++) { f = f + M0[e][k] * v[k]; a = a + M0[e][k] * dx[k]; b = b + M0[e][k] * dy[k]; c = c + M0[e][k] * dz[k]; }
            F[e] = f; J[e][0] = a; J[e][1] = b; J[e][2] = c;
        }
        double A[3][3], g[3];
        for (int i = 0; i < 3; i++) {
            double s = 0.0;
            for (int e = 0; e < 10; e++) s = s + J[e][i] * F[e];
            g[i] = s;
            for (int j = 0; j < 3; j++) {
                double t = 0.0;
                for (int e = 0; e < 10; e++) t = t + J[e][i] * J[e][j];
                A[i][j] = t;
            }
        }
        const double c00 = A[1][1] * A[2][2] - A[1][2] * A[2][1], c01 = A[1][2] * A[2][0] - A[1][0] * A[2][2],
                     c02 = A[1][0] * A[2][1] - A[1][1] * A[2][0];
        const double det = (A[0][0] * c00 + A[0][1] * c01) + A[0][2] * c02;
        if (!(det != 0.0) || det != det) return 0;
        const double c11 = A[0][0] * A[2][2] - A[0][2] * A[2][0], c12 = A[0][1] * A[2][0] - A[0][0] * A[2][1],
                     c22 = A[0][0] * A[1][1] - A[0][1] * A[1][0];
        /* A is symmetric: its adjugate is (c00 c01 c02; c01 c11 c12; c02 c12 c22) */
        x = x - ((c00 * g[0] + c01 * g[1]) + c02 * g[2]) / det;
        y = y - ((c01 * g[0] + c11 * g[1]) + c12 * g[2]) / det;
        z = z - ((c02 * g[0] + c12 * g[1]) + c22 * g[2]) / det;
    }
    *px = x; *py = y; *pz = z;
    return 1;
}

/* the essential matrices (row-major, unit Frobenius norm) of five normalised correspondences q = (x1, y1, x2, y2); returns their number */
int orc_ess_solve5(const double* q, double* sols)
{
    /* a. Householder QR of A = Q^T (9 x 5) */
    double A[9][5], V[5][9], beta[5], N[4][9];
    for (int i = 0; i < 5; i++) {
        const double x1 = q[4 * i], y1 = q[4 * i + 1], x2 = q[4 * i + 2], y2 = q[4 * i + 3];
        const double r[9] = {x1 * x2, y1 * x2, x2, x1 * y2, y1 * y2, y2, x1, y1, 1.0};
        for (int k = 0; k < 9; k++) A[k][i] = r[k];
    }
    for (int k = 0; k < 5; k++) {
        double s = 0.0;
        for (int i = k; i < 9; i++) s = s + A[i][k] * A[i][k];
        const double nrm = sqrt(s);
        const double alpha = A[k][k] >= 0.0 ? -nrm : nrm;
        for (int i = 0; i < 9; i++) V[k][i] = i < k ? 0.0 : A[i][k];
        V[k][k] = A[k][k] - alpha;
        double vtv = 0.0;
        for (int i = k; i < 9; i++) vtv = vtv + V[k][i] * V[k][i];
        beta[k] = vtv > 0.0 ? 2.0 / vtv : 0.0;
        for (int j = k + 1; j < 5; j++) {
            double d = 0.0;
            for (int i = k; i < 9; i++) d = d + V[k][i] * A[i][j];
            const double f = beta[k] * d;
            for (int i = k; i < 9; i++) A[i][j] = A[i][j] - f * V[k][i];
        }
    }
    for (int c = 0; c < 4; c++) {
        for (int i = 0; i < 9; i++) N[c][i] = i == 5 + c ? 1.0 : 0.0;
        for (int k = 4; k >= 0; k--) {
            double d = 0.0;
            for (int i = k; i < 9; i++) d = d + V[k][i] * N[c][i];
            const double f = beta[k] * d;
            for (int i = k; i < 9; i++) N[c][i] = N[c][i] - f * V[k][i];
        }
    }
    /* b. - c. */
    double M[10][20], M0[10][20];
    for (int e = 0; e < 10; e++) constraint(N, e, M[e]);
    memcpy(M0, M, sizeof(M0));
    for (int k = 0; k < 10; k++) {
        int p = k;
        for (int r = k + 1; r < 10; r++)
            if (fabs(M[r][k]) > fabs(M[p][k])) p = r;
        if (p != k)
            for (int j = 0; j < 20; j++) { const double t = M[k][j]; M[k][j] = M[p][j]; M[p][j] = t; }
        const double piv = M[k][k];
        if (piv == 0.0 || piv != piv) return 0;
        double f[10];
        for (int r = 0; r < 10; r++) f[r] = M[r][k];
        for (int j = 0; j < 20; j++) M[k][j] = M[k][j] / piv;
        for (int r = 0; r < 10; r++)
            if (r != k)
                for (int j = 0; j < 20; j++) M[r][j] = M[r][j] - f[r] * M[k][j];
    }
    /* d. */
    double P[3][4], Qp[3][4], R[3][5];
    for (int i = 0; i < 3; i++) {
        const double* e = M[4 + 2 * i] + 10;
        const double* f = M[5 + 2 * i] + 10;
        P[i][0] = e[2]; P[i][1] = e[1] - f[2]; P[i][2] = e[0] - f[1]; P[i][3] = -f[0];
        Qp[i][0] = e[5]; Qp[i][1] = e[4] - f[5]; Qp[i][2] = e[3] - f[4]; Qp[i][3] = -f[3];
        R[i][0] = e[9]; R[i][1] = e[8] - f[9]; R[i][2] = e[7] - f[8]; R[i][3] = e[6] - f[7]; R[i][4] = -f[6];
    }
    double t1[8], t2[8], m0[8], m1[8], m2[7], d0[11], d1[11], d2[11], poly[11];
    pmul(Qp[1], 4, R[2], 5, t1); pmul(Qp[2], 4, R[1], 5, t2);
    for (int k = 0; k < 8; k++) m0[k] = t1[k] - t2[k];
    pmul(P[1], 4, R[2], 5, t1); pmul(P[2], 4, R[1], 5, t2);
    for (int k = 0; k < 8; k++) m1[k] = t1[k] - t2[k];
    pmul(P[1], 4, Qp[2], 4, t1); pmul(P[2], 4, Qp[1], 4, t2);
    for (int k = 0; k < 7; k++) m2[k] = t1[k] - t2[k];
    pmul(P[0], 4, m0, 8, d0); pmul(Qp[0], 4, m1, 8, d1); pmul(R[0], 5, m2, 7, d2);
    for (int k = 0; k < 11; k++) poly[k] = (d0[k] - d1[k]) + d2[k];
    /* e. */
    double roots[10];
    const int nr = real_roots(poly, roots);
    /* f. */
    int ns = 0;
    for (int r = 0; r < nr; r++) {
        const double z = roots[r];
        double B[3][3];
        for (int i = 0; i < 3; i++) { B[i][0] = horner(P[i], 3, z); B[i][1] = horner(Qp[i], 3, z); B[i][2] = horner(R[i], 4, z); }
        static const int PR[3][2] = {{0, 1}, {0, 2}, {1, 2}};
        double v[3] = {0.0, 0.0, 0.0}, n2 = 0.0;
        for (int s = 0; s < 3; s++) {
            const double* a = B[PR[s][0]];
            const double* b = B[PR[s][1]];
            const double c[3] = {a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]};
            const double cn = (c[0] * c[0] + c[1] * c[1]) + c[2] * c[2];
            if (s == 0 || cn > n2) { n2 = cn; v[0] = c[0]; v[1] = c[1]; v[2] = c[2]; }
        }
        if (!(n2 > 0.0)) continue;
        const double nv = sqrt(n2);
        const double u0 = v[0] / nv, u1 = v[1] / nv, u2 = v[2] / nv;
        if (!(fabs(u2) >= 1e-10)) continue;
        double x = u0 / u2, y = u1 / u2, zz = z;
        if (!polish(M0, &x, &y, &zz)) continue;
        double* E = sols + 9 * ns;
        double ss = 0.0;
        for (int k = 0; k < 9; k++) {
            E[k] = ((x * N[0][k] + y * N[1][k]) + zz * N[2][k]) + N[3][k];
            ss = ss + E[k] * E[k];
        }
        const double en = sqrt(ss);
        if (!(en > 0.0)) continue;
        for (int k = 0; k < 9; k++) E[k] = E[k] / en;
        ns++;
    }
    return ns;
}

/* the Sampson error of correspondence q under E (row-major), in double (the registrator stores it as float) */
double orc_ess_sampson(const double* E, const double* q)
{
    const double x1 = q[0], y1 = q[1], x2 = q[2], y2 = q[3];
    const double ex0 = (E[0] * x1 + E[1] * y1) + E[2];
    const double ex1 = (E[3] * x1 + E[4] * y1) + E[5];
    const double ex2 = (E[6] * x1 + E[7] * y1) + E[8];
    const double et0 = (E[0] * x2 + E[3] * y2) + E[6];
    const double et1 = (E[1] * x2 + E[4] * y2) + E[7];
    const double r = (x2 * ex0 + y2 * ex1) + ex2;
    const double a = ex0 * ex0, b = ex1 * ex1, c = et0 * et0, d = et1 * et1;
    return r * r / (((a + b) + c) + d);
}

static unsigned rng_next(uint64_t* s)
{
    *s = (uint64_t)(unsigned)*s * 4164903690u + (unsigned)(*s >> 32);
    return (unsigned)*s;
}

/* cv::RANSACUpdateNumIters(p, ep, 5, niters) for p in (0, 1), ep in [0, 1] */
int orc_ess_update_niters(double p, double ep, int niters)
{
    double num = 1.0 - p;
    if (num < DBL_MIN) num = DBL_MIN;
    double denom = 1.0 - pow(1.0 - ep, 5.0);
    if (denom < DBL_MIN) return 0;
    num = log(num);
    denom = log(denom);
    return denom >= 0.0 || -num >= niters * (-denom) ? niters : (int)nearbyint(num / denom);
}

/* the used points, normalised (x1, y1, x2, y2) and their original indices; returns m */
int orc_ess_compact(const float* xy1, const float* xy2, const uint8_t* status, int n, double fx, double fy, double cx, double cy,
                    double* q, int* idx)
{
    const double ax = 1.0 / fx, bx = -cx * ax, ay = 1.0 / fy, by = -cy * ay;
    int m = 0;
    for (int i = 0; i < n; i++) {
        if (status && !status[i]) continue;
        q[4 * m] = (double)xy1[2 * i] * ax + bx;
        q[4 * m + 1] = (double)xy1[2 * i + 1] * ay + by;
        q[4 * m + 2] = (double)xy2[2 * i] * ax + bx;
        q[4 * m + 3] = (double)xy2[2 * i + 1] * ay + by;
        if (idx) idx[m] = i;
        m++;
    }
    return m;
}

/* the draws of the first `iters` iterations: 5 distinct indices of [0, m) each */
void orc_ess_subsets(int m, int iters, int* sub)
{
    uint64_t s = ~0ull;
    for (int it = 0; it < iters; it++) {
        int* d = sub + 5 * it;
        for (int i = 0; i < 5; i++) {
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

static float ess_thr2(double threshold, double fx, double fy)
{
    const double t = threshold / ((fx + fy) / 2.0);
    return (float)(t * t);
}

static int ess_count(const double* E, const double* q, int m, float t2)
{
    int c = 0;
    for (int j = 0; j < m; j++) c += (float)orc_ess_sampson(E, q + 4 * j) <= t2;
    return c;
}

/* the whole call; E: 10 column-major 3 x 3 slots. Returns 0, or -1 when out of memory. */
int orc_find_essential(const float* xy1, const float* xy2, const uint8_t* status, int n, double fx, double fy, double cx, double cy,
                       double prob, double threshold, int max_iters, double* Eout, int* nsol, uint8_t* mask, int* inliers)
{
    double* q = (double*)malloc(sizeof(double) * 4 * (size_t)(n > 0 ? n : 1));
    int* idx = (int*)malloc(sizeof(int) * (size_t)(n > 0 ? n : 1));
    if (!q || !idx) { free(q); free(idx); return -1; }
    const int m = orc_ess_compact(xy1, xy2, status, n, fx, fy, cx, cy, q, idx);
    const float t2 = ess_thr2(threshold, fx, fy);
    double sols[ESS_MAX_SOL * 9], best[9];
    int ns = 0, good = 0;
    for (int i = 0; i < n; i++) mask[i] = 0;
    if (m == 5) {
        ns = orc_ess_solve5(q, sols);
        if (ns > 0)
            for (int j = 0; j < 5; j++) mask[idx[j]] = 1;
        good = ns > 0 ? 5 : 0;
    } else if (m > 5) {
        int niters = max_iters > 1 ? max_iters : 1;
        uint64_t s = ~0ull;
        for (int it = 0; it < niters; it++) {
            int d[5];
            for (int i = 0; i < 5; i++) {
                int v;
                for (;;) {
                    v = (int)(rng_next(&s) % (unsigned)m);
                    int dup = 0;
                    for (int k = 0; k < i; k++) dup |= d[k] == v;
                    if (!dup) break;
                }
                d[i] = v;
            }
            double sub[20];
            for (int i = 0; i < 5; i++) memcpy(sub + 4 * i, q + 4 * d[i], 4 * sizeof(double));
            const int k = orc_ess_solve5(sub, sols);
            for (int r = 0; r < k; r++) {
                const int c = ess_count(sols + 9 * r, q, m, t2);
                if (c > (good > 4 ? good : 4)) {
                    good = c;
                    memcpy(best, sols + 9 * r, sizeof(best));
                    niters = orc_ess_update_niters(prob, (double)(m - c) / m, niters);
                }
            }
        }
        if (good > 0) {
            ns = 1;
            memcpy(sols, best, sizeof(best));
            for (int j = 0; j < m; j++) mask[idx[j]] = (float)orc_ess_sampson(best, q + 4 * j) <= t2;
        }
    }
    for (int s2 = 0; s2 < ESS_MAX_SOL; s2++)
        for (int r = 0; r < 3; r++)
            for (int c = 0; c < 3; c++) Eout[9 * s2 + 3 * c + r] = s2 < ns ? sols[9 * s2 + 3 * r + c] : 0.0;
    *nsol = ns;
    *inliers = good;
    free(q); free(idx);
    return 0;
}

/* TESTS ONLY: the solutions and their errors of given subsets of the compacted points, without the acceptance loop.
 * sub: iters x 5 indices; nsols: iters; sols: iters x 10 x 9 (row-major); err: iters x 10 x m Sampson errors in double (or NULL). */
int orc_ess_hypotheses(const double* q, int m, const int* sub, int iters, int* nsols, double* sols, double* err)
{
    for (int it = 0; it < iters; it++) {
        double s5[20];
        for (int i = 0; i < 5; i++) memcpy(s5 + 4 * i, q + 4 * sub[5 * it + i], 4 * sizeof(double));
        double* S = sols + (size_t)90 * it;
        memset(S, 0, 90 * sizeof(double));
        nsols[it] = orc_ess_solve5(s5, S);
        if (err)
            for (int r = 0; r < ESS_MAX_SOL; r++)
                for (int j = 0; j < m; j++)
                    err[((size_t)it * ESS_MAX_SOL + r) * m + j] = r < nsols[it] ? orc_ess_sampson(S + 9 * r, q + 4 * j) : INFINITY;
    }
    return 0;
}
