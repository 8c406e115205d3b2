// hybvio_b200/csrc/essential.cu -- cv::findEssentialMat(xy1[used], xy2[used], K, RANSAC, prob, threshold, maxIters, mask) on the device
// (OCV/calib3d/src/five-point.cpp, ptsetreg.cpp): the five-point RANSAC between the optical flow and the filter's update.
//
// One CTA per job (one launch for one call or a batch of up to HV_ESSENTIAL_BATCH_MAX). Per job:
//   1. the used points (status != 0) are compacted in index order by a block scan, normalised as findEssentialMat's MatExpr does it
//      (x * (1 / fx) + (-cx) * (1 / fx) in double) into scratch; the mask is zeroed;
//   2. m > 5: RANSAC in waves of ESS_WARPS iterations. Thread 0 replays cv::RNG((uint64)-1)'s draws for the wave (rng.uniform(0, m),
//      a repeated index drawn again); warp w solves iteration base + w (ess_solve5 says how its lanes share the work) and scores every
//      solution over the m points (all lanes, Sampson error as float <= (float)(threshold'^2), counts reduced exactly); thread 0 then
//      runs the acceptance scan in
//      iteration order: a count above max(best, 4) wins and niters = RANSACUpdateNumIters(prob, (m - count) / m, 5, niters). The
//      loop stops once the next wave starts at or past niters, so the result does not depend on the wave size;
//   3. m == 5: every solution of the five points; m < 5: none;
//   4. E (column-major slots), nsol, inliers and the mask of the best solution (scattered to the original indices).
// The five-point solver is the oracle's (oracle/hv_oracle_essential.c, which says what it computes) operation for operation; this file
// is built with --fmad=false, so both round every product and sum alike. Only log and pow (the iteration bound) are CUDA's own;
// tests/test_oracle_essential.py shows that their error cannot move cvRound's result for any point count up to the limit.
#include "hv_common.cuh"
#include <cfloat>

#define ESS_WARPS 16                  // subsets per wave: one per warp
#define ESS_THREADS (32 * ESS_WARPS)
#define ESS_MAX_SOL 10

// quadratic monomial (xx xy xz x yy yz y zz z 1) of the product of linear variables u, v (x, y, z, 1); cubic monomial (Nister's order:
// x3 y3 x2y xy2 x2z x2 y2z y2 xyz xy | xz2 xz x yz2 yz y z3 z2 z 1) of quadratic monomial i times variable v. Compile-time tables and
// fully unrolled loops, so that every index folds and the polynomials stay in registers.
__device__ constexpr int ess_qi(int u, int v)
{
    constexpr int T[4][4] = {{0, 1, 2, 3}, {1, 4, 5, 6}, {2, 5, 7, 8}, {3, 6, 8, 9}};
    return T[u][v];
}
__device__ constexpr int ess_ci(int i, int v)
{
    constexpr int T[10][4] = {{0, 2, 4, 5}, {2, 3, 8, 9}, {4, 8, 10, 11}, {5, 9, 11, 12}, {3, 1, 6, 7},
                              {8, 6, 13, 14}, {9, 7, 14, 15}, {10, 13, 16, 17}, {11, 14, 17, 18}, {12, 15, 18, 19}};
    return T[i][v];
}

__device__ __forceinline__ void ess_mul_ll(const double* a, const double* b, double* q)
{
#pragma unroll
    for (int k = 0; k < 10; k++) q[k] = 0.0;
#pragma unroll
    for (int u = 0; u < 4; u++)
#pragma unroll
        for (int v = 0; v < 4; v++) q[ess_qi(u, v)] = q[ess_qi(u, v)] + a[u] * b[v];
}

__device__ __forceinline__ void ess_mul_ql(const double* q, const double* l, double* c)
{
#pragma unroll
    for (int k = 0; k < 20; k++) c[k] = 0.0;
#pragma unroll
    for (int i = 0; i < 10; i++)
#pragma unroll
        for (int v = 0; v < 4; v++) c[ess_ci(i, v)] = c[ess_ci(i, v)] + q[i] * l[v];
}

__device__ __forceinline__ void ess_elin(const double (*N)[9], int i, int j, double* l)
{
#pragma unroll
    for (int b = 0; b < 4; b++) l[b] = N[b][3 * i + j];
}

__device__ __forceinline__ void ess_eet(const double (*N)[9], int i, int j, double* q)
{
    double a[4], b[4], t[10];
#pragma unroll
    for (int k = 0; k < 10; k++) q[k] = 0.0;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        ess_elin(N, i, k, a); ess_elin(N, j, k, b);
        ess_mul_ll(a, b, t);
#pragma unroll
        for (int s = 0; s < 10; s++) q[s] = q[s] + t[s];
    }
}

// constraint 1 + 3 I + J, (E E^T E - tr(E E^T) E / 2)_IJ, as 20 cubic coefficients
template <int I, int J>
__device__ __forceinline__ void ess_trace_constraint(const double (*N)[9], double* row)
{
    double c[20], l[4], q[10], tr[10], t[10];
    ess_eet(N, 0, 0, tr);
    ess_eet(N, 1, 1, t);
#pragma unroll
    for (int k = 0; k < 10; k++) tr[k] = tr[k] + t[k];
    ess_eet(N, 2, 2, t);
#pragma unroll
    for (int k = 0; k < 10; k++) tr[k] = (tr[k] + t[k]) * 0.5;
    double acc[20];
#pragma unroll
    for (int k = 0; k < 20; k++) acc[k] = 0.0;
#pragma unroll
    for (int s = 0; s < 3; s++) {
        ess_eet(N, I, s, q);
        ess_elin(N, s, J, l);
        ess_mul_ql(q, l, c);
#pragma unroll
        for (int k = 0; k < 20; k++) acc[k] = acc[k] + c[k];
    }
    ess_elin(N, I, J, l);
    ess_mul_ql(tr, l, c);
#pragma unroll
    for (int k = 0; k < 20; k++) row[k] = acc[k] - c[k];
}

// constraint e (0: det E; 1 + 3 i + j: (E E^T E - tr(E E^T) E / 2)_ij) as 20 cubic coefficients (Nister's monomial order)
__device__ __noinline__ static void ess_constraint(const double (*N)[9], int e, double* row)
{
    if (e == 0) {
        constexpr int TI[3][8] = {{1, 1, 2, 2, 1, 2, 2, 1}, {1, 0, 2, 2, 1, 2, 2, 0}, {1, 0, 2, 1, 1, 1, 2, 0}};
        double a[4], b[4], q1[10], q2[10], t[3][10], c[20], l[4], acc[20];
#pragma unroll
        for (int s = 0; s < 3; s++) {
            ess_elin(N, TI[s][0], TI[s][1], a); ess_elin(N, TI[s][2], TI[s][3], b); ess_mul_ll(a, b, q1);
            ess_elin(N, TI[s][4], TI[s][5], a); ess_elin(N, TI[s][6], TI[s][7], b); ess_mul_ll(a, b, q2);
#pragma unroll
            for (int k = 0; k < 10; k++) t[s][k] = q1[k] - q2[k];
        }
        ess_elin(N, 0, 0, l); ess_mul_ql(t[0], l, acc);
        ess_elin(N, 0, 1, l); ess_mul_ql(t[1], l, c);
#pragma unroll
        for (int k = 0; k < 20; k++) acc[k] = acc[k] - c[k];
        ess_elin(N, 0, 2, l); ess_mul_ql(t[2], l, c);
#pragma unroll
        for (int k = 0; k < 20; k++) row[k] = acc[k] + c[k];
        return;
    }
    switch (e) {
    case 1: ess_trace_constraint<0, 0>(N, row); break;
    case 2: ess_trace_constraint<0, 1>(N, row); break;
    case 3: ess_trace_constraint<0, 2>(N, row); break;
    case 4: ess_trace_constraint<1, 0>(N, row); break;
    case 5: ess_trace_constraint<1, 1>(N, row); break;
    case 6: ess_trace_constraint<1, 2>(N, row); break;
    case 7: ess_trace_constraint<2, 0>(N, row); break;
    case 8: ess_trace_constraint<2, 1>(N, row); break;
    default: ess_trace_constraint<2, 2>(N, row); break;
    }
}

// double-double arithmetic (hi + lo), operation for operation as the oracle's dd_* (fma only where written out): the elimination, the
// determinant and the determinant's sign in the root brackets lose digits to cancellation in double
struct EssDD { double hi, lo; };

__device__ __forceinline__ EssDD ess_dd_fast(double s, double e)
{
    const double h = s + e;
    return EssDD{h, e - (h - s)};
}

__device__ __forceinline__ EssDD ess_dd_two_sum(double a, double b)
{
    const double s = a + b, bb = s - a;
    return EssDD{s, (a - (s - bb)) + (b - bb)};
}

__device__ __forceinline__ EssDD ess_dd_add(EssDD a, EssDD b)
{
    EssDD s = ess_dd_two_sum(a.hi, b.hi);
    const EssDD t = ess_dd_two_sum(a.lo, b.lo);
    s = ess_dd_fast(s.hi, s.lo + t.hi);
    return ess_dd_fast(s.hi, s.lo + t.lo);
}

__device__ __forceinline__ EssDD ess_dd_sub(EssDD a, EssDD b) { return ess_dd_add(a, EssDD{-b.hi, -b.lo}); }

__device__ __forceinline__ EssDD ess_dd_mul(EssDD a, EssDD b)
{
    const double p = a.hi * b.hi;
    const double e = fma(a.hi, b.hi, -p) + (a.hi * b.lo + a.lo * b.hi);
    return ess_dd_fast(p, e);
}

__device__ __forceinline__ EssDD ess_dd_mul_d(EssDD a, double x)
{
    const double p = a.hi * x;
    return ess_dd_fast(p, fma(a.hi, x, -p) + a.lo * x);
}

__device__ __forceinline__ EssDD ess_dd_div(EssDD a, EssDD b)
{
    const double q1 = a.hi / b.hi;
    const EssDD r = ess_dd_sub(a, ess_dd_mul(b, EssDD{q1, 0.0}));
    return ess_dd_fast(q1, r.hi / b.hi);
}

// coefficient k of the product of the polynomials a (na coefficients) and b (nb), summed in ascending order of a's index
__device__ static EssDD ess_dd_conv(const EssDD* a, int na, const EssDD* b, int nb, int k)
{
    EssDD s{0.0, 0.0};
    for (int i = 0; i < na; i++)
        if (k - i >= 0 && k - i < nb) s = ess_dd_add(s, ess_dd_mul(a[i], b[k - i]));
    return s;
}

__device__ static int ess_sgn(double v) { return (v > 0.0) - (v < 0.0); }

// order-preserving map of doubles (not NaN) to integers, and back
__device__ static long long ess_okey(double x)
{
    const long long b = __double_as_longlong(x);
    return b >= 0 ? b : -(b & 0x7fffffffffffffffll);
}

__device__ static double ess_ofrom(long long k)
{
    return __longlong_as_double(k >= 0 ? k : (long long)((unsigned long long)(-k) | 0x8000000000000000ull));
}

// Horner's rule for a degree-D polynomial, unrolled (D is a compile-time constant)
template <int D>
__device__ __forceinline__ double ess_horner_reg(const double* c, double x)
{
    double s = c[D];
#pragma unroll
    for (int i = D - 1; i >= 0; i--) s = s * x + c[i];
    return s;
}

// interval (lo, hi] of the degree-D polynomial g (shared memory): *root and 1 when it holds a root, else 0. The root is bracketed by
// ESS_BISECT bisection steps on the ordered bit patterns of doubles: at most 2^16 ulps of the root after 48 steps from any interval,
// about 1.5e-11 of its magnitude, which the Gauss-Newton polish (ess_polish) takes to full precision.
#define ESS_BISECT 48
template <int D>
__device__ __noinline__ int ess_interval_root(const double* g, double lo, double hi, double* root)
{
    double c[D + 1];
#pragma unroll
    for (int i = 0; i <= D; i++) c[i] = g[i];
    const int slo = ess_sgn(ess_horner_reg<D>(c, lo)), shi = ess_sgn(ess_horner_reg<D>(c, hi));
    if (slo != 0 && shi == 0) { *root = hi; return 1; }
    if (slo == 0 || shi == 0 || slo == shi) return 0;
    long long kl = ess_okey(lo), kh = ess_okey(hi);
    for (int it = 0; it < ESS_BISECT; it++) {
        const unsigned long long span = (unsigned long long)kh - (unsigned long long)kl;
        if (span <= 1) continue;
        const long long km = kl + (long long)(span >> 1);
        if (ess_sgn(ess_horner_reg<D>(c, ess_ofrom(km))) == slo) kl = km; else kh = km;
    }
    *root = ess_ofrom(kh);
    return 1;
}

// the interval (lo, hi] of the determinant itself (double-double coefficients c, degree d, shared memory), as ess_interval_root<D>
// with the sign of its value in double-double (Horner's rule, ess_dd_mul_d then ess_dd_add per coefficient)
__device__ static double ess_horner_dd(const EssDD* c, int d, double x)
{
    EssDD s = c[d];
    for (int i = d - 1; i >= 0; i--) s = ess_dd_add(ess_dd_mul_d(s, x), c[i]);
    return s.hi;
}

__device__ __noinline__ int ess_interval_root_dd(const EssDD* c, int d, double lo, double hi, double* root)
{
    const int slo = ess_sgn(ess_horner_dd(c, d, lo)), shi = ess_sgn(ess_horner_dd(c, d, hi));
    if (slo != 0 && shi == 0) { *root = hi; return 1; }
    if (slo == 0 || shi == 0 || slo == shi) return 0;
    long long kl = ess_okey(lo), kh = ess_okey(hi);
    for (int it = 0; it < ESS_BISECT; it++) {
        const unsigned long long span = (unsigned long long)kh - (unsigned long long)kl;
        if (span <= 1) continue;
        const long long km = kl + (long long)(span >> 1);
        if (ess_sgn(ess_horner_dd(c, d, ess_ofrom(km))) == slo) kl = km; else kh = km;
    }
    *root = ess_ofrom(kh);
    return 1;
}

// per-warp solver workspace (shared memory)
struct EssWarp {
    EssDD M[10][20];                  // the coefficient matrix during elimination (double-double)
    double M0[10][20];                // as formed
    double N[4][9];                   // null-space basis X, Y, Z, W
    EssDD Pd[3][4], Qd[3][4], Rd[3][5], m0[8], m1[8], m2[7];
    EssDD pdd[11];                    // the determinant
    double P[3][4], Qp[3][4], R[3][5];  // Pd, Qd, Rd rounded to double (the recovery)
    double poly[11];                  // pdd rounded to double (the derivatives)
    double der[11][11];               // der[d]: the derivative of degree d of the determinant
    double crit[10];                  // the real roots of the previous level, ascending
};

// the real roots (ascending, into w.crit) of w.poly (ascending coefficients, degree <= 10) by recursion on its derivatives; every lane
// of the warp calls it, lane k owns interval k of a level. Returns their number.
__device__ static int ess_real_roots(EssWarp& w, int lane)
{
    const double* p = w.poly;
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
    if (lane == 0) {
        for (int i = 0; i <= D; i++) w.der[D][i] = p[i];
        for (int d = D; d > 1; d--)
            for (int i = 0; i < d; i++) w.der[d - 1][i] = (double)(i + 1) * w.der[d][i + 1];
    }
    __syncwarp();
    int ncrit = 0;
    for (int d = 1; d <= D; d++) {
        double root = 0.0;
        int has = 0;
        if (lane <= ncrit) {
            const double lo = lane == 0 ? -R : w.crit[lane - 1], hi = lane == ncrit ? R : w.crit[lane];
            const double* g = w.der[d];
            if (d == D) has = ess_interval_root_dd(w.pdd, D, lo, hi, &root);
            else switch (d) {
            case 1: has = ess_interval_root<1>(g, lo, hi, &root); break;
            case 2: has = ess_interval_root<2>(g, lo, hi, &root); break;
            case 3: has = ess_interval_root<3>(g, lo, hi, &root); break;
            case 4: has = ess_interval_root<4>(g, lo, hi, &root); break;
            case 5: has = ess_interval_root<5>(g, lo, hi, &root); break;
            case 6: has = ess_interval_root<6>(g, lo, hi, &root); break;
            case 7: has = ess_interval_root<7>(g, lo, hi, &root); break;
            case 8: has = ess_interval_root<8>(g, lo, hi, &root); break;
            case 9: has = ess_interval_root<9>(g, lo, hi, &root); break;
            default: has = ess_interval_root<10>(g, lo, hi, &root); break;
            }
        }
        const unsigned bal = __ballot_sync(0xffffffffu, has);
        if (has) w.crit[__popc(bal & ((1u << lane) - 1u))] = root;
        ncrit = __popc(bal);
        __syncwarp();
    }
    return ncrit;
}

// monomial k (Nister's order) at (x, y, z) and its derivatives by x, y and z; xx ... yz are the products of two variables
__device__ __forceinline__ void ess_monomial(int k, double x, double y, double z, double xx, double yy, double zz, double xy, double xz,
                                             double yz, double& v, double& dx, double& dy, double& dz)
{
    switch (k) {
    case 0: v = xx * x; dx = 3.0 * xx; dy = 0.0; dz = 0.0; break;
    case 1: v = yy * y; dx = 0.0; dy = 3.0 * yy; dz = 0.0; break;
    case 2: v = xx * y; dx = 2.0 * xy; dy = xx; dz = 0.0; break;
    case 3: v = x * yy; dx = yy; dy = 2.0 * xy; dz = 0.0; break;
    case 4: v = xx * z; dx = 2.0 * xz; dy = 0.0; dz = xx; break;
    case 5: v = xx; dx = 2.0 * x; dy = 0.0; dz = 0.0; break;
    case 6: v = yy * z; dx = 0.0; dy = 2.0 * yz; dz = yy; break;
    case 7: v = yy; dx = 0.0; dy = 2.0 * y; dz = 0.0; break;
    case 8: v = xy * z; dx = yz; dy = xz; dz = xy; break;
    case 9: v = xy; dx = y; dy = x; dz = 0.0; break;
    case 10: v = x * zz; dx = zz; dy = 0.0; dz = 2.0 * xz; break;
    case 11: v = xz; dx = z; dy = 0.0; dz = x; break;
    case 12: v = x; dx = 1.0; dy = 0.0; dz = 0.0; break;
    case 13: v = y * zz; dx = 0.0; dy = zz; dz = 2.0 * yz; break;
    case 14: v = yz; dx = 0.0; dy = z; dz = y; break;
    case 15: v = y; dx = 0.0; dy = 1.0; dz = 0.0; break;
    case 16: v = zz * z; dx = 0.0; dy = 0.0; dz = 3.0 * zz; break;
    case 17: v = zz; dx = 0.0; dy = 0.0; dz = 2.0 * z; break;
    case 18: v = z; dx = 0.0; dy = 0.0; dz = 1.0; break;
    default: v = 1.0; dx = 0.0; dy = 0.0; dz = 0.0; break;
    }
}

// ESS_POLISH Gauss-Newton steps on the ten constraints M0 from (x, y, z); 0 when the normal equations are singular. Each of the 40
// sums runs over the monomials in ascending order, as the oracle forms them.
#define ESS_POLISH 4
__device__ __noinline__ static int ess_polish(const double (*M0)[20], double* px, double* py, double* pz)
{
    double x = *px, y = *py, z = *pz;
    for (int it = 0; it < ESS_POLISH; it++) {
        const double xx = x * x, yy = y * y, zz = z * z, xy = x * y, xz = x * z, yz = y * z;
        double F[10], J[10][3];
#pragma unroll
        for (int e = 0; e < 10; e++) { F[e] = 0.0; J[e][0] = 0.0; J[e][1] = 0.0; J[e][2] = 0.0; }
        // two passes of 20 sums each (F and dF/dx, then dF/dy and dF/dz), so that the sums stay in registers
#pragma unroll 1
        for (int k = 0; k < 20; k++) {
            double v, dx, dy, dz;
            ess_monomial(k, x, y, z, xx, yy, zz, xy, xz, yz, v, dx, dy, dz);
#pragma unroll
            for (int e = 0; e < 10; e++) { const double m = M0[e][k]; F[e] = F[e] + m * v; J[e][0] = J[e][0] + m * dx; }
        }
#pragma unroll 1
        for (int k = 0; k < 20; k++) {
            double v, dx, dy, dz;
            ess_monomial(k, x, y, z, xx, yy, zz, xy, xz, yz, v, dx, dy, dz);
#pragma unroll
            for (int e = 0; e < 10; e++) { const double m = M0[e][k]; J[e][1] = J[e][1] + m * dy; J[e][2] = J[e][2] + m * dz; }
        }
        double A[3][3], g[3];
#pragma unroll
        for (int i = 0; i < 3; i++) {
            double s = 0.0;
#pragma unroll
            for (int e = 0; e < 10; e++) s = s + J[e][i] * F[e];
            g[i] = s;
#pragma unroll
            for (int j = 0; j < 3; j++) {
                double t = 0.0;
#pragma unroll
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
        x = x - ((c00 * g[0] + c01 * g[1]) + c02 * g[2]) / det;
        y = y - ((c01 * g[0] + c11 * g[1]) + c12 * g[2]) / det;
        z = z - ((c02 * g[0] + c12 * g[1]) + c22 * g[2]) / det;
    }
    *px = x; *py = y; *pz = z;
    return 1;
}

// the essential matrix (row-major, unit Frobenius norm) of root z; 0 when the root yields none
__device__ __noinline__ static int ess_recover(const EssWarp& w, double z, double* E)
{
    double B[3][3];
    for (int i = 0; i < 3; i++) { B[i][0] = ess_horner_reg<3>(w.P[i], z); B[i][1] = ess_horner_reg<3>(w.Qp[i], z); B[i][2] = ess_horner_reg<4>(w.R[i], z); }
    const int PR[3][2] = {{0, 1}, {0, 2}, {1, 2}};
    double v[3] = {0.0, 0.0, 0.0}, n2 = 0.0;
    for (int s = 0; s < 3; s++) {
        const double* a = B[PR[s][0]];
        const double* b = B[PR[s][1]];
        const double c[3] = {a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]};
        const double cn = (c[0] * c[0] + c[1] * c[1]) + c[2] * c[2];
        if (s == 0 || cn > n2) { n2 = cn; v[0] = c[0]; v[1] = c[1]; v[2] = c[2]; }
    }
    if (!(n2 > 0.0)) return 0;
    const double nv = sqrt(n2);
    const double u0 = v[0] / nv, u1 = v[1] / nv, u2 = v[2] / nv;
    if (!(fabs(u2) >= 1e-10)) return 0;
    double x = u0 / u2, y = u1 / u2, zz = z;
    if (!ess_polish(w.M0, &x, &y, &zz)) return 0;
    double ss = 0.0;
    for (int k = 0; k < 9; k++) {
        E[k] = ((x * w.N[0][k] + y * w.N[1][k]) + zz * w.N[2][k]) + w.N[3][k];
        ss = ss + E[k] * E[k];
    }
    const double en = sqrt(ss);
    if (!(en > 0.0)) return 0;
    for (int k = 0; k < 9; k++) E[k] = E[k] / en;
    return 1;
}

// every essential matrix (row-major, unit Frobenius norm) of five normalised correspondences q = (x1, y1, x2, y2) into sols, in
// ascending order of their roots. Every lane of the warp calls it: lane 0 forms the null space, lanes 0-9 the constraints, lanes 0-19
// one column each of the elimination, lanes 0-10 the determinant, lane k the roots in interval k of each level and the matrix of root k.
// Returns their number.
__device__ static int ess_solve5(const double* q, double (*sols)[9], EssWarp& w, int lane)
{
    if (lane == 0) {
        double A[9][5], V[5][9], beta[5];
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
            double N[9];
            for (int i = 0; i < 9; i++) N[i] = i == 5 + c ? 1.0 : 0.0;
            for (int k = 4; k >= 0; k--) {
                double d = 0.0;
                for (int i = k; i < 9; i++) d = d + V[k][i] * N[i];
                const double f = beta[k] * d;
                for (int i = k; i < 9; i++) N[i] = N[i] - f * V[k][i];
            }
            for (int i = 0; i < 9; i++) w.N[c][i] = N[i];
        }
    }
    __syncwarp();
    if (lane < 10) {
        ess_constraint(w.N, lane, w.M0[lane]);
        for (int j = 0; j < 20; j++) w.M[lane][j] = EssDD{w.M0[lane][j], 0.0};
    }
    __syncwarp();
    // Gauss-Jordan with partial pivoting in double-double, lane j < 20 owning column j
    for (int k = 0; k < 10; k++) {
        int p = k;
        for (int r = k + 1; r < 10; r++)
            if (fabs(w.M[r][k].hi) > fabs(w.M[p][k].hi)) p = r;
        EssDD f[10];
        for (int r = 0; r < 10; r++) f[r] = w.M[r == k ? p : r == p ? k : r][k];
        const EssDD piv = f[k];
        __syncwarp();
        if (piv.hi == 0.0 || piv.hi != piv.hi) return 0;
        if (lane < 20) {
            const int j = lane;
            if (p != k) { const EssDD t = w.M[k][j]; w.M[k][j] = w.M[p][j]; w.M[p][j] = t; }
            w.M[k][j] = ess_dd_div(w.M[k][j], piv);
            for (int r = 0; r < 10; r++)
                if (r != k) w.M[r][j] = ess_dd_sub(w.M[r][j], ess_dd_mul(f[r], w.M[k][j]));
        }
        __syncwarp();
    }
    // the determinant in double-double: lane 0 the 3 x 3 matrix, lanes 0-7 the 2 x 2 minors' coefficients, lanes 0-10 its own
    if (lane == 0) {
        for (int i = 0; i < 3; i++) {
            const EssDD* e = w.M[4 + 2 * i] + 10;
            const EssDD* f = w.M[5 + 2 * i] + 10;
            const EssDD z{0.0, 0.0};
            w.Pd[i][0] = e[2]; w.Pd[i][1] = ess_dd_sub(e[1], f[2]); w.Pd[i][2] = ess_dd_sub(e[0], f[1]); w.Pd[i][3] = ess_dd_sub(z, f[0]);
            w.Qd[i][0] = e[5]; w.Qd[i][1] = ess_dd_sub(e[4], f[5]); w.Qd[i][2] = ess_dd_sub(e[3], f[4]); w.Qd[i][3] = ess_dd_sub(z, f[3]);
            w.Rd[i][0] = e[9]; w.Rd[i][1] = ess_dd_sub(e[8], f[9]); w.Rd[i][2] = ess_dd_sub(e[7], f[8]); w.Rd[i][3] = ess_dd_sub(e[6], f[7]);
            w.Rd[i][4] = ess_dd_sub(z, f[6]);
            for (int c = 0; c < 4; c++) { w.P[i][c] = w.Pd[i][c].hi; w.Qp[i][c] = w.Qd[i][c].hi; }
            for (int c = 0; c < 5; c++) w.R[i][c] = w.Rd[i][c].hi;
        }
    }
    __syncwarp();
    if (lane < 8) {
        const int k = lane;
        w.m0[k] = ess_dd_sub(ess_dd_conv(w.Qd[1], 4, w.Rd[2], 5, k), ess_dd_conv(w.Qd[2], 4, w.Rd[1], 5, k));
        w.m1[k] = ess_dd_sub(ess_dd_conv(w.Pd[1], 4, w.Rd[2], 5, k), ess_dd_conv(w.Pd[2], 4, w.Rd[1], 5, k));
        if (k < 7) w.m2[k] = ess_dd_sub(ess_dd_conv(w.Pd[1], 4, w.Qd[2], 4, k), ess_dd_conv(w.Pd[2], 4, w.Qd[1], 4, k));
    }
    __syncwarp();
    if (lane < 11) {
        const int k = lane;
        const EssDD v = ess_dd_add(ess_dd_sub(ess_dd_conv(w.Pd[0], 4, w.m0, 8, k), ess_dd_conv(w.Qd[0], 4, w.m1, 8, k)),
                                   ess_dd_conv(w.Rd[0], 5, w.m2, 7, k));
        w.pdd[k] = v;
        w.poly[k] = v.hi;
    }
    __syncwarp();
    const int nr = ess_real_roots(w, lane);
    double E[9];
    const int ok = lane < nr ? ess_recover(w, w.crit[lane], E) : 0;
    const unsigned bal = __ballot_sync(0xffffffffu, ok);
    if (ok) {
        double* S = sols[__popc(bal & ((1u << lane) - 1u))];
        for (int k = 0; k < 9; k++) S[k] = E[k];
    }
    __syncwarp();
    return __popc(bal);
}

__device__ __forceinline__ float ess_sampson(const double* E, const double4 p)
{
    const double x1 = p.x, y1 = p.y, x2 = p.z, y2 = p.w;
    const double ex0 = (E[0] * x1 + E[1] * y1) + E[2];
    const double ex1 = (E[3] * x1 + E[4] * y1) + E[5];
    const double ex2 = (E[6] * x1 + E[7] * y1) + E[8];
    const double et0 = (E[0] * x2 + E[3] * y2) + E[6];
    const double et1 = (E[1] * x2 + E[4] * y2) + E[7];
    const double r = (x2 * ex0 + y2 * ex1) + ex2;
    const double a = ex0 * ex0, b = ex1 * ex1, c = et0 * et0, d = et1 * et1;
    return (float)(r * r / (((a + b) + c) + d));
}

__device__ static int ess_update_niters(double p, double ep, int niters)
{
    double num = 1.0 - p;
    if (num < DBL_MIN) num = DBL_MIN;
    double denom = 1.0 - pow(1.0 - ep, 5.0);
    if (denom < DBL_MIN) return 0;
    num = log(num);
    denom = log(denom);
    return denom >= 0.0 || -num >= niters * (-denom) ? niters : __double2int_rn(num / denom);
}

__device__ __forceinline__ unsigned ess_rng_next(unsigned long long* s)
{
    *s = (unsigned long long)(unsigned)*s * 4164903690ull + (unsigned)(*s >> 32);
    return (unsigned)*s;
}

struct EssShared {
    EssWarp ws[ESS_WARPS];
    double sol[ESS_WARPS][ESS_MAX_SOL][9];
    double best[9];
    int nsol[ESS_WARPS], cnt[ESS_WARPS][ESS_MAX_SOL];
    int sub[ESS_WARPS][5];
    int warpSum[ESS_WARPS];
    unsigned long long rng;
    int m, niters, good, base;
};

__device__ static void ess_job(const EssentialArgs& a, double prob, double threshold, int maxIters, EssShared& s)
{
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n = a.n;
    // 1. compaction in index order: thread t scans [t c, (t + 1) c)
    const int chunk = (n + ESS_THREADS - 1) / ESS_THREADS;
    const int i0 = min(n, tid * chunk), i1 = min(n, i0 + chunk);
    int used = 0;
    for (int i = i0; i < i1; i++) used += a.status == nullptr || a.status[i] != 0;
    int incl = used;
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    if (lane == 31) s.warpSum[warp] = incl;
    __syncthreads();
    int off = incl - used;
    for (int w = 0; w < warp; w++) off += s.warpSum[w];
    if (tid == ESS_THREADS - 1) s.m = off + used;
    const double ax = 1.0 / a.fx, bx = -a.cx * ax, ay = 1.0 / a.fy, by = -a.cy * ay;
    for (int i = i0; i < i1; i++) {
        a.mask[i] = 0;
        if (a.status != nullptr && a.status[i] == 0) continue;
        const float2 p1 = a.xy1[i], p2 = a.xy2[i];
        reinterpret_cast<double4*>(a.q)[off] = make_double4((double)p1.x * ax + bx, (double)p1.y * ay + by, (double)p2.x * ax + bx, (double)p2.y * ay + by);
        a.idx[off] = i;
        off++;
    }
    __syncthreads();
    const int m = s.m;
    const double thr = threshold / ((a.fx + a.fy) / 2.0);
    const float t2 = (float)(thr * thr);
    int nsol = 0, good = 0;
    if (m == 5) {
        if (warp == 0) {
            double q5[20];
            for (int j = 0; j < 5; j++) { const double4 p = reinterpret_cast<double4*>(a.q)[j]; q5[4 * j] = p.x; q5[4 * j + 1] = p.y; q5[4 * j + 2] = p.z; q5[4 * j + 3] = p.w; }
            const int k = ess_solve5(q5, s.sol[0], s.ws[0], lane);
            if (lane == 0) s.nsol[0] = k;
        }
        __syncthreads();
        nsol = s.nsol[0];
        good = nsol > 0 ? 5 : 0;
        if (tid < 5 && nsol > 0) a.mask[a.idx[tid]] = 1;
    } else if (m > 5) {
        if (tid == 0) { s.niters = maxIters > 1 ? maxIters : 1; s.good = 0; s.rng = ~0ull; s.base = 0; }
        __syncthreads();
        for (;;) {
            const int base = s.base, niters = s.niters;
            if (base >= niters) break;
            if (tid == 0) {
                unsigned long long st = s.rng;
                for (int w = 0; w < ESS_WARPS && base + w < niters; w++)
                    for (int i = 0; i < 5; i++) {
                        int v;
                        for (;;) {
                            v = (int)(ess_rng_next(&st) % (unsigned)m);
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
                double q5[20];
                for (int j = 0; j < 5; j++) {
                    const double4 p = reinterpret_cast<double4*>(a.q)[s.sub[warp][j]];
                    q5[4 * j] = p.x; q5[4 * j + 1] = p.y; q5[4 * j + 2] = p.z; q5[4 * j + 3] = p.w;
                }
                const int k = ess_solve5(q5, s.sol[warp], s.ws[warp], lane);
                if (lane == 0) s.nsol[warp] = k;
                for (int r = 0; r < k; r++) {
                    const double* E = s.sol[warp][r];
                    int c = 0;
                    for (int j = lane; j < m; j += 32) c += ess_sampson(E, reinterpret_cast<double4*>(a.q)[j]) <= t2;
                    c = __reduce_add_sync(0xffffffffu, c);
                    if (lane == 0) s.cnt[warp][r] = c;
                }
            }
            __syncthreads();
            if (tid == 0) {
                int nit = niters, g = s.good;
                for (int w = 0; w < ESS_WARPS && base + w < nit; w++)
                    for (int r = 0; r < s.nsol[w]; r++) {
                        const int c = s.cnt[w][r];
                        if (c > (g > 4 ? g : 4)) {
                            g = c;
                            for (int k = 0; k < 9; k++) s.best[k] = s.sol[w][r][k];
                            nit = ess_update_niters(prob, (double)(m - c) / m, nit);
                        }
                    }
                s.good = g; s.niters = nit; s.base = base + ESS_WARPS;
            }
            __syncthreads();
        }
        good = s.good;
        nsol = good > 0 ? 1 : 0;
        if (good > 0) {
            for (int k = 0; k < 9; k++) s.sol[0][0][k] = s.best[k];
            for (int j = tid; j < m; j += ESS_THREADS) a.mask[a.idx[j]] = ess_sampson(s.best, reinterpret_cast<double4*>(a.q)[j]) <= t2;
        }
        __syncthreads();
    }
    if (tid < 9 * ESS_MAX_SOL) {
        const int sl = tid / 9, e = tid % 9, c = e / 3, r = e % 3;     // slot sl, column-major entry e = 3 c + r
        const double* S = &s.sol[0][0][0];
        a.E[tid] = sl < nsol ? S[9 * sl + 3 * r + c] : 0.0;
    }
    if (tid == 0) { *a.nsol = nsol; *a.inliers = good; }
}

__global__ void __launch_bounds__(ESS_THREADS, 1) hv_essential_kernel(const __grid_constant__ EssentialBatchArgs b)
{
    extern __shared__ __align__(16) unsigned char ess_smem[];
    ess_job(b.job[blockIdx.x], b.prob, b.threshold, b.maxIters, *reinterpret_cast<EssShared*>(ess_smem));
}

cudaError_t hv_launch_essential(const EssentialBatchArgs& b, int njobs, cudaStream_t stream)
{
    static_assert(sizeof(EssShared) <= 227 * 1024, "essential workspace exceeds the shared memory of a CTA");
    const cudaError_t e = cudaFuncSetAttribute(hv_essential_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(EssShared));
    if (e != cudaSuccess) return e;
    hv_essential_kernel<<<njobs, ESS_THREADS, sizeof(EssShared), stream>>>(b);
    return cudaGetLastError();
}
