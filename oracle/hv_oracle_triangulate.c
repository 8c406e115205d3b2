/* oracle/hv_oracle_triangulate.c -- TEST INFRASTRUCTURE: plain-C restatement of
 *   cv::triangulatePoints(P1, P2, xy1, xy2, X4) and cv::convertPointsFromHomogeneous(X4^T, xyz)
 * (OCV/calib3d/src/triangulate.cpp, OCV/core/src/lapack.cpp, OCV/calib3d/src/fundam.cpp) for float32 points, as the device computes it
 * (hybvio_b200/csrc/triangulate.cu), operation for operation:
 *   1. per point, in double from the float inputs, the 4 x 4 DLT matrix A with rows
 *      x1 P1[2,:] - P1[0,:], y1 P1[2,:] - P1[1,:], x2 P2[2,:] - P2[0,:], y2 P2[2,:] - P2[1,:]   (cvTriangulatePoints);
 *   2. OpenCV's JacobiSVDImpl_ on A^T (what _SVDcompute hands it for a square matrix), m = n = 4:
 *      W_i = |row i|^2 (sums in index order), V^T = I; up to max(m, 30) sweeps over the pairs (i, j), i < j, in order: p = row i . row j;
 *      the pair is skipped when |p| <= 10 DBL_EPSILON sqrt(W_i W_j); else p = 2 p, beta = W_i - W_j, gamma = sqrt(p^2 + beta^2) (hypot
 *      restated), beta < 0: s = sqrt(((gamma - beta) 0.5) / gamma), c = p / (gamma s 2); beta >= 0: c = sqrt((gamma + beta) / (gamma 2)),
 *      s = p / (gamma c 2); rows i, j <- c row_i + s row_j, -s row_i + c row_j, W_i, W_j their new squared norms; V^T's rows alike; the
 *      sweeps stop after the first that rotates no pair; W_i = sqrt(|row i|^2); selection sort by W, descending, a later row taken only
 *      when strictly larger, exchanging V^T's rows (A^T's exchanged rows are never read again and are left out);
 *   3. X4's column = row 3 of V^T rounded to float;
 *   4. xyz = (X, Y, Z) * scale in float, scale = 1 / w (float) where |w| > FLT_EPSILON, 1 elsewhere.
 * A point is used when status and status2 (NULL: all non-zero) are both non-zero there; an unused point gives a zero column, zero xyz,
 * used 0. Built with -ffp-contract=off, so no multiply-add is contracted; the kernel is built with --fmad=false.
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#define TRI_MAX_SWEEPS 30

/* the SVD state after the sweeps, for the tests that need it: V^T (row-major) and W before the sort */
static void tri_svd(const double* P1, const double* P2, double x1, double y1, double x2, double y2, double At[4][4], double Vt[4][4],
                    double W[4], int sort, int* sweeps)
{
    int i, j, k, it;
    for (k = 0; k < 4; k++) {
        At[k][0] = x1 * P1[8 + k] - P1[k];
        At[k][1] = y1 * P1[8 + k] - P1[4 + k];
        At[k][2] = x2 * P2[8 + k] - P2[k];
        At[k][3] = y2 * P2[8 + k] - P2[4 + k];
    }
    for (i = 0; i < 4; i++) {
        double sd = 0.0;
        for (k = 0; k < 4; k++) sd = sd + At[i][k] * At[i][k];
        W[i] = sd;
        for (k = 0; k < 4; k++) Vt[i][k] = i == k ? 1.0 : 0.0;
    }
    for (it = 0; it < TRI_MAX_SWEEPS; it++) {
        int changed = 0;
        for (i = 0; i < 3; i++)
            for (j = i + 1; j < 4; j++) {
                double a = W[i], b = W[j], p = 0.0, beta, gamma, c, s;
                for (k = 0; k < 4; k++) p = p + At[i][k] * At[j][k];
                if (fabs(p) <= (10.0 * DBL_EPSILON) * sqrt(a * b)) continue;
                p = p * 2.0;
                beta = a - b;
                gamma = sqrt(p * p + beta * beta);
                if (beta < 0.0) {
                    const double delta = (gamma - beta) * 0.5;
                    s = sqrt(delta / gamma);
                    c = p / (gamma * s * 2.0);
                } else {
                    c = sqrt((gamma + beta) / (gamma * 2.0));
                    s = p / (gamma * c * 2.0);
                }
                a = 0.0; b = 0.0;
                for (k = 0; k < 4; k++) {
                    const double t0 = c * At[i][k] + s * At[j][k], t1 = -s * At[i][k] + c * At[j][k];
                    At[i][k] = t0; At[j][k] = t1;
                    a = a + t0 * t0; b = b + t1 * t1;
                }
                W[i] = a; W[j] = b;
                for (k = 0; k < 4; k++) {
                    const double t0 = c * Vt[i][k] + s * Vt[j][k], t1 = -s * Vt[i][k] + c * Vt[j][k];
                    Vt[i][k] = t0; Vt[j][k] = t1;
                }
                changed = 1;
            }
        if (!changed) break;
    }
    if (sweeps) *sweeps = it;
    for (i = 0; i < 4; i++) {
        double sd = 0.0;
        for (k = 0; k < 4; k++) sd = sd + At[i][k] * At[i][k];
        W[i] = sqrt(sd);
    }
    if (!sort) return;
    for (i = 0; i < 3; i++) {
        j = i;
        for (k = i + 1; k < 4; k++)
            if (W[j] < W[k]) j = k;
        if (i != j) {
            double t = W[i]; W[i] = W[j]; W[j] = t;
            for (k = 0; k < 4; k++) { t = Vt[i][k]; Vt[i][k] = Vt[j][k]; Vt[j][k] = t; }
        }
    }
}

/* The whole call: X4 (4 x n, row r at X4 + r n), xyz (n x 3), used (n) -- each may be NULL. sort = 0 leaves the selection sort out
 * (the tests show that without it the result is not OpenCV's). */
void orc_triangulate_points_ex(const double* P1, const double* P2, const float* xy1, const float* xy2, const uint8_t* status,
                               const uint8_t* status2, int n, float* X4, float* xyz, uint8_t* used, int sort)
{
    int i, k;
    for (i = 0; i < n; i++) {
        const int use = (!status || status[i] != 0) && (!status2 || status2[i] != 0);
        float X[4] = {0.0f, 0.0f, 0.0f, 0.0f}, e[3] = {0.0f, 0.0f, 0.0f};
        if (use) {
            double At[4][4], Vt[4][4], W[4];
            float scale;
            tri_svd(P1, P2, (double)xy1[2 * i], (double)xy1[2 * i + 1], (double)xy2[2 * i], (double)xy2[2 * i + 1], At, Vt, W, sort, 0);
            for (k = 0; k < 4; k++) X[k] = (float)Vt[3][k];
            scale = fabsf(X[3]) > FLT_EPSILON ? 1.0f / X[3] : 1.0f;
            for (k = 0; k < 3; k++) e[k] = X[k] * scale;
        }
        if (X4)
            for (k = 0; k < 4; k++) X4[(size_t)k * n + i] = X[k];
        if (xyz)
            for (k = 0; k < 3; k++) xyz[3 * (size_t)i + k] = e[k];
        if (used) used[i] = (uint8_t)use;
    }
}

void orc_triangulate_points(const double* P1, const double* P2, const float* xy1, const float* xy2, const uint8_t* status,
                            const uint8_t* status2, int n, float* X4, float* xyz, uint8_t* used)
{
    orc_triangulate_points_ex(P1, P2, xy1, xy2, status, status2, n, X4, xyz, used, 1);
}

/* One point's double-precision null vector (row 3 of V^T before rounding) and the number of sweeps it took. */
void orc_triangulate_one(const double* P1, const double* P2, const float* x1, const float* x2, double* Q, int* sweeps)
{
    double At[4][4], Vt[4][4], W[4];
    int k;
    tri_svd(P1, P2, (double)x1[0], (double)x1[1], (double)x2[0], (double)x2[1], At, Vt, W, 1, sweeps);
    for (k = 0; k < 4; k++) Q[k] = Vt[3][k];
}
