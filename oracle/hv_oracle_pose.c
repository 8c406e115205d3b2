/* oracle/hv_oracle_pose.c -- TEST INFRASTRUCTURE: plain-C restatement of
 *   cv::recoverPose(E, xy1, xy2, K, R, t, distanceThresh, mask)
 * (OCV/calib3d/src/five-point.cpp, triangulate.cpp) as the device computes it (hybvio_b200/csrc/pose.cu), operation for operation:
 *   1. points in double, normalised as recoverPose's MatExpr does it: x' = x * (1 / fx) + (-cx) * (1 / fx), y' likewise with fy, cy;
 *   2. decomposeEssentialMat: E = U D V^T with U and V of determinant +1 (OpenCV negates a factor whose determinant is negative);
 *      R1 = U W V^T, R2 = U W^T V^T, t = U[:, 2], W = [[0, 1, 0], [-1, 0, 0], [0, 0, 1]];
 *   3. candidates (R1, t), (R2, t), (R1, -t), (R2, -t); per candidate P = [R | t'] and point, the DLT triangulation against
 *      P0 = [I | 0]: Q is the right singular vector, for the smallest singular value, of the 4 x 4 matrix with rows
 *      x1 P0[2,:] - P0[0,:], y1 P0[2,:] - P0[1,:], x2 P[2,:] - P[0,:], y2 P[2,:] - P[1,:];
 *   4. the point is good for the candidate iff Q2 Q3 > 0, Q2 / Q3 < dist, z > 0 and z < dist, where
 *      z = ((P20 X + P21 Y) + P22 Z) + P23 W with (X, Y, Z, W) = Q / Q3; and the input mask (if any) is non-zero;
 *   5. the counts pick the candidate in OpenCV's order (good1 >= all, else good2 >= all, else good3 >= all, else the fourth).
 * OpenCV's SVD iterates until it converges and is not restated. Both SVDs here are one-sided (Hestenes) Jacobi with a fixed number of
 * cyclic sweeps, so the work does not depend on the data:
 *   - 3 x 3 (E): POSE_SWEEPS3 sweeps over the column pairs (0,1), (0,2), (1,2); columns sorted by norm, descending, by a three-compare
 *     network that swaps on a strict <; u1, u2 the first two columns over their norms (e1, and then the unit axis least aligned with u1
 *     orthogonalised against it, where a norm is 0), u3 = u1 x u2, so det U = +1; V negated when the sort swapped an odd number of times;
 *   - 4 x 4 (DLT): POSE_SWEEPS4 sweeps over (0,1), (0,2), (0,3), (1,2), (1,3), (2,3); Q is the column of V whose column of A has the
 *     smallest squared norm (the first such).
 *   A rotation of columns p < q: a = |A_p|^2, b = |A_q|^2, g = A_p . A_q (sums in row order); none when g == 0; zeta = (b - a) / (2 g),
 *   t = 1 / (|zeta| + sqrt(1 + zeta^2)) with zeta's sign, c = 1 / sqrt(1 + t^2), s = c t; A_p <- c A_p - s A_q, A_q <- s A_p + c A_q,
 *   the same for V.
 * Any SVD of E gives the same four candidates (only their order changes with its sign conventions), so the result is OpenCV's wherever
 * one candidate wins alone. Built with -ffp-contract=off, so no multiply-add is contracted; the kernel is built with --fmad=false.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define POSE_SWEEPS3 8
#define POSE_SWEEPS4 6

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

static void swap_cols3(double* A, double* V, double* nrm, int p, int q)
{
    for (int r = 0; r < 3; r++) {
        double x = A[3 * r + p]; A[3 * r + p] = A[3 * r + q]; A[3 * r + q] = x;
        x = V[3 * r + p]; V[3 * r + p] = V[3 * r + q]; V[3 * r + q] = x;
    }
    const double x = nrm[p]; nrm[p] = nrm[q]; nrm[q] = x;
}

/* decomposeEssentialMat of E (column-major, 9 doubles): R1, R2 row-major, t */
void orc_pose_decompose(const double* Ecm, double* R1, double* R2, double* t)
{
    double A[9], V[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, nrm[3], u[3][3];
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) A[3 * r + c] = Ecm[3 * c + r];
    for (int s = 0; s < POSE_SWEEPS3; s++) {
        jacobi_rotate(A, V, 3, 3, 0, 1);
        jacobi_rotate(A, V, 3, 3, 0, 2);
        jacobi_rotate(A, V, 3, 3, 1, 2);
    }
    for (int c = 0; c < 3; c++) nrm[c] = sqrt((A[c] * A[c] + A[3 + c] * A[3 + c]) + A[6 + c] * A[6 + c]);
    int swaps = 0;
    if (nrm[0] < nrm[1]) { swap_cols3(A, V, nrm, 0, 1); swaps++; }
    if (nrm[1] < nrm[2]) { swap_cols3(A, V, nrm, 1, 2); swaps++; }
    if (nrm[0] < nrm[1]) { swap_cols3(A, V, nrm, 0, 1); swaps++; }
    for (int c = 0; c < 2; c++)
        for (int r = 0; r < 3; r++) u[c][r] = A[3 * r + c] / nrm[c];
    if (!(nrm[0] > 0.0)) { u[0][0] = 1.0; u[0][1] = 0.0; u[0][2] = 0.0; }
    if (!(nrm[1] > 0.0)) {
        int k = 0;
        for (int r = 1; r < 3; r++)
            if (fabs(u[0][r]) < fabs(u[0][k])) k = r;
        for (int r = 0; r < 3; r++) u[1][r] = -u[0][k] * u[0][r];
        u[1][k] = u[1][k] + 1.0;
        const double l = sqrt((u[1][0] * u[1][0] + u[1][1] * u[1][1]) + u[1][2] * u[1][2]);
        for (int r = 0; r < 3; r++) u[1][r] = u[1][r] / l;
    }
    u[2][0] = u[0][1] * u[1][2] - u[0][2] * u[1][1];
    u[2][1] = u[0][2] * u[1][0] - u[0][0] * u[1][2];
    u[2][2] = u[0][0] * u[1][1] - u[0][1] * u[1][0];
    if (swaps & 1)
        for (int k = 0; k < 9; k++) V[k] = -V[k];
    /* R1 = U W V^T = -u2 v1^T + u1 v2^T + u3 v3^T, R2 = U W^T V^T = u2 v1^T - u1 v2^T + u3 v3^T */
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            const double a = u[1][i] * V[3 * j], b = u[0][i] * V[3 * j + 1], c = u[2][i] * V[3 * j + 2];
            R1[3 * i + j] = (b - a) + c;
            R2[3 * i + j] = (a - b) + c;
        }
    for (int i = 0; i < 3; i++) t[i] = u[2][i];
}

/* the four decisions' conjunction for one point and candidate P (3 x 4 row-major); Qout (4) the null vector if not NULL */
static int pose_good(const double* P, double x1, double y1, double x2, double y2, double dist, double* Qout)
{
    double A[16] = {-1.0, 0.0, x1, 0.0, 0.0, -1.0, y1, 0.0}, V[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    for (int k = 0; k < 4; k++) {
        A[8 + k] = x2 * P[8 + k] - P[k];
        A[12 + k] = y2 * P[8 + k] - P[4 + k];
    }
    for (int s = 0; s < POSE_SWEEPS4; s++)
        for (int p = 0; p < 3; p++)
            for (int q = p + 1; q < 4; q++) jacobi_rotate(A, V, 4, 4, p, q);
    int jm = 0;
    double nm = 0.0;
    for (int j = 0; j < 4; j++) {
        const double v = ((A[j] * A[j] + A[4 + j] * A[4 + j]) + A[8 + j] * A[8 + j]) + A[12 + j] * A[12 + j];
        if (j == 0 || v < nm) { nm = v; jm = j; }
    }
    const double Q0 = V[jm], Q1 = V[4 + jm], Q2 = V[8 + jm], Q3 = V[12 + jm];
    if (Qout) { Qout[0] = Q0; Qout[1] = Q1; Qout[2] = Q2; Qout[3] = Q3; }
    const double X = Q0 / Q3, Y = Q1 / Q3, Z = Q2 / Q3, W = Q3 / Q3;
    const double z = ((P[8] * X + P[9] * Y) + P[10] * Z) + P[11] * W;
    return (Q2 * Q3 > 0.0) & (Z < dist) & (z > 0.0) & (z < dist);
}

/* the whole call. E column-major, nsol its count (0: none, > 1: the first is used). R column-major, t, mask_out 0/1 (may be mask_in),
 * good. flags (n x 4, the candidates' decisions before the input mask) and Q (n x 4 x 4, the null vectors) may be NULL. */
int orc_recover_pose_ex(const double* E, int nsol, const float* xy1, const float* xy2, const uint8_t* mask_in, int n, double fx, double fy,
                        double cx, double cy, double dist, double* R, double* t, uint8_t* mask_out, int* good, uint8_t* flags, double* Q)
{
    if (nsol == 0) {
        memset(R, 0, 9 * sizeof(double));
        memset(t, 0, 3 * sizeof(double));
        for (int i = 0; i < n; i++) mask_out[i] = 0;
        *good = 0;
        return 0;
    }
    double R1[9], R2[9], tt[3], P[4][12];
    orc_pose_decompose(E, R1, R2, tt);
    for (int k = 0; k < 4; k++)
        for (int r = 0; r < 3; r++) {
            const double* Rk = (k & 1) ? R2 : R1;
            for (int c = 0; c < 3; c++) P[k][4 * r + c] = Rk[3 * r + c];
            P[k][4 * r + 3] = (k & 2) ? -tt[r] : tt[r];
        }
    const double ax = 1.0 / fx, bx = -cx * ax, ay = 1.0 / fy, by = -cy * ay;
    int cnt[4] = {0, 0, 0, 0};
    uint8_t* f = flags ? flags : (uint8_t*)malloc(4 * (size_t)(n > 0 ? n : 1));
    if (!f) return -1;
    for (int i = 0; i < n; i++) {
        const double x1 = (double)xy1[2 * i] * ax + bx, y1 = (double)xy1[2 * i + 1] * ay + by;
        const double x2 = (double)xy2[2 * i] * ax + bx, y2 = (double)xy2[2 * i + 1] * ay + by;
        const int use = mask_in == NULL || mask_in[i] != 0;
        for (int k = 0; k < 4; k++) {
            const int g = pose_good(P[k], x1, y1, x2, y2, dist, Q ? Q + 16 * (size_t)i + 4 * k : NULL);
            f[4 * (size_t)i + k] = (uint8_t)g;
            cnt[k] += g & use;
        }
    }
    int w;
    if (cnt[0] >= cnt[1] && cnt[0] >= cnt[2] && cnt[0] >= cnt[3]) w = 0;
    else if (cnt[1] >= cnt[0] && cnt[1] >= cnt[2] && cnt[1] >= cnt[3]) w = 1;
    else if (cnt[2] >= cnt[0] && cnt[2] >= cnt[1] && cnt[2] >= cnt[3]) w = 2;
    else w = 3;
    for (int i = 0; i < n; i++) mask_out[i] = f[4 * (size_t)i + w] & (mask_in == NULL || mask_in[i] != 0);
    if (!flags) free(f);
    for (int r = 0; r < 3; r++) {
        for (int c = 0; c < 3; c++) R[3 * c + r] = P[w][4 * r + c];
        t[r] = P[w][4 * r + 3];
    }
    *good = cnt[w];
    return 0;
}

int orc_recover_pose(const double* E, int nsol, const float* xy1, const float* xy2, const uint8_t* mask_in, int n, double fx, double fy,
                     double cx, double cy, double dist, double* R, double* t, uint8_t* mask_out, int* good)
{
    return orc_recover_pose_ex(E, nsol, xy1, xy2, mask_in, n, fx, fy, cx, cy, dist, R, t, mask_out, good, NULL, NULL);
}
