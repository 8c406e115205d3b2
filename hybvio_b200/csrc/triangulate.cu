// hybvio_b200/csrc/triangulate.cu -- cv::triangulatePoints(P1, P2, xy1, xy2) and cv::convertPointsFromHomogeneous on the device
// (OCV/calib3d/src/triangulate.cpp, OCV/core/src/lapack.cpp, OCV/calib3d/src/fundam.cpp): the homogeneous and Euclidean 3-D points of
// two views' correspondences, for float32 points as the LK calls leave them in HBM.
//
// One thread per point; the grid is (points, jobs), so one call or a batch of up to HV_ESSENTIAL_BATCH_MAX is one launch. Per point:
//   1. the DLT rows x P[2,k] - P[0,k], y P[2,k] - P[1,k] of both views, in double from the float inputs (cvTriangulatePoints);
//   2. OpenCV's JacobiSVDImpl_ on A^T (_SVDcompute transposes a square input), restated: W the squared row norms; sweeps over the pairs
//      i < j, a pair skipped when |p| <= 10 DBL_EPSILON sqrt(W_i W_j), the rotation of OpenCV's beta < 0 / beta >= 0 branch with hypot
//      as sqrt(p^2 + beta^2), V^T rotated alongside; at most max(4, 30) sweeps, stopping after the first that changes nothing; the
//      final norms; OpenCV's selection sort (the first of equal norms kept first). Row 3 of V^T, rounded to float, is the column of X4;
//   3. xyz = the column over w in float (1 / w, then three products) where |w| > FLT_EPSILON, the column itself elsewhere.
// The oracle (oracle/hv_oracle_triangulate.c) is the same arithmetic operation for operation with only + - * / and sqrt; this file is
// built with --fmad=false, so both round every product and sum alike.
#include "hv_common.cuh"
#include <cfloat>

#define TRI_THREADS 128
#define TRI_MAX_SWEEPS 30             // max(m, 30) with m = 4

// One rotation of rows I < J of A^T (4 x 4) and V^T as JacobiSVDImpl_ does it; indices folded at compile time so that every entry
// stays in a register. Returns whether the pair rotated.
template <int I, int J>
__device__ __forceinline__ bool tri_rotate(double (&At)[4][4], double (&Vt)[4][4], double (&W)[4])
{
    double a = W[I], b = W[J], p = 0.0;
#pragma unroll
    for (int k = 0; k < 4; k++) p = p + At[I][k] * At[J][k];
    if (fabs(p) <= (10.0 * DBL_EPSILON) * sqrt(a * b)) return false;
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
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const double t0 = c * At[I][k] + s * At[J][k], t1 = -s * At[I][k] + c * At[J][k];
        At[I][k] = t0; At[J][k] = t1;
        a = a + t0 * t0; b = b + t1 * t1;
    }
    W[I] = a; W[J] = b;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const double t0 = c * Vt[I][k] + s * Vt[J][k], t1 = -s * Vt[I][k] + c * Vt[J][k];
        Vt[I][k] = t0; Vt[J][k] = t1;
    }
    return true;
}

// The sort's exchange of rows I and J of V^T and of W, predicated (a select per entry, no branch on register indices). A^T is not
// exchanged: nothing reads it after the sort (its rows become U only in the U-side of OpenCV's SVD, which Vt does not depend on).
template <int I, int J>
__device__ __forceinline__ void tri_swap(bool doSwap, double (&Vt)[4][4], double (&W)[4])
{
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const double x = Vt[I][k], y = Vt[J][k];
        Vt[I][k] = doSwap ? y : x;
        Vt[J][k] = doSwap ? x : y;
    }
    const double x = W[I], y = W[J];
    W[I] = doSwap ? y : x;
    W[J] = doSwap ? x : y;
}

// The last row of V^T of the DLT system of one correspondence (x1, y1) in P1, (x2, y2) in P2 -- cv::triangulatePoints' column
__device__ __forceinline__ void tri_point(const double* P1, const double* P2, double x1, double y1, double x2, double y2, double (&Q)[4])
{
    double At[4][4], Vt[4][4], W[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {      // A's row r is At's column r
        At[k][0] = x1 * P1[8 + k] - P1[k];
        At[k][1] = y1 * P1[8 + k] - P1[4 + k];
        At[k][2] = x2 * P2[8 + k] - P2[k];
        At[k][3] = y2 * P2[8 + k] - P2[4 + k];
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
        double sd = 0.0;
#pragma unroll
        for (int k = 0; k < 4; k++) sd = sd + At[i][k] * At[i][k];
        W[i] = sd;
#pragma unroll
        for (int k = 0; k < 4; k++) Vt[i][k] = i == k ? 1.0 : 0.0;
    }
#pragma unroll 1
    for (int it = 0; it < TRI_MAX_SWEEPS; it++) {
        bool changed = tri_rotate<0, 1>(At, Vt, W);
        changed |= tri_rotate<0, 2>(At, Vt, W);
        changed |= tri_rotate<0, 3>(At, Vt, W);
        changed |= tri_rotate<1, 2>(At, Vt, W);
        changed |= tri_rotate<1, 3>(At, Vt, W);
        changed |= tri_rotate<2, 3>(At, Vt, W);
        if (!changed) break;
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
        double sd = 0.0;
#pragma unroll
        for (int k = 0; k < 4; k++) sd = sd + At[i][k] * At[i][k];
        W[i] = sqrt(sd);
    }
    // selection sort, descending: position i takes the first largest of i..3 (selects, never an index into a register array)
    int j = 0;
    if (W[0] < W[1]) j = 1;
    if ((j == 1 ? W[1] : W[0]) < W[2]) j = 2;
    if ((j == 0 ? W[0] : (j == 1 ? W[1] : W[2])) < W[3]) j = 3;
    tri_swap<0, 1>(j == 1, Vt, W);
    tri_swap<0, 2>(j == 2, Vt, W);
    tri_swap<0, 3>(j == 3, Vt, W);
    j = 1;
    if (W[1] < W[2]) j = 2;
    if ((j == 1 ? W[1] : W[2]) < W[3]) j = 3;
    tri_swap<1, 2>(j == 2, Vt, W);
    tri_swap<1, 3>(j == 3, Vt, W);
    tri_swap<2, 3>(W[2] < W[3], Vt, W);
#pragma unroll
    for (int k = 0; k < 4; k++) Q[k] = Vt[3][k];
}

__global__ void __launch_bounds__(TRI_THREADS) hv_triangulate_kernel(const __grid_constant__ TriBatchArgs b)
{
    const TriArgs& a = b.job[blockIdx.y];
    const int i = blockIdx.x * TRI_THREADS + threadIdx.x;
    const int n = a.n;
    if (i >= n) return;
    // every read of the statuses comes before the write of used, in the same thread, so used may be either of them
    const bool use = (a.status == nullptr || a.status[i] != 0) && (a.status2 == nullptr || a.status2[i] != 0);
    float X[4] = {0.0f, 0.0f, 0.0f, 0.0f}, e[3] = {0.0f, 0.0f, 0.0f};
    if (use) {
        const float2 p1 = a.xy1[i], p2 = a.xy2[i];
        double Q[4];
        tri_point(a.P1, a.P2, (double)p1.x, (double)p1.y, (double)p2.x, (double)p2.y, Q);
#pragma unroll
        for (int k = 0; k < 4; k++) X[k] = (float)Q[k];
        const float scale = fabsf(X[3]) > FLT_EPSILON ? 1.0f / X[3] : 1.0f;
#pragma unroll
        for (int k = 0; k < 3; k++) e[k] = X[k] * scale;
    }
    if (a.X4) {
#pragma unroll
        for (int k = 0; k < 4; k++) a.X4[(size_t)k * n + i] = X[k];
    }
    if (a.xyz) {
#pragma unroll
        for (int k = 0; k < 3; k++) a.xyz[3 * (size_t)i + k] = e[k];
    }
    if (a.used) a.used[i] = use ? 1 : 0;
}

cudaError_t hv_launch_triangulate(const TriBatchArgs& b, int njobs, int maxn, cudaStream_t stream)
{
    const dim3 grid((unsigned)((maxn > 0 ? maxn : 1) + TRI_THREADS - 1) / TRI_THREADS, (unsigned)njobs);
    hv_triangulate_kernel<<<grid, TRI_THREADS, 0, stream>>>(b);
    return cudaGetLastError();
}
