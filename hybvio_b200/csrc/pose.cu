// hybvio_b200/csrc/pose.cu -- cv::recoverPose(E, xy1, xy2, K, R, t, distanceThresh, mask) on the device (OCV/calib3d/src/five-point.cpp,
// triangulate.cpp): the relative rotation, the translation direction and the points in front of both cameras, from the essential
// matrix that hv_find_essential* leaves in HBM.
//
// One CTA per job (one launch for one call or a batch of up to HV_ESSENTIAL_BATCH_MAX). Per job:
//   1. thread 0 reads the solution count (nsol NULL: one matrix; 0: no result) and decomposes the first E (decomposeEssentialMat) with
//      a one-sided Jacobi SVD of POSE_SWEEPS3 sweeps into the four candidates [R1 | t], [R2 | t], [R1 | -t], [R2 | -t];
//   2. work item k = 4 i + c is point i under candidate c (POSE_THREADS is a multiple of 4, so a thread keeps one candidate): the
//      point normalised as recoverPose's MatExpr does it, the 4 x 4 DLT system against [I | 0], its smallest right singular vector
//      from a one-sided Jacobi SVD of POSE_SWEEPS4 sweeps, the four depth tests; the decision goes to a byte in shared memory;
//   3. the candidates' counts (decisions AND the input mask) are reduced exactly, the winner picked in OpenCV's order, and its R, t,
//      count and mask (0/1, at the original indices) written.
// The arithmetic is the oracle's (oracle/hv_oracle_pose.c, which says what it computes) operation for operation, with only + - * /
// and sqrt; this file is built with --fmad=false, so both round every product and sum alike.
#include "hv_common.cuh"

#define POSE_THREADS 512
#define POSE_WARPS (POSE_THREADS / 32)
#define POSE_SWEEPS3 8                // 3 x 3 (E): converged to rounding after 3 on the test scenes
#define POSE_SWEEPS4 6                // 4 x 4 (DLT): converged to rounding after 5 on the test scenes
static_assert(POSE_THREADS % 4 == 0, "a thread keeps one candidate");

// one Jacobi rotation of columns P < Q of A (ROWS x N) and V (N x N), indices folded at compile time so that both stay in registers
template <int P, int Q, int ROWS, int N>
__device__ __forceinline__ void pose_rotate(double (&A)[ROWS][N], double (&V)[N][N])
{
    double a = 0.0, b = 0.0, g = 0.0;
#pragma unroll
    for (int r = 0; r < ROWS; r++) {
        const double x = A[r][P], y = A[r][Q];
        a = a + x * x;
        b = b + y * y;
        g = g + x * y;
    }
    if (g == 0.0) return;
    const double zeta = (b - a) / (2.0 * g);
    double t = 1.0 / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
    if (zeta < 0.0) t = -t;
    const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
#pragma unroll
    for (int r = 0; r < ROWS; r++) {
        const double x = A[r][P], y = A[r][Q];
        A[r][P] = c * x - s * y;
        A[r][Q] = s * x + c * y;
    }
#pragma unroll
    for (int r = 0; r < N; r++) {
        const double x = V[r][P], y = V[r][Q];
        V[r][P] = c * x - s * y;
        V[r][Q] = s * x + c * y;
    }
}

template <int P, int Q>
__device__ __forceinline__ void pose_swap3(bool doSwap, double (&A)[3][3], double (&V)[3][3], double* nrm)
{
    if (!doSwap) return;
#pragma unroll
    for (int r = 0; r < 3; r++) {
        double x = A[r][P]; A[r][P] = A[r][Q]; A[r][Q] = x;
        x = V[r][P]; V[r][P] = V[r][Q]; V[r][Q] = x;
    }
    const double x = nrm[P]; nrm[P] = nrm[Q]; nrm[Q] = x;
}

// decomposeEssentialMat of E (column-major) into the four candidates P[k] = [R | t'] (3 x 4 row-major)
__device__ __noinline__ static void pose_decompose(const double* E, double (*P)[12])
{
    double A[3][3], V[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}}, nrm[3], u0[3], u1[3], u2[3];
#pragma unroll
    for (int r = 0; r < 3; r++)
#pragma unroll
        for (int c = 0; c < 3; c++) A[r][c] = E[3 * c + r];
#pragma unroll 1
    for (int s = 0; s < POSE_SWEEPS3; s++) {
        pose_rotate<0, 1>(A, V);
        pose_rotate<0, 2>(A, V);
        pose_rotate<1, 2>(A, V);
    }
#pragma unroll
    for (int c = 0; c < 3; c++) nrm[c] = sqrt((A[0][c] * A[0][c] + A[1][c] * A[1][c]) + A[2][c] * A[2][c]);
    int swaps = 0;
    bool sw = nrm[0] < nrm[1]; pose_swap3<0, 1>(sw, A, V, nrm); swaps += sw;
    sw = nrm[1] < nrm[2]; pose_swap3<1, 2>(sw, A, V, nrm); swaps += sw;
    sw = nrm[0] < nrm[1]; pose_swap3<0, 1>(sw, A, V, nrm); swaps += sw;
#pragma unroll
    for (int r = 0; r < 3; r++) { u0[r] = A[r][0] / nrm[0]; u1[r] = A[r][1] / nrm[1]; }
    if (!(nrm[0] > 0.0)) { u0[0] = 1.0; u0[1] = 0.0; u0[2] = 0.0; }
    if (!(nrm[1] > 0.0)) {          // rank 1 or 0: the unit axis least aligned with u0, orthogonalised against it
        int k = 0;
        if (fabs(u0[1]) < fabs(u0[k])) k = 1;
        if (fabs(u0[2]) < fabs(u0[k == 1 ? 1 : 0])) k = 2;
        const double uk = k == 0 ? u0[0] : (k == 1 ? u0[1] : u0[2]);
#pragma unroll
        for (int r = 0; r < 3; r++) {
            u1[r] = -uk * u0[r];
            if (r == k) u1[r] = u1[r] + 1.0;
        }
        const double l = sqrt((u1[0] * u1[0] + u1[1] * u1[1]) + u1[2] * u1[2]);
#pragma unroll
        for (int r = 0; r < 3; r++) u1[r] = u1[r] / l;
    }
    u2[0] = u0[1] * u1[2] - u0[2] * u1[1];
    u2[1] = u0[2] * u1[0] - u0[0] * u1[2];
    u2[2] = u0[0] * u1[1] - u0[1] * u1[0];
    if (swaps & 1)
#pragma unroll
        for (int r = 0; r < 3; r++)
#pragma unroll
            for (int c = 0; c < 3; c++) V[r][c] = -V[r][c];
    // R1 = U W V^T = -u1 v0^T + u0 v1^T + u2 v2^T, R2 = U W^T V^T = u1 v0^T - u0 v1^T + u2 v2^T
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) {
            const double a = u1[i] * V[j][0], b = u0[i] * V[j][1], c = u2[i] * V[j][2];
            const double r1 = (b - a) + c, r2 = (a - b) + c;
            P[0][4 * i + j] = r1; P[2][4 * i + j] = r1;
            P[1][4 * i + j] = r2; P[3][4 * i + j] = r2;
        }
#pragma unroll
    for (int i = 0; i < 3; i++) {
        P[0][4 * i + 3] = u2[i]; P[1][4 * i + 3] = u2[i];
        P[2][4 * i + 3] = -u2[i]; P[3][4 * i + 3] = -u2[i];
    }
}

// triangulatePoints of one normalised correspondence against [I | 0] and P, and recoverPose's four depth tests
__device__ __forceinline__ int pose_good(const double* P, double x1, double y1, double x2, double y2, double dist)
{
    double A[4][4], V[4][4] = {{1, 0, 0, 0}, {0, 1, 0, 0}, {0, 0, 1, 0}, {0, 0, 0, 1}};
    A[0][0] = -1.0; A[0][1] = 0.0; A[0][2] = x1; A[0][3] = 0.0;
    A[1][0] = 0.0; A[1][1] = -1.0; A[1][2] = y1; A[1][3] = 0.0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        A[2][k] = x2 * P[8 + k] - P[k];
        A[3][k] = y2 * P[8 + k] - P[4 + k];
    }
#pragma unroll 1
    for (int s = 0; s < POSE_SWEEPS4; s++) {
        pose_rotate<0, 1>(A, V);
        pose_rotate<0, 2>(A, V);
        pose_rotate<0, 3>(A, V);
        pose_rotate<1, 2>(A, V);
        pose_rotate<1, 3>(A, V);
        pose_rotate<2, 3>(A, V);
    }
    double nm = 0.0, Q0 = 0.0, Q1 = 0.0, Q2 = 0.0, Q3 = 0.0;
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const double v = ((A[0][j] * A[0][j] + A[1][j] * A[1][j]) + A[2][j] * A[2][j]) + A[3][j] * A[3][j];
        if (j == 0 || v < nm) { nm = v; Q0 = V[0][j]; Q1 = V[1][j]; Q2 = V[2][j]; Q3 = V[3][j]; }
    }
    const double X = Q0 / Q3, Y = Q1 / Q3, Z = Q2 / Q3, W = Q3 / Q3;
    const double z = ((P[8] * X + P[9] * Y) + P[10] * Z) + P[11] * W;
    return (Q2 * Q3 > 0.0) & (Z < dist) & (z > 0.0) & (z < dist);
}

struct PoseShared {
    double P[4][12];
    int cnt[POSE_WARPS][4];
    int nsol, win;
    uint8_t flags[4 * HV_ESSENTIAL_MAX_POINTS];     // the decision of point i under candidate c at 4 i + c
};

__device__ static void pose_job(const PoseArgs& a, double dist, PoseShared& s)
{
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n = a.n;
    if (tid == 0) {
        s.nsol = a.nsol ? *a.nsol : 1;
        if (s.nsol != 0) pose_decompose(a.E, s.P);
    }
    __syncthreads();
    if (s.nsol == 0) {
        for (int i = tid; i < n; i += POSE_THREADS) a.maskOut[i] = 0;
        if (tid < 9) a.R[tid] = 0.0;
        if (tid < 3) a.t[tid] = 0.0;
        if (tid == 0) *a.good = 0;
        return;
    }
    const double ax = 1.0 / a.fx, bx = -a.cx * ax, ay = 1.0 / a.fy, by = -a.cy * ay;
    const int cand = tid & 3;
    int cnt = 0;
    for (int k = tid; k < 4 * n; k += POSE_THREADS) {
        const int i = k >> 2;
        const float2 p1 = a.xy1[i], p2 = a.xy2[i];
        const int g = pose_good(s.P[cand], (double)p1.x * ax + bx, (double)p1.y * ay + by, (double)p2.x * ax + bx, (double)p2.y * ay + by, dist);
        s.flags[k] = (uint8_t)g;
        cnt += g & (a.maskIn == nullptr || a.maskIn[i] != 0);
    }
#pragma unroll
    for (int c = 0; c < 4; c++) {
        const int v = __reduce_add_sync(0xffffffffu, cand == c ? cnt : 0);
        if (lane == 0) s.cnt[warp][c] = v;
    }
    __syncthreads();
    if (tid == 0) {
        int g[4] = {0, 0, 0, 0};
        for (int w = 0; w < POSE_WARPS; w++)
#pragma unroll
            for (int c = 0; c < 4; c++) g[c] += s.cnt[w][c];
        int w;
        if (g[0] >= g[1] && g[0] >= g[2] && g[0] >= g[3]) w = 0;
        else if (g[1] >= g[0] && g[1] >= g[2] && g[1] >= g[3]) w = 1;
        else if (g[2] >= g[0] && g[2] >= g[1] && g[2] >= g[3]) w = 2;
        else w = 3;
        s.win = w;
        *a.good = w == 0 ? g[0] : (w == 1 ? g[1] : (w == 2 ? g[2] : g[3]));
    }
    __syncthreads();
    const int w = s.win;
    // every read of maskIn is behind the barrier, so maskOut may be maskIn
    for (int i = tid; i < n; i += POSE_THREADS) a.maskOut[i] = s.flags[4 * i + w] & (a.maskIn == nullptr || a.maskIn[i] != 0);
    if (tid < 9) a.R[tid] = s.P[w][4 * (tid % 3) + tid / 3];       // column-major: R[3 c + r] = P[r][c]
    else if (tid < 12) a.t[tid - 9] = s.P[w][4 * (tid - 9) + 3];
}

__global__ void __launch_bounds__(POSE_THREADS, 1) hv_pose_kernel(const __grid_constant__ PoseBatchArgs b)
{
    __shared__ PoseShared pose_smem;
    pose_job(b.job[blockIdx.x], b.dist, pose_smem);
}

cudaError_t hv_launch_pose(const PoseBatchArgs& b, int njobs, cudaStream_t stream)
{
    hv_pose_kernel<<<njobs, POSE_THREADS, 0, stream>>>(b);
    return cudaGetLastError();
}
