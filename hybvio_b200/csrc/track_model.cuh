// hybvio_b200/csrc/track_model.cuh -- body of the per-track measurement-model kernel (track_model.cu: hv_track_model_kernel).
//
// What Session::trackerVisualUpdate computes on the host for every track before it can call the EKF
// (src/odometry/backend.cpp:1050-1160), here on the device, from the state mean that is already resident:
//   extractCameraPoseTrail                 src/odometry/triangulation.cpp:65-103
//   triangulateWithTwoCameras + pinv/dpinv src/odometry/triangulation.cpp:610-710, 32-51, 1000-1004
//   Triangulator::triangulate              src/odometry/triangulation.cpp:120-407   (Gauss-Newton in inverse depth, with
//                                          the derivative of every iterate w.r.t. every pose and the time shift)
//   per-pose sum of the two cameras        src/odometry/backend.cpp:1105-1116
//   prepareVisualUpdate(truncated)         src/odometry/triangulation.cpp:897-987   -> H (2 n_obs x l, column-major), f
// so that H never exists on the host: the outlier check / update kernels read it where this kernel wrote it.
//
// One CTA of 256 threads per track, any number of tracks per launch (tracks of one launch see the same state mean).
//
// The reference evaluates, for every observation i and every derivative column j (7 per pose + the time shift), the full
// product rule of the residual block: O(n_obs^2) blocks of ~250 flops per Gauss-Newton iteration. The block is LINEAR in
// (dC, dt, d pfi, d residual), and (dC, dt) of observation i are non-zero only for the columns of i's own pose and of pose 0.
// The kernel therefore splits every column into
//   generic part   G d(pfi)_j, TS d(pfi)_j   with G = sum_i d(E_i' e_i)/d pfi, TS = sum_i d(E_i' E_i)/d pfi . step
//                  (3 unit-vector evaluations per observation, reduced once, applied per column)
//   explicit part  14 evaluations per observation (7 own-pose columns, 7 pose-0 columns) + E_i' velocity_i for the time column
// i.e. 18 n_obs block evaluations per iteration instead of n_obs (7 n_obs + 1), spread over the CTA. Sums are taken in a
// different order than the reference's, fp64 differences are rounding only (tests: 1e-9 relative).
//
// Every thread factorises the same 3x3 normal matrix itself (pivoted LDL^T as Eigen's LDLT, the rcond estimate of Eigen's
// ConditionEstimator: the BAD_COND gate has to see the same number) instead of waiting for a broadcast.
//
// Written against the CUDA subset tests/emu runs on the host (threads, __syncthreads, full-warp shuffles):
// tests/emu/emu_track_model.cpp runs this body against oracle/hv_oracle_tri.c without a GPU.
#pragma once
#include <float.h>
#include <math.h>
#include "track_model.h"

// shared-memory carve (doubles)
#define TM_S_POSE 0                                   // n x 48: p 3, R 9, dR 4 x 9
#define TM_S_PP (TM_S_POSE + TM_MAXOBS * 48)          // n x 24: C 9, t 3, h 3, err 2, E 6, 1 / h_z
#define TM_S_DQ (TM_S_PP + TM_MAXOBS * 24)            // (7n + 1) x 3: d pfi
#define TM_S_EXO (TM_S_DQ + (TM_MAXCOL + 1) * 3)      // (7n + 1) x 6: explicit part of d(E'e) (3) and d(E'E) step (3), own-pose columns
#define TM_S_P0 (TM_S_EXO + (TM_MAXCOL + 1) * 6)      // n x 7 x 6: pose-0 items
#define TM_S_GEN (TM_S_P0 + TM_MAXOBS * 42)           // n x 3 x 6: generic items
#define TM_S_TMV (TM_S_GEN + TM_MAXOBS * 18)          // n x 3: E' velocity
#define TM_S_RED (TM_S_TMV + TM_MAXOBS * 3)           // 64: reduced G (18), pose-0 sums (42), time (3)
#define TM_S_SC (TM_S_RED + 64)                       // 32 scalars: ETE 9, Eerror 3, error2, pfi 3 (13..15), pf 3 (16..18)
#define TM_S_TOTAL (TM_S_SC + 32)
// after the iterations the EXO region is reused: d pf after the stereo sum, own blocks and dip R of prepareVisualUpdate
#define TM_S_DPF TM_S_EXO                             // (7 npose + 1) x 3
#define TM_S_OWN (TM_S_DPF + (7 * TM_MAXPOSE + 1) * 3)        // n x 14
#define TM_S_DIPR (TM_S_OWN + TM_MAXOBS * 14)                 // n x 6
static_assert(TM_S_DIPR + TM_MAXOBS * 6 <= TM_S_P0, "stage-E scratch must fit into the EXO region");

__host__ __device__ inline size_t tm_smem_bytes() { return (size_t)TM_S_TOTAL * sizeof(double); }

// ---------------------------------------------------------------------------------------------------- 3x3 helpers (row-major)
__device__ __forceinline__ void tm_mv(const double* A, const double* x, double* y)
{
    for (int i = 0; i < 3; i++) y[i] = A[3 * i] * x[0] + A[3 * i + 1] * x[1] + A[3 * i + 2] * x[2];
}
__device__ __forceinline__ void tm_mtv(const double* A, const double* x, double* y)
{
    for (int i = 0; i < 3; i++) y[i] = A[i] * x[0] + A[3 + i] * x[1] + A[6 + i] * x[2];
}
__device__ __forceinline__ void tm_mm(const double* A, const double* B, double* C)          // C = A B
{
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
__device__ __forceinline__ void tm_mmt(const double* A, const double* B, double* C)         // C = A B'
{
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) C[3 * i + j] = A[3 * i] * B[3 * j] + A[3 * i + 1] * B[3 * j + 1] + A[3 * i + 2] * B[3 * j + 2];
}
__device__ __forceinline__ double tm_nrm(const double* x) { return sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]); }

// rotation of a quaternion and one of its four derivatives (src/odometry/util.cpp:10-47); which = -1: R, 0..3: dR/dq_which
__device__ __forceinline__ void tm_quat_mat(const double* q, int which, double* M)
{
    const double a = 2 * q[0], b = 2 * q[1], c = 2 * q[2], d = 2 * q[3];
    if (which < 0) {
        M[0] = q[0] * q[0] + q[1] * q[1] - q[2] * q[2] - q[3] * q[3]; M[1] = 2 * q[1] * q[2] - 2 * q[0] * q[3]; M[2] = 2 * q[1] * q[3] + 2 * q[0] * q[2];
        M[3] = 2 * q[1] * q[2] + 2 * q[0] * q[3]; M[4] = q[0] * q[0] - q[1] * q[1] + q[2] * q[2] - q[3] * q[3]; M[5] = 2 * q[2] * q[3] - 2 * q[0] * q[1];
        M[6] = 2 * q[1] * q[3] - 2 * q[0] * q[2]; M[7] = 2 * q[2] * q[3] + 2 * q[0] * q[1]; M[8] = q[0] * q[0] - q[1] * q[1] - q[2] * q[2] + q[3] * q[3];
    } else if (which == 0) { M[0] = a; M[1] = -d; M[2] = c; M[3] = d; M[4] = a; M[5] = -b; M[6] = -c; M[7] = b; M[8] = a; }
    else if (which == 1) { M[0] = b; M[1] = c; M[2] = d; M[3] = c; M[4] = -b; M[5] = -a; M[6] = d; M[7] = a; M[8] = -b; }
    else if (which == 2) { M[0] = -c; M[1] = b; M[2] = a; M[3] = b; M[4] = c; M[5] = d; M[6] = -a; M[7] = d; M[8] = -c; }
    else { M[0] = -d; M[1] = -a; M[2] = b; M[3] = a; M[4] = -d; M[5] = c; M[6] = b; M[7] = c; M[8] = d; }
}

// (x, y, z) -> (x, y, 1) / z and its Jacobian (triangulation.cpp:1006-1030); the map is its own inverse
__device__ __forceinline__ void tm_inverse_depth(const double* p, double* ip, double* dip)
{
    ip[0] = p[0] / p[2]; ip[1] = p[1] / p[2]; ip[2] = 1.0 / p[2];
    for (int i = 0; i < 9; i++) dip[i] = 0.0;
    dip[0] = 1.0 / p[2]; dip[4] = 1.0 / p[2];
    for (int i = 0; i < 3; i++) dip[3 * i + 2] = -ip[i] / p[2];
}

// ---------------------------------------------------------------------------------------------------- 3x2 pseudo-inverse
// A[3][2] row-major -> iA[2][3]; column-pivoted QR, rank threshold 2 eps (Eigen's completeOrthogonalDecomposition of a 3x2)
__device__ inline void tm_pinv32(const double* A, double* iA)
{
    double c[2][3] = {{A[0], A[2], A[4]}, {A[1], A[3], A[5]}};
    const int a = tm_nrm(c[1]) > tm_nrm(c[0]) ? 1 : 0, b = 1 - a;
    const double r11 = tm_nrm(c[a]);
    double q1[3], q2[3], u[3];
    for (int i = 0; i < 3; i++) q1[i] = c[a][i] / r11;
    double r12 = q1[0] * c[b][0] + q1[1] * c[b][1] + q1[2] * c[b][2];
    for (int i = 0; i < 3; i++) u[i] = c[b][i] - r12 * q1[i];
    const double r12b = q1[0] * u[0] + q1[1] * u[1] + q1[2] * u[2];
    for (int i = 0; i < 3; i++) u[i] -= r12b * q1[i];
    r12 += r12b;
    const double r22 = tm_nrm(u);
    if (r22 <= 2 * DBL_EPSILON * r11) {
        const double s = r11 * r11 + r12 * r12;
        for (int i = 0; i < 3; i++) { iA[3 * a + i] = r11 * q1[i] / s; iA[3 * b + i] = r12 * q1[i] / s; }
        return;
    }
    for (int i = 0; i < 3; i++) q2[i] = u[i] / r22;
    for (int i = 0; i < 3; i++) { iA[3 * b + i] = q2[i] / r22; iA[3 * a + i] = (q1[i] - r12 * q2[i] / r22) / r11; }
}

// d pinv(A) for a given dA (Golub & Pereyra 1973, eq. 4.12; triangulation.cpp:32-51):
//   -iA dA iA + (iA iA') dA' (I - A iA) + (I - iA A) dA' (iA' iA)
__device__ inline void tm_dpinv32(const double* A, const double* iA, const double* dA, double* diA)
{
    double X[4], t1[6], AiA[9], iAA[4], G2[4], G3[9], u[6];
    for (int i = 0; i < 2; i++) for (int j = 0; j < 2; j++) { double s = 0; for (int k = 0; k < 3; k++) s += iA[3 * i + k] * dA[2 * k + j]; X[2 * i + j] = s; }      // iA dA
    for (int i = 0; i < 2; i++) for (int j = 0; j < 3; j++) t1[3 * i + j] = X[2 * i] * iA[j] + X[2 * i + 1] * iA[3 + j];                                             // (iA dA) iA
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) AiA[3 * i + j] = (i == j ? 1.0 : 0.0) - (A[2 * i] * iA[j] + A[2 * i + 1] * iA[3 + j]);                   // I - A iA
    for (int i = 0; i < 2; i++) for (int j = 0; j < 2; j++) {
        double s = 0, g = 0;
        for (int k = 0; k < 3; k++) { s += iA[3 * i + k] * A[2 * k + j]; g += iA[3 * i + k] * iA[3 * j + k]; }
        iAA[2 * i + j] = (i == j ? 1.0 : 0.0) - s;                                                                                                                     // I - iA A
        G2[2 * i + j] = g;                                                                                                                                             // iA iA'
    }
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) G3[3 * i + j] = iA[i] * iA[j] + iA[3 + i] * iA[3 + j];                                                   // iA' iA
    for (int i = 0; i < 2; i++) for (int j = 0; j < 3; j++) u[3 * i + j] = G2[2 * i] * dA[2 * j] + G2[2 * i + 1] * dA[2 * j + 1];                                    // (iA iA') dA'
    double t2[6], w[6], v[6];
    for (int i = 0; i < 2; i++) for (int j = 0; j < 3; j++) t2[3 * i + j] = u[3 * i] * AiA[j] + u[3 * i + 1] * AiA[3 + j] + u[3 * i + 2] * AiA[6 + j];
    for (int i = 0; i < 2; i++) for (int j = 0; j < 3; j++) v[3 * i + j] = iAA[2 * i] * dA[2 * j] + iAA[2 * i + 1] * dA[2 * j + 1];                                  // (I - iA A) dA'
    for (int i = 0; i < 2; i++) for (int j = 0; j < 3; j++) w[3 * i + j] = v[3 * i] * G3[j] + v[3 * i + 1] * G3[3 + j] + v[3 * i + 2] * G3[6 + j];
    for (int i = 0; i < 6; i++) diA[i] = -t1[i] + t2[i] + w[i];
}

// ---------------------------------------------------------------------------------------------------- 3x3 LDL^T (diagonal pivoting)
// Eigen's LDLT (lower, unblocked, left-looking: the pivot of step k is the largest ORIGINAL diagonal entry among the remaining
// ones, the Schur complement is applied afterwards) written out for 3x3 in scalars, so that it lives in registers: p0 in
// {0,1,2} is the index exchanged with 0, p1 = 1 when indices 1 and 2 were exchanged in the second step.
struct TmLdlt { double l10, l20, l21, i0, i1, i2, l1; int p0, p1; };     // i*: reciprocal pivots (0 below DBL_MIN: pseudo-inverse of D)

__device__ __forceinline__ void tm_swap(double& a, double& b) { const double t = a; a = b; b = t; }

__device__ __forceinline__ void tm_ldlt(const double* A, TmLdlt& X)
{
    double a00 = A[0], a10 = A[3], a11 = A[4], a20 = A[6], a21 = A[7], a22 = A[8];
    const double c0 = fabs(a00) + fabs(a10) + fabs(a20), c1 = fabs(a10) + fabs(a11) + fabs(a21), c2 = fabs(a20) + fabs(a21) + fabs(a22);
    X.l1 = fmax(c0, fmax(c1, c2));                     // max abs column sum of the self-adjoint matrix (lower triangle)
    X.p0 = 0; X.p1 = 0;
    if (fabs(a11) > fabs(a00) && fabs(a11) >= fabs(a22)) { X.p0 = 1; tm_swap(a00, a11); tm_swap(a20, a21); }
    else if (fabs(a22) > fabs(a00) && fabs(a22) > fabs(a11)) { X.p0 = 2; tm_swap(a00, a22); tm_swap(a10, a21); }
    X.l10 = X.l20 = X.l21 = 0.0; X.i0 = X.i1 = X.i2 = 0.0;
    const double d0 = a00;
    if (!(fabs(d0) > 0)) { X.p0 = 0; return; }        // zero matrix: Eigen stops here; every solve returns 0
    const double r0 = 1.0 / d0;
    X.i0 = fabs(d0) > DBL_MIN ? r0 : 0.0;
    double l10 = a10 * r0, l20 = a20 * r0;
    if (fabs(a22) > fabs(a11)) { X.p1 = 1; tm_swap(a11, a22); tm_swap(l10, l20); }
    const double t0 = d0 * l10;
    const double d1 = a11 - l10 * t0;
    double l21 = a21 - l20 * t0;
    if (fabs(d1) > 0) { const double r1 = 1.0 / d1; X.i1 = fabs(d1) > DBL_MIN ? r1 : 0.0; l21 *= r1; }
    const double d2 = a22 - (l20 * (d0 * l20) + l21 * (d1 * l21));
    if (fabs(d2) > DBL_MIN) X.i2 = 1.0 / d2;
    X.l10 = l10; X.l20 = l20; X.l21 = l21;
}

__device__ __forceinline__ void tm_solve(const TmLdlt& X, const double* rhs, double* x)
{
    double v0 = rhs[0], v1 = rhs[1], v2 = rhs[2];
    if (X.p0 == 1) tm_swap(v0, v1); else if (X.p0 == 2) tm_swap(v0, v2);
    if (X.p1) tm_swap(v1, v2);
    v1 -= X.l10 * v0;
    v2 -= X.l20 * v0 + X.l21 * v1;
    v0 *= X.i0; v1 *= X.i1; v2 *= X.i2;
    v1 -= X.l21 * v2;
    v0 -= X.l10 * v1 + X.l20 * v2;
    if (X.p1) tm_swap(v1, v2);
    if (X.p0 == 1) tm_swap(v0, v1); else if (X.p0 == 2) tm_swap(v0, v2);
    x[0] = v0; x[1] = v1; x[2] = v2;
}

// Hager's 1-norm estimate of the inverse with Higham's alternating-sign safeguard, as Eigen's LDLT::rcond()
__device__ inline double tm_rcond(const TmLdlt& X)
{
    if (X.l1 == 0) return 0;
    double v[3] = {1.0 / 3, 1.0 / 3, 1.0 / 3}, sgn[3], old_sgn[3] = {0, 0, 0};
    tm_solve(X, v, v);
    double lower = fabs(v[0]) + fabs(v[1]) + fabs(v[2]), old_lower = lower;
    int jmax = -1, old_jmax = -1;
    for (int k = 0; k < 4; k++) {
        for (int i = 0; i < 3; i++) sgn[i] = v[i] < 0 ? -1.0 : 1.0;
        if (k > 0 && sgn[0] == old_sgn[0] && sgn[1] == old_sgn[1] && sgn[2] == old_sgn[2]) break;
        tm_solve(X, sgn, v);
        jmax = 0; for (int i = 1; i < 3; i++) if (fabs(v[i]) > fabs(v[jmax])) jmax = i;
        if (jmax == old_jmax) break;
        double e[3] = {0, 0, 0}; e[jmax] = 1.0;
        tm_solve(X, e, v);
        lower = fabs(v[0]) + fabs(v[1]) + fabs(v[2]);
        if (lower <= old_lower) break;
        for (int i = 0; i < 3; i++) old_sgn[i] = sgn[i];
        old_jmax = jmax; old_lower = lower;
    }
    double a[3] = {1.0, -1.5, 2.0};
    tm_solve(X, a, a);
    const double alt = 2 * (fabs(a[0]) + fabs(a[1]) + fabs(a[2])) / 9.0;
    const double inv = lower > alt ? lower : alt;
    return inv == 0 ? 0 : (1.0 / inv) / X.l1;
}

// ---------------------------------------------------------------------------------------------------- residual block derivative
// One term of the product rule of triangulation.cpp:216-318 for observation data pp = [C 9 | t 3 | h 3 | err 2 | E 6]:
// given (dC, dt, d pfi) returns a = dE' err + E' dErr (3) and w = (dE' E + E' dE) step (3). extra = additive d residual (2) or NULL.
__device__ inline void tm_block_term(const double* pp, const double* pfi, const double* dC, const double* dt, const double* dq, const double* extra,
                                     const double* step, double* a, double* w)
{
    const double *C = pp, *t = pp + 9, *h = pp + 12, *err = pp + 15, *E = pp + 17;
    double dh[3];
    for (int r = 0; r < 3; r++) {
        double s = dq[2] * t[r] + C[3 * r] * dq[0] + C[3 * r + 1] * dq[1];
        if (dC) s += dC[3 * r] * pfi[0] + dC[3 * r + 1] * pfi[1] + dC[3 * r + 2] + pfi[2] * dt[r];
        dh[r] = s;
    }
    const double ih2 = pp[23], ih2sq = ih2 * ih2;                      // 1 / h_z, computed once per observation and iteration
    const double dih2 = -dh[2] * ih2sq;
    const double dih2sq = -2 * dh[2] * ih2sq * ih2;
    double dErr[2], dE[6];
    for (int r = 0; r < 2; r++) {
        dErr[r] = (extra ? extra[r] : 0.0) - dh[r] * ih2 - dih2 * h[r];
        const double k1 = dh[r] * ih2sq + dih2sq * h[r];
        for (int c = 0; c < 2; c++) {
            double s = -dih2 * C[3 * r + c] + k1 * C[6 + c];
            if (dC) s += -ih2 * dC[3 * r + c] + h[r] * ih2sq * dC[6 + c];
            dE[3 * r + c] = s;
        }
        double s = -t[r] * dih2 + k1 * t[2];
        if (dC) s += -dt[r] * ih2 + h[r] * ih2sq * dt[2];
        dE[3 * r + 2] = s;
    }
    double Es[2] = {E[0] * step[0] + E[1] * step[1] + E[2] * step[2], E[3] * step[0] + E[4] * step[1] + E[5] * step[2]};
    double dEs[2] = {dE[0] * step[0] + dE[1] * step[1] + dE[2] * step[2], dE[3] * step[0] + dE[4] * step[1] + dE[5] * step[2]};
    for (int c = 0; c < 3; c++) {
        a[c] = (dE[c] * err[0] + dE[3 + c] * err[1]) + (E[c] * dErr[0] + E[3 + c] * dErr[1]);
        w[c] = (dE[c] * Es[0] + dE[3 + c] * Es[1]) + (E[c] * dEs[0] + E[3 + c] * dEs[1]);
    }
}

__device__ __forceinline__ int tm_pos_index(int i) { return i == 0 ? TM_POS : TM_CAM + 7 * (i - 1); }          // getPosOriIndices, triangulation.cpp:989-998
__device__ __forceinline__ int tm_ori_index(int i) { return i == 0 ? TM_ORI : TM_CAM + 7 * (i - 1) + 3; }

// ---------------------------------------------------------------------------------------------------- the kernel body
// block: the CTA's index among the tracks of a.  The CTA handles track block + a.trackOffset.
__device__ __forceinline__ void tm_body(const TmArgs& a, double* sm, int block)
{
    __shared__ int s_colmap[TM_MAXN], s_code[TM_MAXOBS];
    // NT threads (a multiple of 32, >= 256: the 4-lane reductions of stage C4 address 63 x 4 threads): TM_NT in its own kernel, the
    // 512 threads of a cluster CTA when the persistent chain kernel runs the model in its CTA 0
    const int NT = (int)blockDim.x;
    const int tid = threadIdx.x, trk = block + a.trackOffset, lane = tid & 31, wrp = tid >> 5;
#ifndef HV_EMU
    if (a.pdl) {        // the next kernel of the chain may be scheduled now (it reads nothing of ours before its own wait); then wait for our predecessor
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
        asm volatile("griddepcontrol.wait;" ::: "memory");
    }
#endif
    if (a.counter && *(volatile const int*)a.counter >= a.counterMax) {      // uniform: written by a kernel that has completed
        if (tid == 0) { int* st = a.status + 4 * (size_t)trk; st[0] = TM_SKIPPED; st[1] = TM_VU_NOT_RUN; st[2] = 0; st[3] = 0; }
        return;
    }
    const int npose = a.npose[trk], ncam = a.stereo ? 2 : 1, n = npose * ncam, dDim = 7 * n;
    const int* idx = a.idx + (size_t)trk * TM_MAXPOSE;
    const double* ip = a.ip + (size_t)trk * TM_MAXOBS * 2;
    const double* vel = a.vel + (size_t)trk * TM_MAXOBS * 2;
    const double* m = a.m;
    double *POSE = sm + TM_S_POSE, *PP = sm + TM_S_PP, *DQ = sm + TM_S_DQ, *EXO = sm + TM_S_EXO, *P0 = sm + TM_S_P0, *GEN = sm + TM_S_GEN;
    double *TMV = sm + TM_S_TMV, *RED = sm + TM_S_RED, *SC = sm + TM_S_SC;

    // ---- A: camera pose trail (triangulation.cpp:65-103): item = (pose, part), part 0: R and p, parts 1..4: dR/dq
    for (int it = tid; it < 5 * n; it += NT) {
        const int k = it / 5, part = it % 5, cam = k / npose, i = idx[k % npose];
        const double* q = m + tm_ori_index(i);
        double Q[9], M[9];
        tm_quat_mat(q, part - 1, Q);
        tm_mm(a.Rc[cam], Q, M);
        double* o = POSE + 48 * k;
        if (part == 0) {
            const double* p = m + tm_pos_index(i);
            double rb[3]; tm_mtv(M, a.base[cam], rb);
            for (int r = 0; r < 3; r++) o[r] = p[r] - rb[r];
            for (int r = 0; r < 9; r++) o[3 + r] = M[r];
        } else {
            for (int r = 0; r < 9; r++) o[12 + 9 * (part - 1) + r] = M[r];
        }
    }
    for (int j = tid; j < 3 * (dDim + 1); j += NT) DQ[j] = 0.0;
    __syncthreads();

    // ---- B: two-view start (triangulation.cpp:610-710) between observation 0 and the last one of camera 0 (:157-158)
    const int ind1 = a.stereo ? n / 2 - 1 : n - 1;
    const double *P0p = POSE, *P1p = POSE + 48 * ind1;
    if (tid < 15) {
        const double *R0 = P0p + 3, *R1 = P1p + 3;
        double C[9], d[3], b[3], v0[3] = {ip[0], ip[1], 1.0}, v1[3] = {ip[2 * ind1], ip[2 * ind1 + 1], 1.0};
        tm_mmt(R0, R1, C);
        for (int r = 0; r < 3; r++) d[r] = P1p[r] - P0p[r];
        tm_mv(R0, d, b);
        const double n0 = tm_nrm(v0), n1 = tm_nrm(v1);
        double vn0[3], vn1[3], Cv[3], A[6], iA[6];
        for (int r = 0; r < 3; r++) { vn0[r] = v0[r] / n0; vn1[r] = v1[r] / n1; }
        tm_mv(C, vn1, Cv);
        for (int r = 0; r < 3; r++) { A[2 * r] = vn0[r]; A[2 * r + 1] = -Cv[r]; }
        tm_pinv32(A, iA);
        const double s0 = iA[0] * b[0] + iA[1] * b[1] + iA[2] * b[2];
        double pf0[3] = {s0 * vn0[0], s0 * vn0[1], s0 * vn0[2]}, pfi[3], dpfi_dpf[9];
        tm_inverse_depth(pf0, pfi, dpfi_dpf);
        // this thread's derivative column: 0..2 p0, 3..6 q0, 7..9 p1, 10..13 q1, 14 time shift
        double dA[6] = {0, 0, 0, 0, 0, 0}, db[3] = {0, 0, 0}, col[3];
        const int j = tid;
        if (j < 3) { for (int r = 0; r < 3; r++) db[r] = -R0[3 * r + j]; }
        else if (j < 7) {
            const double* dR0 = P0p + 12 + 9 * (j - 3);
            double dC[9], x[3];
            tm_mmt(dR0, R1, dC); tm_mv(dC, vn1, x);
            for (int r = 0; r < 3; r++) dA[2 * r + 1] = -x[r];
            tm_mv(dR0, d, db);
        } else if (j < 10) { for (int r = 0; r < 3; r++) db[r] = R0[3 * r + (j - 7)]; }
        else if (j < 14) {
            const double* dR1 = P1p + 12 + 9 * (j - 10);
            double dC[9], x[3];
            tm_mmt(R0, dR1, dC); tm_mv(dC, vn1, x);
            for (int r = 0; r < 3; r++) dA[2 * r + 1] = -x[r];
        }
        if (j < 14) {
            double diA[6];
            tm_dpinv32(A, iA, dA, diA);
            const double ds = (iA[0] * db[0] + iA[1] * db[1] + iA[2] * db[2]) + (diA[0] * b[0] + diA[1] * b[1] + diA[2] * b[2]);
            for (int r = 0; r < 3; r++) col[r] = ds * vn0[r];
        } else if (a.timeShift) {
            double w0[3] = {vel[0], vel[1], 0.0}, w1[3] = {vel[2 * ind1], vel[2 * ind1 + 1], 0.0}, x[3], y[3], Cy[3], diA[6];
            for (int r = 0; r < 3; r++) {
                x[r] = (w0[r] - vn0[r] * (vn0[0] * w0[0] + vn0[1] * w0[1] + vn0[2] * w0[2])) / n0;         // (I - vn vn') w / |v|
                y[r] = (w1[r] - vn1[r] * (vn1[0] * w1[0] + vn1[1] * w1[1] + vn1[2] * w1[2])) / n1;
            }
            tm_mv(C, y, Cy);
            for (int r = 0; r < 3; r++) { dA[2 * r] = x[r]; dA[2 * r + 1] = -Cy[r]; }
            tm_dpinv32(A, iA, dA, diA);
            const double ds0 = diA[0] * b[0] + diA[1] * b[1] + diA[2] * b[2];
            for (int r = 0; r < 3; r++) col[r] = s0 * x[r] + vn0[r] * ds0;
        } else { col[0] = col[1] = col[2] = 0.0; }
        // in inverse depth (triangulation.cpp:183-198). The columns of the second pose are written by threads 7..13; for
        // ind1 == 0 they would overwrite those of the first, as in the reference -- tracks have >= 2 poses (checked by the host)
        double cq[3]; tm_mv(dpfi_dpf, col, cq);
        const int dst = j < 7 ? j : j < 14 ? 7 * ind1 + (j - 7) : dDim;
        for (int r = 0; r < 3; r++) DQ[3 * dst + r] = cq[r];
        if (tid == 0) for (int r = 0; r < 3; r++) { SC[13 + r] = pfi[r]; SC[16 + r] = pf0[r]; }
    }
    __syncthreads();

    // ---- C: Gauss-Newton (triangulation.cpp:200-346)
    const double* R0 = POSE + 3;
    const double* p0 = POSE;
    double Jprev = 1e10, rcond = 0.0;
    bool converged = false;
    TmLdlt X;
    for (unsigned iter = 0; iter < a.gnIterations; iter++) {
        // C1: warp 0 evaluates the residual blocks of its observations (lane, lane + 32) and reduces E'E, E'e, |e|^2
        if (wrp == 0) {
            double acc[13];
            for (int r = 0; r < 13; r++) acc[r] = 0.0;
            const double pfi[3] = {SC[13], SC[14], SC[15]};
            for (int i = lane; i < n; i += 32) {
                const double* cur = POSE + 48 * i;
                double* pp = PP + 24 * i;
                double C[9], dp[3], t[3], h[3], err[2], E[6];
                tm_mmt(cur + 3, R0, C);
                for (int r = 0; r < 3; r++) dp[r] = p0[r] - cur[r];
                tm_mv(cur + 3, dp, t);
                for (int r = 0; r < 3; r++) h[r] = (C[3 * r] * pfi[0] + C[3 * r + 1] * pfi[1] + C[3 * r + 2]) + pfi[2] * t[r];
                const double ih2 = 1.0 / h[2], ih2sq = ih2 * ih2;       // the only division of the block (the reference divides per term)
                for (int r = 0; r < 2; r++) {
                    err[r] = ip[2 * i + r] - h[r] * ih2;
                    for (int c = 0; c < 2; c++) E[3 * r + c] = -ih2 * C[3 * r + c] + h[r] * ih2sq * C[6 + c];
                    E[3 * r + 2] = -t[r] * ih2 + h[r] * ih2sq * t[2];
                }
                pp[23] = ih2;
                for (int r = 0; r < 9; r++) pp[r] = C[r];
                for (int r = 0; r < 3; r++) { pp[9 + r] = t[r]; pp[12 + r] = h[r]; }
                pp[15] = err[0]; pp[16] = err[1];
                for (int r = 0; r < 6; r++) pp[17 + r] = E[r];
                for (int x = 0; x < 3; x++) {
                    for (int y = 0; y < 3; y++) acc[3 * x + y] += E[x] * E[y] + E[3 + x] * E[3 + y];
                    acc[9 + x] += E[x] * err[0] + E[3 + x] * err[1];
                }
                acc[12] += err[0] * err[0] + err[1] * err[1];
            }
            for (int r = 0; r < 13; r++) {
                double v = acc[r];
                for (int o = 16; o > 0; o >>= 1) v += __shfl_sync(0xffffffffu, v, lane ^ o);
                if (lane == 0) SC[r] = v;
            }
        }
        __syncthreads();
        // C2: every thread factorises E'E and solves for the step itself
        double ETE[9], Eerr[3], step[3], pfi[3];
        for (int r = 0; r < 9; r++) ETE[r] = SC[r];
        for (int r = 0; r < 3; r++) { Eerr[r] = SC[9 + r]; pfi[r] = SC[13 + r]; }
        const double error2 = SC[12];
        tm_ldlt(ETE, X);
        tm_solve(X, Eerr, step);
        // C3: the 18 n block terms
        for (int it = tid; it < 18 * n; it += NT) {
            double av[3], wv[3];
            if (it < 3 * n) {                                   // generic: d pfi = e_k
                const int i = it / 3, k = it % 3;
                double dq[3] = {0, 0, 0}; dq[k] = 1.0;
                tm_block_term(PP + 24 * i, pfi, nullptr, nullptr, dq, nullptr, step, av, wv);
                double* o = GEN + 18 * i + 6 * k;
                for (int r = 0; r < 3; r++) { o[r] = av[r]; o[3 + r] = wv[r]; }
            } else if (it < 17 * n) {
                const bool own = it < 10 * n;
                const int e = own ? it - 3 * n : it - 10 * n, i = e / 7, comp = e % 7;
                const double* cur = POSE + 48 * i;
                double dC[9], dt[3];
                const double zero3[3] = {0, 0, 0};
                if (own) {                                      // column of observation i's own pose: dRi, dpi
                    if (comp < 3) {
                        for (int r = 0; r < 9; r++) dC[r] = 0.0;
                        for (int r = 0; r < 3; r++) dt[r] = -cur[3 + 3 * r + comp];                       // Ri (-e_comp)
                    } else {
                        const double* dRi = cur + 12 + 9 * (comp - 3);
                        double dpi[3], dp[3], x[3], y[3];
                        tm_mtv(dRi, a.base[i / npose], dpi);                                              // dpi = -dRi' baseline
                        tm_mmt(dRi, R0, dC);
                        for (int r = 0; r < 3; r++) dp[r] = p0[r] - cur[r];
                        tm_mv(dRi, dp, x); tm_mv(cur + 3, dpi, y);                                         // Ri (0 - dpi) = +Ri (dRi' baseline)
                        for (int r = 0; r < 3; r++) dt[r] = x[r] + y[r];
                    }
                } else {                                        // column of pose 0: dR0, dp0
                    if (comp < 3) {
                        for (int r = 0; r < 9; r++) dC[r] = 0.0;
                        for (int r = 0; r < 3; r++) dt[r] = cur[3 + 3 * r + comp];                        // Ri e_comp
                    } else {
                        const double* dR0 = POSE + 12 + 9 * (comp - 3);
                        double dp0[3];
                        tm_mtv(dR0, a.base[0], dp0);
                        for (int r = 0; r < 3; r++) dp0[r] = -dp0[r];
                        tm_mmt(cur + 3, dR0, dC);
                        tm_mv(cur + 3, dp0, dt);
                    }
                }
                tm_block_term(PP + 24 * i, pfi, dC, dt, zero3, nullptr, step, av, wv);
                double* o = own ? EXO + 6 * (7 * i + comp) : P0 + 42 * i + 6 * comp;
                for (int r = 0; r < 3; r++) { o[r] = av[r]; o[3 + r] = wv[r]; }
            } else {                                            // time column: E_i' velocity_i
                const int i = it - 17 * n;
                const double* E = PP + 24 * i + 17;
                for (int r = 0; r < 3; r++) TMV[3 * i + r] = a.timeShift ? E[r] * vel[2 * i] + E[3 + r] * vel[2 * i + 1] : 0.0;
            }
        }
        __syncthreads();
        // C4: 63 sums over the observations: generic (18), pose-0 columns (42), time column (3); four lanes per sum
        {
            const int sidx = tid >> 2, part = tid & 3;
            const double* src = GEN; int stride = 0;
            if (sidx < 18) { src = GEN + sidx; stride = 18; }
            else if (sidx < 60) { src = P0 + (sidx - 18); stride = 42; }
            else if (sidx < 63) { src = TMV + (sidx - 60); stride = 3; }
            double sacc = 0.0;
            if (sidx < 63) for (int i = part; i < n; i += 4) sacc += src[(size_t)i * stride];
            sacc += __shfl_sync(0xffffffffu, sacc, lane ^ 1);
            sacc += __shfl_sync(0xffffffffu, sacc, lane ^ 2);
            if (sidx < 63 && part == 0) RED[sidx] = sacc;
        }
        __syncthreads();
        // C5: d pfi_j += X^-1 (w_j - a_j)   (:322-327 with the two solves of the reference merged into one)
        for (int j = tid; j <= dDim; j += NT) {
            double* dq = DQ + 3 * j;
            double rhs[3], upd[3];
            for (int r = 0; r < 3; r++) {
                double av = RED[r] * dq[0] + RED[6 + r] * dq[1] + RED[12 + r] * dq[2];
                double wv = RED[3 + r] * dq[0] + RED[9 + r] * dq[1] + RED[15 + r] * dq[2];
                if (j < dDim) { av += EXO[6 * j + r]; wv += EXO[6 * j + 3 + r]; }
                if (j < 7) { av += RED[18 + 6 * j + r]; wv += RED[18 + 6 * j + 3 + r]; }
                if (j == dDim) av += RED[60 + r];
                rhs[r] = wv - av;
            }
            if (j == dDim && !a.timeShift) continue;
            tm_solve(X, rhs, upd);
            for (int r = 0; r < 3; r++) dq[r] += upd[r];
        }
        if (tid == 0) for (int r = 0; r < 3; r++) SC[13 + r] = pfi[r] - step[r];
        // convergence (:337-345): uniform over the CTA, everybody computes it
        const double J = 0.5 * error2 / (a.convR * a.convR);
        const double Jd = fabs((J - Jprev) / J);
        Jprev = J;
        __syncthreads();
        if (Jd < a.convThreshold) { converged = true; break; }
    }
    rcond = tm_rcond(X);

    int tri = TM_OK;
    if (!converged) tri = TM_NO_CONVERGENCE;
    else if (rcond < a.rcondThreshold) tri = TM_BAD_COND;
    double pf[3] = {SC[16], SC[17], SC[18]};            // the two-view point, in the frame of observation 0 (what the reference leaves in out.pf)
    if (tri == TM_OK) {
        // ---- D: back from inverse depth (:359-395), behind-camera test (:53-59)
        double pfi[3] = {SC[13], SC[14], SC[15]}, pf0[3], dpf0[9], rp[3], R0T[9], M[9];
        tm_inverse_depth(pfi, pf0, dpf0);
        tm_mtv(R0, pf0, rp);
        for (int r = 0; r < 3; r++) pf[r] = rp[r] + p0[r];
        if (pf[0] == p0[0] && pf[1] == p0[1] && pf[2] == p0[2]) tri = TM_UNKNOWN_PROBLEM;
        else {
            for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) R0T[3 * r + c] = R0[3 * c + r];
            tm_mm(R0T, dpf0, M);
            for (int j = tid; j <= dDim; j += NT) {
                double x[3], y[3] = {0, 0, 0};
                tm_mv(M, DQ + 3 * j, x);
                if (j >= 3 && j < 7) tm_mtv(POSE + 12 + 9 * (j - 3), pf0, y);
                for (int r = 0; r < 3; r++) DQ[3 * j + r] = y[r] + x[r] + (j == r ? 1.0 : 0.0);
            }
            if (tid < n) {
                const double* cur = POSE + 48 * tid;
                double d[3], c3[3];
                for (int r = 0; r < 3; r++) d[r] = pf[r] - cur[r];
                tm_mv(cur + 3, d, c3);
                s_code[tid] = c3[2] < 0 ? 1 : 0;                    // one word per observation: no two threads write the same address
            }
        }
    }
    __syncthreads();
    if (tri == TM_OK) { int behind = 0; for (int i = 0; i < n; i++) behind |= s_code[i]; if (behind) tri = TM_BEHIND; }
    const double depth = sqrt((pf[0] - p0[0]) * (pf[0] - p0[0]) + (pf[1] - p0[1]) * (pf[1] - p0[1]) + (pf[2] - p0[2]) * (pf[2] - p0[2]));
    if (depth < a.minDist || depth > a.maxDist) tri = TM_BAD_DEPTH;                                     // backend.cpp:1095-1098

    int* st = a.status + 4 * (size_t)trk;
    if (tid == 0) { for (int r = 0; r < 3; r++) a.pf[4 * (size_t)trk + r] = pf[r]; a.pf[4 * (size_t)trk + 3] = depth; }
    double* dpfOut = a.dpf ? a.dpf + (size_t)trk * 3 * (7 * TM_MAXPOSE + 1) : nullptr;
    if (tri != TM_OK) {
        if (tid == 0) { st[0] = tri; st[1] = TM_VU_NOT_RUN; st[2] = 0; st[3] = 0; }
        if (dpfOut) for (int j = tid; j < 3 * (7 * npose + 1); j += NT) dpfOut[j] = 0.0;
        return;
    }

    // ---- E: stereo sum (backend.cpp:1105-1116) and prepareVisualUpdate (triangulation.cpp:897-987)
    double *DPF = sm + TM_S_DPF, *OWN = sm + TM_S_OWN, *DIPR = sm + TM_S_DIPR;
    double held[2][3];                                  // DPF aliases EXO, not DQ: no hazard, but keep the sum in registers until the barrier for clarity
    int nheld = 0;
    for (int j = tid; j < 7 * npose + 1; j += NT, nheld++)
        for (int r = 0; r < 3; r++)
            held[nheld][r] = j == 7 * npose ? DQ[3 * dDim + r] : DQ[3 * j + r] + (a.stereo ? DQ[3 * (7 * npose + j) + r] : 0.0);
    nheld = 0;
    for (int j = tid; j < 7 * npose + 1; j += NT, nheld++)
        for (int r = 0; r < 3; r++) { DPF[3 * j + r] = held[nheld][r]; if (dpfOut) dpfOut[3 * j + r] = held[nheld][r]; }
    int end = 0;
    for (int k = 0; k < npose; k++) { const int e = tm_ori_index(idx[k]) + 4 > tm_pos_index(idx[k]) + 3 ? tm_ori_index(idx[k]) + 4 : tm_pos_index(idx[k]) + 3; if (e > end) end = e; }
    for (int c = tid; c < end; c += NT) s_colmap[c] = -1;
    __syncthreads();
    if (tid < npose) {
        const int pos = tm_pos_index(idx[tid]), ori = tm_ori_index(idx[tid]);
        for (int c = 0; c < 3; c++) s_colmap[pos + c] = 7 * tid + c;
        for (int c = 0; c < 4; c++) s_colmap[ori + c] = 7 * tid + 3 + c;
    }
    if (tid < n) {
        const double* cur = POSE + 48 * tid;
        double pt[3], pfc[3], ipH[3], dipH[9];
        for (int r = 0; r < 3; r++) pt[r] = pf[r] - cur[r];
        tm_mv(cur + 3, pt, pfc);
        s_code[tid] = pfc[2] == 0 ? TM_VU_ZERO_DEPTH : pfc[2] < 0 ? TM_VU_BEHIND : TM_VU_OK;
        tm_inverse_depth(pfc, ipH, dipH);
        a.f[(size_t)trk * 2 * TM_MAXOBS + 2 * tid] = ipH[0];
        a.f[(size_t)trk * 2 * TM_MAXOBS + 2 * tid + 1] = ipH[1];
        double* dr = DIPR + 6 * tid;
        for (int r = 0; r < 2; r++) for (int c = 0; c < 3; c++) dr[3 * r + c] = dipH[3 * r] * cur[3 + c] + dipH[3 * r + 1] * cur[6 + c] + dipH[3 * r + 2] * cur[9 + c];
        double* ow = OWN + 14 * tid;
        for (int r = 0; r < 2; r++) for (int c = 0; c < 3; c++) ow[7 * r + c] = -dr[3 * r + c];
        for (int j = 0; j < 4; j++) {
            const double* dRj = cur + 12 + 9 * j;
            double x[3], b[3], y[3];
            tm_mv(dRj, pt, x); tm_mtv(dRj, a.base[tid / npose], b); tm_mv(cur + 3, b, y);
            for (int r = 0; r < 2; r++) ow[7 * r + 3 + j] = dipH[3 * r] * (x[0] + y[0]) + dipH[3 * r + 1] * (x[1] + y[1]) + dipH[3 * r + 2] * (x[2] + y[2]);
        }
    }
    __syncthreads();
    int vu = TM_VU_OK;
    for (int i = 0; i < n && vu == TM_VU_OK; i++) vu = s_code[i];         // the first failing observation decides (:924-931)
    const int rows = 2 * n;
    if (tid == 0) { st[0] = TM_OK; st[1] = vu; st[2] = rows; st[3] = end; }
    if (vu != TM_VU_OK) return;
    // H(2i + r, c): every element written exactly once; a warp per column, lanes along the rows (contiguous in memory)
    double* H = a.H + (size_t)trk * a.Hstride;
    for (int c = wrp; c < end; c += NT / 32) {
        const int mc = s_colmap[c];
        const bool sft = mc < 0 && c == TM_SFT && a.timeShift;
        const double* d = mc >= 0 ? DPF + 3 * mc : DPF + 3 * 7 * npose;
        const int ownPose = mc >= 0 ? mc / 7 : -1, comp = mc >= 0 ? mc % 7 : 0;
        for (int rr = lane; rr < rows; rr += 32) {
            const int i = rr >> 1, r = rr & 1;
            const double* dr = DIPR + 6 * i + 3 * r;
            double v = 0.0;
            if (mc >= 0) {
                v = dr[0] * d[0] + dr[1] * d[1] + dr[2] * d[2];
                if (ownPose == (i >= npose ? i - npose : i)) v = OWN[14 * i + 7 * r + comp] + v;
            } else if (sft) {
                v = (dr[0] * d[0] + dr[1] * d[1] + dr[2] * d[2]) - vel[2 * i + r];
            }
            H[(size_t)c * rows + rr] = v;
        }
    }
}
// CTA blockIdx.x of a batch (the emulator drivers of tests/emu call this form)
__device__ __forceinline__ void tm_body(const TmArgs& a, double* sm) { tm_body(a, sm, (int)blockIdx.x); }

// CTA `inst` of a group launch (hv_track_model_group_kernel): the first track of its own argument block args[inst], one filter's
// chain step, read from device memory
__device__ __forceinline__ void tm_group_body(const TmArgs* __restrict__ args, int inst, double* sm) { tm_body(args[inst], sm, 0); }
