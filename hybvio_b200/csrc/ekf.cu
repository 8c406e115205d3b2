// hybvio_b200/csrc/ekf.cu -- EKF kernels (fp64) for sm_90a. State m (N) and covariance P (N x N, column-major)
// stay resident in HBM/L2; every reference EKF method is ONE kernel launch of a single persistent CTA that keeps
// its working set in shared memory.
//
// Replaces EKFImplementation (src/odometry/ekf.cpp):
//   ekf_predict_kernel      predict()                          ekf.cpp:320-514
//   ekf_update_kernel       update() + the fixed-H updates     ekf.cpp:57-82, 573-677
//                           visualTrackUpdateCommon/OutlierCheck/updateVisualTrack   ekf.cpp:760-844
//                           updateVisualPoseAugmentation + updateCommonJosephForm    ekf.cpp:848-885, 35-50
//   ekf_ew_kernel           updateUndoAugmentation, maintainPositiveSemiDefinite, normalizeQuaternions,
//                           translateTo/transformTo, insertMapPoint, conditionOnLastPose, lockBiases,
//                           initializeOrientation              ekf.cpp:888-947, 1024-1067, 696-758, 299-317
//
// Kalman update algebra. The reference forms HP = H P[0:l,:], S = HP[:,0:l] H' + R, a pivoted LDLT of S,
// K = (S^-1 HP)', m += K v, P -= K HP (and, for the augmentation, the Joseph form with two dense N^3 GEMMs).
// Here one tableau  T = [ S | HP | v ]  (n x (n+N+1), shared memory) is reduced by unpivoted forward elimination
// (S is SPD: R > 0), which turns it into [ D L' | Y | y ] with Y = L^-1 HP; after scaling row k by d_k^-1/2:
//   chi2 = |z_v|^2,   m += Z' z_v,   P -= Z' Z        (Z = D^-1/2 L^-1 HP)
// i.e. K HP = HP' S^-1 HP = Z'Z. No back substitution, no explicit gain, P's update is a symmetric rank-n
// downdate computed once per (i >= j) 4x4 block and mirrored. The Joseph form of the augmentation is
// algebraically the same matrix (K S K' = K HP for the optimal gain), so augmentation = shift + this update
// with the sparse 7 x 27 visAugH + symmetrisation: O(N^2) instead of the reference's O(N^3).
// fp64 differences to the reference are rounding-order only (tests: relative 1e-9 on P, 1e-10 on m).
#include "ekf.cuh"
#include "hv_device_once.cuh"
#include <math.h>
#include <stdlib.h>

// ------------------------------------------------------------------------------------------------ helpers
__device__ __forceinline__ void normalize_quat(double* q)
{
    // Eigen's normalize(): if squaredNorm > 0, divide by its sqrt (zero trail slots stay zero, ekf.cpp:1028-1030)
    const double z = (q[0] * q[0] + q[2] * q[2]) + (q[1] * q[1] + q[3] * q[3]);
    if (z > 0.0) { const double nrm = sqrt(z); q[0] /= nrm; q[1] /= nrm; q[2] /= nrm; q[3] /= nrm; }
}

__device__ __forceinline__ void normalize_all(double* m, int trail, bool onlyCurrent)
{
    for (int q = threadIdx.x; q < (onlyCurrent ? 1 : trail + 1); q += blockDim.x)
        normalize_quat(q == 0 ? m + EKF_ORI : m + EKF_CAM + EKF_POSE * (q - 1) + 3);
}

__device__ __forceinline__ void symmetrize(double* P, int N)
{
    // P = 0.5 (P + P')  (ekf.cpp:1065); grid-stride: every (i > j) pair is owned by exactly one thread
    for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < N * N; idx += gridDim.x * blockDim.x) {
        const int i = idx % N, j = idx / N;
        if (i > j) {
            const double s = 0.5 * (P[i + (size_t)j * N] + P[j + (size_t)i * N]);
            P[i + (size_t)j * N] = s; P[j + (size_t)i * N] = s;
        }
    }
}

// source index of the augmentation shift A (ekf.cpp:230-248): row i of A*x takes x[src], -1 = zero
__device__ __forceinline__ int aug_src(int i, int drop)
{
    if (i < EKF_CAM) return i;
    if (i < EKF_CAM + EKF_POSE) return -1;
    if (i < EKF_CAM + (drop + 1) * EKF_POSE) return i - EKF_POSE;
    return i;
}
// visUnaugmentA (ekf.cpp:250-265)
__device__ __forceinline__ int unaug_src(int i, int poseTrailDim)
{
    if (i < EKF_CAM) return i;
    if (i >= poseTrailDim) return i;
    if (i + EKF_POSE < poseTrailDim) return i + EKF_POSE;
    return -1;
}

// sym: a deferred maintainPositiveSemiDefinite() is applied while P is read (the operand pair of symmetrize())
template <class SrcFn>
__device__ __forceinline__ void shift_state(const double* __restrict__ P, double* __restrict__ P2, double* m, int N, SrcFn src, bool sym = false)
{
    for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < N * N; idx += gridDim.x * blockDim.x) {
        const int i = idx % N, j = idx / N;
        const int si = src(i), sj = src(j);
        double v = (si < 0 || sj < 0) ? 0.0 : P[si + (size_t)sj * N];
        if (sym && si >= 0 && sj >= 0 && si != sj) v = 0.5 * (v + P[sj + (size_t)si * N]);
        P2[idx] = v;
    }
    if (blockIdx.x != 0) return;   // the state vector is shifted by block 0
    double tmp[4];   // N <= 4 * EKF_NT
#pragma unroll
    for (int r = 0; r < 4; r++) {
        const int i = threadIdx.x + r * blockDim.x;
        if (i < N) { const int s = src(i); tmp[r] = s < 0 ? 0.0 : m[s]; }
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 4; r++) {
        const int i = threadIdx.x + r * blockDim.x;
        if (i < N) m[i] = tmp[r];
    }
}

// ------------------------------------------------------------------------------------------------ update
__global__ void __launch_bounds__(EKF_NT) ekf_update_kernel(EkfUpdateArgs a)
{
    extern __shared__ double dyn_smem[];
    __shared__ double s_scalar[4];
    const int tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5, nwarps = EKF_NT / 32;
    const int N = a.b.N;
    int n = a.n, l = a.l;
    double* m = a.b.m;
    double* P = a.b.P;

    // ---- phase 0 (augmentation only): m = A m, P = A P A' + visAugQ  (ekf.cpp:853-857), out of place into P2
    if (a.op == EKF_OP_AUGMENT) {
        const int drop = a.dropIdx;
        shift_state(P, a.b.P2, m, N, [drop](int i) { return aug_src(i, drop); }, a.symFirst != 0);
        __syncthreads();
        P = a.b.P2;
        if (tid < EKF_POSE) P[(EKF_CAM + tid) * (size_t)(N + 1)] += tid < 3 ? a.augNoisePos : a.augNoiseOri;
        __syncthreads();
    }

    // ---- phase 1: measurement model. Built-in models write the dense (truncated) H into b.Hs (ld = n).
    const double* H = a.H;
    double hspeed = 0.0;
    if (a.op != EKF_OP_DENSE) {
        double* Hs = a.b.Hs;
        for (int i = tid; i < n * l; i += EKF_NT) Hs[i] = 0.0;
        if (a.op == EKF_OP_PSEUDO_VELOCITY) {
            hspeed = sqrt(m[EKF_VEL] * m[EKF_VEL] + m[EKF_VEL + 1] * m[EKF_VEL + 1]);
            if (hspeed <= 1e-7) return;                               // ekf.cpp:635-637
        }
        __syncthreads();
        if (tid == 0) {
            switch (a.op) {
                case EKF_OP_ZUPT: for (int i = 0; i < 3; i++) Hs[i + (EKF_VEL + i) * n] = 1.0; break;
                case EKF_OP_ZRUPT: for (int i = 0; i < 3; i++) Hs[i + (EKF_BGA + i) * n] = 1.0; break;
                case EKF_OP_PSEUDO_VELOCITY: for (int i = 0; i < 2; i++) Hs[(EKF_VEL + i) * n] = m[EKF_VEL + i] / hspeed; break;
                case EKF_OP_POSITION: for (int i = 0; i < 3; i++) Hs[i + (EKF_POS + i) * n] = 1.0; break;
                case EKF_OP_ZERO_HEIGHT: Hs[(EKF_POS + 2) * n] = 1.0; break;
                case EKF_OP_ORIENTATION: for (int i = 0; i < 4; i++) Hs[i + (EKF_ORI + i) * n] = 1.0; break;
                case EKF_OP_AUGMENT:   // visAugH (ekf.cpp:267-277), truncated to its 27 non-zero columns
                    for (int i = 0; i < 3; i++) { Hs[i + (EKF_POS + i) * n] = 1.0; Hs[i + (EKF_CAM + i) * n] = -1.0; }
                    for (int i = 0; i < 4; i++) { Hs[3 + i + (EKF_ORI + i) * n] = 1.0; Hs[3 + i + (EKF_CAM + 3 + i) * n] = -1.0; }
                    break;
            }
        }
        __syncthreads();
        H = Hs;
    }

    const bool joseph = a.op == EKF_OP_AUGMENT;     // needs the explicit gain: carry an identity block through
    const int W = (n + N + 1 + (joseph ? n : 0)) | 1;   // odd row length: conflict-free column walks
    double* T = a.useGlobalWork ? a.b.work : dyn_smem;
    const int cv = n + N;                           // column of the residual
    const int cend = joseph ? cv + n : cv;          // last tableau column
    if (joseph) for (int t = tid; t < n * n; t += EKF_NT) T[(size_t)(t / n) * W + cv + 1 + (t % n)] = (t / n == t % n) ? 1.0 : 0.0;

    // residual v = y - f (visual) or y - H m[0:l] (update(), ekf.cpp:77-79)
    for (int i = tid; i < n; i += EKF_NT) {
        double v;
        if (a.op == EKF_OP_PSEUDO_VELOCITY) v = a.defaultSpeed - hspeed;
        else {
            const double yi = a.y ? a.y[i] : a.ysmall[i];
            double fi = 0.0;
            if (a.f) fi = a.f[i];
            else for (int k = 0; k < l; k++) fi += H[i + (size_t)k * n] * m[k];
            v = yi - fi;
        }
        T[(size_t)i * W + cv] = v;
    }
    __syncthreads();

    const bool checking = a.mode != EKF_MODE_UPDATE;
    if (checking && a.rmseThr >= 0.0) {               // ekf.cpp:797-801
        if (tid == 0) {
            double ss = 0.0; for (int i = 0; i < n; i++) { const double v = T[(size_t)i * W + cv]; ss += v * v; }
            s_scalar[0] = sqrt(ss / n);
        }
        __syncthreads();
        if (s_scalar[0] > a.rmseThr) { if (tid == 0) ekf_report(a, 2.0, 0.0, 0.0); return; }
    }
    if (checking && a.skipChi2 && a.mode == EKF_MODE_CHECK) {   // ekf.cpp:803
        if (tid == 0) ekf_report(a, 0.0, 0.0, 0.0);
        return;
    }

    // ---- phase 2: HP = H P[0:l, :]  ->  T[:, n .. n+N)      (2 x 4 register tiles)
    {
        const int tm = (n + 1) >> 1, tn = (N + 3) >> 2;
        for (int t = tid; t < tm * tn; t += EKF_NT) {
            const int ti = t % tm, tj = t / tm;
            const int i0 = ti, i1 = min(ti + tm, n - 1);
            const int j0 = tj * 4;
            const double* p0 = P + (size_t)min(j0, N - 1) * N;
            const double* p1 = P + (size_t)min(j0 + 1, N - 1) * N;
            const double* p2 = P + (size_t)min(j0 + 2, N - 1) * N;
            const double* p3 = P + (size_t)min(j0 + 3, N - 1) * N;
            double c00 = 0, c01 = 0, c02 = 0, c03 = 0, c10 = 0, c11 = 0, c12 = 0, c13 = 0;
            for (int k = 0; k < l; k++) {
                const double h0 = H[i0 + (size_t)k * n], h1 = H[i1 + (size_t)k * n];
                const double b0 = p0[k], b1 = p1[k], b2 = p2[k], b3 = p3[k];
                c00 += h0 * b0; c01 += h0 * b1; c02 += h0 * b2; c03 += h0 * b3;
                c10 += h1 * b0; c11 += h1 * b1; c12 += h1 * b2; c13 += h1 * b3;
            }
            double* r0 = T + (size_t)i0 * W + n + j0;
            double* r1 = T + (size_t)i1 * W + n + j0;
            r0[0] = c00; if (j0 + 1 < N) r0[1] = c01; if (j0 + 2 < N) r0[2] = c02; if (j0 + 3 < N) r0[3] = c03;
            if (ti + tm < n) { r1[0] = c10; if (j0 + 1 < N) r1[1] = c11; if (j0 + 2 < N) r1[2] = c12; if (j0 + 3 < N) r1[3] = c13; }
        }
    }
    __syncthreads();
    // ---- phase 3: S = HP[:, 0:l] H' + R  ->  T[:, 0 .. n)
    for (int t = tid; t < n * n; t += EKF_NT) {
        const int j = t % n, i = t / n;
        const double* hp = T + (size_t)i * W + n;
        double s = 0.0;
        for (int k = 0; k < l; k++) s += hp[k] * H[j + (size_t)k * n];
        T[(size_t)i * W + j] = s + (i == j ? a.Rdiag : 0.0);
    }
    __syncthreads();

    // ---- phase 4: unpivoted forward elimination of [S | HP | v]; warps own rows, lanes walk columns
    bool bad = false;
    for (int k = 0; k < n; k++) {
        const double piv = T[(size_t)k * W + k];
        if (!(piv > 0.0)) { bad = true; break; }
        const double rinv = 1.0 / piv;
        const double* rk = T + (size_t)k * W;
        for (int i = k + 1 + wrp; i < n; i += nwarps) {
            double* ri = T + (size_t)i * W;
            const double f = ri[k] * rinv;
            for (int j = k + 1 + lane; j <= cend; j += 32) ri[j] -= f * rk[j];
        }
        __syncthreads();
    }
    if (bad) { if (tid == 0) ekf_report(a, 1.0 /*NOT_COMPUTED*/, 0.0, 1.0); return; }

    // ---- phase 5: scale row k by d_k^-1/2 (Z = D^-1/2 L^-1 [HP | v]); chi2 = noiseScale |z_v|^2 (ekf.cpp:815)
    for (int k = wrp; k < n; k += nwarps) {
        const double sc = 1.0 / sqrt(T[(size_t)k * W + k]);
        double* rk = T + (size_t)k * W;
        for (int j = n + lane; j <= cend; j += 32) rk[j] *= sc;
    }
    __syncthreads();
    if (tid == 0) {
        double t = 0.0; for (int k = 0; k < n; k++) { const double z = T[(size_t)k * W + cv]; t += z * z; }
        s_scalar[1] = a.noiseScale * t;
    }
    __syncthreads();
    const double chi2 = s_scalar[1];
    if (checking) {
        const bool outlier = !a.skipChi2 && chi2 > a.chi2Thr;
        if (tid == 0) ekf_report(a, outlier ? 3.0 : 0.0, chi2, 0.0);
        if (outlier || a.mode == EKF_MODE_CHECK) return;
    } else if (tid == 0) ekf_report(a, 0.0, chi2, 0.0);

    // ---- phase 6: m += Z' z_v;  P -= Z' Z  (lower 4x4 blocks, mirrored)
    for (int i = tid; i < N; i += EKF_NT) {
        double s = 0.0;
        for (int k = 0; k < n; k++) s += T[(size_t)k * W + n + i] * T[(size_t)k * W + cv];
        m[i] += s;
    }
    {
        const int nb = (N + 3) >> 2, nblk = nb * (nb + 1) / 2;
        for (int t = tid; t < nblk; t += EKF_NT) {
            // t -> (bj, bi), bi >= bj, column-major enumeration of the lower triangle of blocks
            int bj = (int)floor(((2.0 * nb + 1.0) - sqrt((2.0 * nb + 1.0) * (2.0 * nb + 1.0) - 8.0 * t)) * 0.5);
            while (bj > 0 && bj * nb - bj * (bj - 1) / 2 > t) --bj;
            while ((bj + 1) * nb - (bj + 1) * bj / 2 <= t) ++bj;
            const int bi = bj + (t - (bj * nb - bj * (bj - 1) / 2));
            const int i0 = bi * 4, j0 = bj * 4;
            double acc[4][4];
#pragma unroll
            for (int x = 0; x < 4; x++)
#pragma unroll
                for (int y = 0; y < 4; y++) acc[x][y] = 0.0;
            const double* zi = T + n + i0;
            const double* zj = T + n + j0;
            for (int k = 0; k < n; k++) {
                double av[4], bv[4];
#pragma unroll
                for (int x = 0; x < 4; x++) { av[x] = zi[min(x, N - 1 - i0)]; bv[x] = zj[min(x, N - 1 - j0)]; }
#pragma unroll
                for (int x = 0; x < 4; x++)
#pragma unroll
                    for (int y = 0; y < 4; y++) acc[x][y] += av[x] * bv[y];
                zi += W; zj += W;
            }
#pragma unroll
            for (int x = 0; x < 4; x++)
#pragma unroll
                for (int y = 0; y < 4; y++) {
                    const int i = i0 + x, j = j0 + y;
                    if (i < N && j < N) {
                        if (bi != bj) { P[i + (size_t)j * N] -= acc[x][y]; P[j + (size_t)i * N] -= acc[x][y]; }
                        else if (i >= j) { P[i + (size_t)j * N] -= acc[x][y]; if (i != j) P[j + (size_t)i * N] -= acc[x][y]; }
                    }
                }
        }
    }
    __syncthreads();
    if (joseph) {
        // ---- Joseph form of the augmentation (ekf.cpp:35-50, 872): P = T1 G' ... precisely
        //   G = T1 P' = P' - K HP   (just computed in place),   P'' = G T1' + K R K',   T1 = I - K visAugH.
        // T1 differs from I in the 14 columns visAugH touches, so G T1' costs 14 FMAs per entry instead of N.
        // The explicit T1 matters numerically: the new pose slot has T1[new,new] = 1 + K[new,r] ~ P_cur/1e8, and it
        // is this small factor that suppresses the 1e-16 * 1e8 cancellation error of G[new,new] (reference
        // comment ekf.cpp:871 "seems to affect results").
        double* Ks = T + (size_t)n * W;              // N x 7 gain  K = Z' M,  M = D^-1/2 L^-1 (identity block)
        double* T1c = Ks + (size_t)N * EKF_POSE;     // N x 14 non-trivial columns of T1
        for (int t = tid; t < N * EKF_POSE; t += EKF_NT) {
            const int i = t % N, r = t / N;
            double s = 0.0;
            for (int k = 0; k < n; k++) s += T[(size_t)k * W + n + i] * T[(size_t)k * W + cv + 1 + r];
            Ks[t] = s;
        }
        __syncthreads();
        auto special_col = [](int c) { return c < 3 ? EKF_POS + c : c < 7 ? EKF_ORI + c - 3 : EKF_CAM + c - 7; };
        for (int t = tid; t < N * 14; t += EKF_NT) {
            const int j = t % N, c = t / N;
            const double kv = c < 7 ? -Ks[j + c * N] : Ks[j + (c - 7) * N];
            T1c[t] = (j == special_col(c) ? 1.0 : 0.0) + kv;
        }
        __syncthreads();
        const double* G = P;
        double* Pout = a.b.P;                        // the pre-shift buffer is free again
        for (int idx = tid; idx < N * N; idx += EKF_NT) {
            const int i = idx % N, j = idx / N;
            const bool jsp = j < 3 || (j >= EKF_ORI && j < EKF_ORI + 4) || (j >= EKF_CAM && j < EKF_CAM + EKF_POSE);
            double s = jsp ? 0.0 : G[idx];
#pragma unroll
            for (int c = 0; c < 14; c++) s += G[i + (size_t)special_col(c) * N] * T1c[j + c * N];
            double kr = 0.0;
#pragma unroll
            for (int r = 0; r < EKF_POSE; r++) kr += Ks[i + r * N] * (a.Rdiag * Ks[j + r * N]);
            Pout[idx] = s + kr;
        }
        __syncthreads();
        P = Pout;
    }
    // ---- phase 7: quaternion normalisation (updateCommon: current only; visual/augment: all) and optional
    //      maintainPositiveSemiDefinite
    normalize_all(m, a.b.trail, !a.normalizeAll);
    if (a.symmetrize) symmetrize(P, N);
}

// ------------------------------------------------------------------------------------------------ predict
#ifdef HV_EKF_TIMING
#define PMARK(i) do { if (threadIdx.x == 0) { unsigned long long t_; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_)); a.b.res[8 + (i)] = (double)t_; } } while (0)
#else
#define PMARK(i) do { } while (0)
#endif
// predict() for `count` consecutive IMU samples in ONE launch (ekf.cpp:320-514 applied count times, with the
// normalizeQuaternions(true) calls that follow them): see ekf_predict.cuh.
#define EKF_PMARK(i) PMARK(i)
#include "ekf_predict.cuh"
__global__ void __launch_bounds__(EKF_NT) ekf_predict_kernel(EkfPredictArgs a)
{
    extern __shared__ __align__(16) double ekf_predict_dyn[];
    ekf_predict_body(a, ekf_predict_dyn);
}
// Group launch (hv_ekf_group_run_device): CTA i runs the IMU burst args[i] of one filter of the group (blocks in device memory)
__global__ void __launch_bounds__(EKF_NT) ekf_group_predict_kernel(const EkfPredictArgs* __restrict__ args)
{
    extern __shared__ __align__(16) double ekf_predict_dyn[];
    ekf_predict_body(args[blockIdx.x], ekf_predict_dyn);
}

// ------------------------------------------------------------------------------------------------ elementwise / structural
__device__ __forceinline__ void quat_to_rot(const double* q /*w,x,y,z*/, double* R /*row-major*/)
{
    // Eigen::Quaternion::toRotationMatrix
    const double tx = 2 * q[1], ty = 2 * q[2], tz = 2 * q[3];
    const double twx = tx * q[0], twy = ty * q[0], twz = tz * q[0];
    const double txx = tx * q[1], txy = ty * q[1], txz = tz * q[1];
    const double tyy = ty * q[2], tyz = tz * q[2], tzz = tz * q[3];
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
    R[3] = txy + twz; R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1 - (txx + tyy);
}

// block structure of trailRotationA (ekf.cpp:740-748): returns block start and kind (0 identity, 1 3x3 p, 2 4x4 q)
__device__ __forceinline__ void xform_block(int i, int poseTrailDim, int& start, int& kind)
{
    if (i < 3) { start = 0; kind = 1; }
    else if (i < 6) { start = 3; kind = 1; }
    else if (i < 10) { start = 6; kind = 2; }
    else if (i < EKF_CAM || i >= poseTrailDim) { start = i; kind = 0; }
    else {
        const int p = (i - EKF_CAM) / EKF_POSE, o = (i - EKF_CAM) % EKF_POSE, base = EKF_CAM + p * EKF_POSE;
        if (o < 3) { start = base; kind = 1; } else { start = base + 3; kind = 2; }
    }
}

__global__ void __launch_bounds__(EKF_NT) ekf_ew_kernel(EkfEwArgs a)
{
    const int tid = threadIdx.x, N = a.b.N;
    double* m = a.b.m; double* P = a.b.P;
    const int poseTrailDim = N - a.b.mapDim;
    switch (a.op) {
    case EKF_EW_SYMMETRIZE: symmetrize(P, N); break;
    case EKF_EW_NORMALIZE: normalize_all(m, a.b.trail, a.ival0 != 0); break;
    case EKF_EW_UNAUGMENT:
        shift_state(P, a.b.P2, m, N, [poseTrailDim](int i) { return unaug_src(i, poseTrailDim); });
        break;
    case EKF_EW_TRANSLATE: {   // ekf.cpp:696-702
        double d[3];
        for (int k = 0; k < 3; k++) d[k] = a.dval[k] - m[EKF_POS + k];
        __syncthreads();
        for (int p = tid; p <= a.b.trail; p += EKF_NT)
            for (int k = 0; k < 3; k++) m[(p == 0 ? EKF_POS : EKF_CAM + EKF_POSE * (p - 1)) + k] += d[k];
    } break;
    case EKF_EW_INIT_ORIENTATION:   // ekf.cpp:305-316
        if (tid < 4) m[EKF_ORI + tid] = a.dval[tid];
        if (tid < 16) { const int i = tid % 4, j = tid / 4; P[EKF_ORI + i + (size_t)(EKF_ORI + j) * N] = (i == j && i < 3) ? a.dval[4] : 0.0; }
        break;
    case EKF_EW_INSERT_MAP_POINT: {   // ekf.cpp:911-921
        const int off = a.ival0;
        for (int idx = tid; idx < 3 * N; idx += EKF_NT) {
            const int k = idx / N, j = idx % N;
            P[off + k + (size_t)j * N] = 0.0; P[j + (size_t)(off + k) * N] = 0.0;
        }
        __syncthreads();
        if (tid < 3) { P[(off + tid) * (size_t)(N + 1)] = 1e3 * 1e3; m[off + tid] = a.dval[tid]; }
    } break;
    case EKF_EW_LOCK_BIASES:   // ekf.cpp:944-947
        for (int idx = tid; idx < 9 * N; idx += EKF_NT) {
            const int k = idx / N, j = idx % N;
            P[EKF_BGA + k + (size_t)j * N] = 0.0; P[j + (size_t)(EKF_BGA + k) * N] = 0.0;
        }
        break;
    }
}

// rare, heavier structural operations (kept out of ekf_ew_kernel so that the per-frame ones stay lean)
__global__ void __launch_bounds__(EKF_NT) ekf_ew_heavy_kernel(EkfEwArgs a)
{
    __shared__ double s_q[16], s_p[9], s_t[3], s_B[49], s_Binv[49];
    const int tid = threadIdx.x, N = a.b.N;
    double* m = a.b.m; double* P = a.b.P;
    const int poseTrailDim = N - a.b.mapDim;
    switch (a.op) {
    case EKF_EW_CONDITION_LAST_POSE: {   // ekf.cpp:928-942
        const int mm = N - EKF_POSE;
        if (tid < 49) s_B[tid] = P[mm + tid % 7 + (size_t)(mm + tid / 7) * N];
        __syncthreads();
        if (tid == 0) {   // 7x7 inverse, Gauss-Jordan with partial pivoting (Eigen: PartialPivLU for sizes > 4)
            double M[7][14];
            for (int i = 0; i < 7; i++) for (int j = 0; j < 7; j++) { M[i][j] = s_B[i + j * 7]; M[i][7 + j] = i == j ? 1.0 : 0.0; }
            for (int c = 0; c < 7; c++) {
                int p = c; for (int r = c + 1; r < 7; r++) if (fabs(M[r][c]) > fabs(M[p][c])) p = r;
                if (p != c) for (int j = 0; j < 14; j++) { const double t = M[c][j]; M[c][j] = M[p][j]; M[p][j] = t; }
                const double inv = 1.0 / M[c][c];
                for (int j = 0; j < 14; j++) M[c][j] *= inv;
                for (int r = 0; r < 7; r++) if (r != c) { const double f = M[r][c]; for (int j = 0; j < 14; j++) M[r][j] -= f * M[c][j]; }
            }
            for (int i = 0; i < 7; i++) for (int j = 0; j < 7; j++) s_Binv[i + j * 7] = M[i][7 + j];
        }
        __syncthreads();
        double* Tm = a.b.work;   // mm x 7: P[0:mm, mm:] * Binv
        for (int idx = tid; idx < mm * 7; idx += EKF_NT) {
            const int i = idx % mm, k = idx / mm;
            double s = 0; for (int r = 0; r < 7; r++) s += P[i + (size_t)(mm + r) * N] * s_Binv[r + k * 7];
            Tm[idx] = s;
        }
        __syncthreads();
        for (int idx = tid; idx < mm * mm; idx += EKF_NT) {
            const int i = idx % mm, j = idx / mm;
            double s = 0; for (int k = 0; k < 7; k++) s += Tm[i + k * mm] * P[mm + k + (size_t)j * N];
            P[i + (size_t)j * N] -= s;
        }
        __syncthreads();
        for (int idx = tid; idx < mm * 7; idx += EKF_NT) {
            const int i = idx % mm, k = idx / mm;
            P[i + (size_t)(mm + k) * N] = 0.0; P[mm + k + (size_t)i * N] = 0.0;
        }
        if (tid < 49) P[mm + tid % 7 + (size_t)(mm + tid / 7) * N] = (tid % 7 == tid / 7) ? 1e3 * 1e3 : 0.0;
    } break;
    case EKF_EW_TRANSFORM: {   // ekf.cpp:704-758, out of place into P2
        if (tid == 0) {
            const int pi = a.ival0;
            const double* q0 = pi < 0 ? m + EKF_ORI : m + EKF_CAM + EKF_POSE * pi + 3;
            const double* rp = pi < 0 ? m + EKF_POS : m + EKF_CAM + EKF_POSE * pi;
            const double* q1 = a.dval + 3;
            // qChange = conj(q0) * q1  (Hamilton product, components w,x,y,z)
            const double aw = q0[0], ax = -q0[1], ay = -q0[2], az = -q0[3];
            const double bw = q1[0], bx = q1[1], by = q1[2], bz = q1[3];
            double qc[4] = {aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                            aw * by + ay * bw + az * bx - ax * bz, aw * bz + az * bw + ax * by - ay * bx};
            const double p1 = qc[0], p2 = qc[1], p3 = qc[2], p4 = qc[3];
            const double Qm[16] = {p1, -p2, -p3, -p4, p2, p1, p4, -p3, p3, -p4, p1, p2, p4, p3, -p2, p1};   // row-major
            for (int i = 0; i < 16; i++) s_q[i] = Qm[i];
            double R[9]; quat_to_rot(qc, R);
            for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) s_p[i * 3 + j] = R[j * 3 + i];      // transpose
            for (int i = 0; i < 3; i++) s_t[i] = a.dval[i] - (s_p[i * 3] * rp[0] + s_p[i * 3 + 1] * rp[1] + s_p[i * 3 + 2] * rp[2]);
        }
        __syncthreads();
        auto Tel = [&](int i, int start, int kind, int c) -> double {   // trailRotationA(i, start + c)
            return kind == 1 ? s_p[(i - start) * 3 + c] : kind == 2 ? s_q[(i - start) * 4 + c] : 1.0;
        };
        for (int idx = tid; idx < N * N; idx += EKF_NT) {
            const int i = idx % N, j = idx / N;
            int si, ki, sj, kj;
            xform_block(i, poseTrailDim, si, ki); xform_block(j, poseTrailDim, sj, kj);
            const int ni = ki == 0 ? 1 : ki + 2, nj = kj == 0 ? 1 : kj + 2;
            double s = 0;
            for (int x = 0; x < ni; x++) {
                double r = 0;
                for (int y = 0; y < nj; y++) r += P[si + x + (size_t)(sj + y) * N] * Tel(j, sj, kj, y);
                s += Tel(i, si, ki, x) * r;
            }
            a.b.P2[idx] = s;
        }
        double tmp[4];
#pragma unroll
        for (int r = 0; r < 4; r++) {
            const int i = tid + r * EKF_NT;
            if (i < N) {
                int si, ki; xform_block(i, poseTrailDim, si, ki);
                const int ni = ki == 0 ? 1 : ki + 2;
                double s = 0; for (int x = 0; x < ni; x++) s += Tel(i, si, ki, x) * m[si + x];
                tmp[r] = s;
            }
        }
        __syncthreads();
#pragma unroll
        for (int r = 0; r < 4; r++) { const int i = tid + r * EKF_NT; if (i < N) m[i] = tmp[r]; }
        __syncthreads();
        // translateTo(position() + translation)
        double d[3];
        for (int k = 0; k < 3; k++) d[k] = (m[EKF_POS + k] + s_t[k]) - m[EKF_POS + k];
        __syncthreads();
        for (int p = tid; p <= a.b.trail; p += EKF_NT)
            for (int k = 0; k < 3; k++) m[(p == 0 ? EKF_POS : EKF_CAM + EKF_POSE * (p - 1)) + k] += d[k];
    } break;
    }
}

// ------------------------------------------------------------------------------------------------ launch
static size_t ekf_update_smem_bytes(int n, int N) { return (size_t)n * (size_t)((n + N + 1) | 1) * sizeof(double); }
static size_t ekf_augment_smem_bytes(int N)
{
    const int n = EKF_POSE;
    return ((size_t)n * (size_t)((n + N + 1 + n) | 1) + (size_t)N * 21) * sizeof(double);
}

cudaError_t ekf_launch_update(const EkfUpdateArgs& args, cudaStream_t s)
{
    // 8-CTA cluster kernel (ekf_cluster2.cuh) whenever its shared-memory working set fits (n <= 84 at N = 160); the single-CTA
    // kernel below only for oversized measurements (batch updates with n up to N, tableau in global memory above 200 KB).
    // (rowChunk > 0: the row-chunked form of the cluster kernel, chosen by the caller for a measurement that does not fit it whole)
    if (args.rowChunk > 0 || ekf_cluster2_fits(args.n, args.l, args.b.N, args.op == EKF_OP_AUGMENT)) return ekf_launch_update_cluster2(args, s);
    static bool seen[64];                             // per device: function attributes belong to the device's context
    if (hv_first_use_on_device(seen)) {
        cudaError_t e = cudaFuncSetAttribute(ekf_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
        if (e != cudaSuccess) return e;
    }
    EkfUpdateArgs a = args;
    size_t smem;
    if (a.op == EKF_OP_AUGMENT) { a.useGlobalWork = 0; smem = ekf_augment_smem_bytes(a.b.N); }
    else {
        smem = ekf_update_smem_bytes(a.n, a.b.N);
        a.useGlobalWork = smem > 200 * 1024 ? 1 : 0;
        if (a.useGlobalWork) smem = 0;
    }
    ekf_update_kernel<<<1, EKF_NT, smem, s>>>(a);
    return cudaGetLastError();
}
cudaError_t ekf_launch_predict(const EkfPredictArgs& a, cudaStream_t s)
{
    static bool seen[64];
    if (hv_first_use_on_device(seen)) {
        cudaError_t e = cudaFuncSetAttribute(ekf_predict_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ekf_predict_smem_bytes(EKF_MAX_PREDICT));
        if (e != cudaSuccess) return e;
    }
    // programmatic dependent launch (see ekf_cluster2.cu): the kernel may be scheduled while its predecessor on the stream still runs; it
    // waits in griddepcontrol.wait before it reads the state. HV_EKF_NO_PDL=1 switches it off.
    static const bool pdl = getenv("HV_EKF_NO_PDL") == nullptr;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(1); cfg.blockDim = dim3(EKF_NT); cfg.dynamicSmemBytes = ekf_predict_smem_bytes(a.count); cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, ekf_predict_kernel, a);
}
cudaError_t ekf_launch_group_predict(const EkfPredictArgs* hArgs, const EkfPredictArgs* dArgs, int count, cudaStream_t s)
{
    static bool seen[64];
    if (hv_first_use_on_device(seen)) {
        cudaError_t e = cudaFuncSetAttribute(ekf_group_predict_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ekf_predict_smem_bytes(EKF_MAX_PREDICT));
        if (e != cudaSuccess) return e;
    }
    int maxCount = 0;
    for (int i = 0; i < count; i++) if (hArgs[i].count > maxCount) maxCount = hArgs[i].count;
    static const bool pdl = getenv("HV_EKF_NO_PDL") == nullptr;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(count); cfg.blockDim = dim3(EKF_NT); cfg.dynamicSmemBytes = ekf_predict_smem_bytes(maxCount); cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, ekf_group_predict_kernel, dArgs);
}
cudaError_t ekf_launch_elementwise(const EkfEwArgs& a, cudaStream_t s)
{
    if (a.op == EKF_EW_CONDITION_LAST_POSE || a.op == EKF_EW_TRANSFORM) ekf_ew_heavy_kernel<<<1, EKF_NT, 0, s>>>(a);
    else {
        // purely elementwise N x N passes are spread over several SMs (they are L2-latency bound on one)
        int grid = 1;
        if (a.op == EKF_EW_SYMMETRIZE || a.op == EKF_EW_UNAUGMENT) { grid = (a.b.N * a.b.N + 4 * EKF_NT - 1) / (4 * EKF_NT); if (grid > 32) grid = 32; }
        ekf_ew_kernel<<<grid, EKF_NT, 0, s>>>(a);
    }
    return cudaGetLastError();
}
