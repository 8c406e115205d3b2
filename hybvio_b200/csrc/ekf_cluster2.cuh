// hybvio_b200/csrc/ekf_cluster2.cuh -- body of the Kalman update / outlier check / pose augmentation kernel (cluster of 8
// CTAs, fp64): second generation of ekf_cluster.cu. Same reference functions (src/odometry/ekf.cpp:57-82, 573-677,
// 760-844, 848-885, 35-50) and the same algebra (elimination tableau [S | HP | v], Z = D^-1/2 L^-1 HP, P -= Z'Z, Joseph
// form with the explicit 14-column T1); what changed is where the data lives and how the CTAs talk:
//
//   * CTA c owns the column block J_c of P and keeps ALL of it (N x B) in shared memory from the first load to the
//     final store: P is read once and written once per update (the first generation re-read it for the downdate);
//   * small exchanges between CTAs go through DISTRIBUTED SHARED MEMORY (cluster.map_shared_rank) instead of a
//     write -> cluster barrier -> read round trip through L2:
//       - innovation covariance: when S is small (n*n <= 1024) every CTA leaves its partial S in shared memory and, after
//         one cluster barrier, sums all of them itself in a fixed order (bitwise identical in every CTA); a larger S goes
//         through L2 (partial slices -> reduced slices -> every CTA);
//       - small Z slices are gathered straight out of the neighbours' tableaus (a large Z goes through L2);
//       - symmetrisation sends every entry to the owner of its mirror image; the Joseph form reads the 14 special columns
//         of G from the CTAs that own them;
//   * the augmentation builds its shifted block A P A' + Q while loading (no P2 pass, no barrier), and a deferred
//     maintainPositiveSemiDefinite() is applied in the same pass (EkfUpdateArgs::symFirst);
//   * the state mean is staged in shared memory; CTA 0 writes it back once.
//
// Decisions (chi2 / RMSE / pivot sign) are computed redundantly from identical data in identical order, so that every
// CTA takes the same branch; every path that leaves the kernel after the first exposure of shared memory to the
// neighbours passes a final cluster barrier (a CTA must not exit while its shared memory may still be read).
//
// Written against the primitives tests/emu can run on the host (tests/emu/emu_update.cpp runs this body against the C
// oracle without a GPU).
#pragma once
#include "ekf.cuh"
#include "hv_dmma.cuh"

#define EK2_NT 512
#define EK2_C 8                       // CTAs per cluster (the portable maximum)
#define EK2_MAXN 768
#ifndef EK2_PHASE
#define EK2_PHASE(i) do { } while (0)
#endif
#ifndef EK2_ELIM_MARK                 // tools/ubench_elim2.cu: cycle stamps inside the blocked elimination
#define EK2_ELIM_MARK(i) do { } while (0)
#define EK2_ELIM_DECL
#endif

struct Ek2Geom { int B, X, W, T, PB, RS, EXTRA, SYM, oneStage, LD; };
__host__ __device__ inline int ek2_pad4mod16(int w) { return w + ((20 - (w & 15)) & 15); }
__host__ __device__ inline Ek2Geom ek2_geom(int n, int l, int N, bool joseph)
{
    Ek2Geom g;
    g.B = (N + EK2_C - 1) / EK2_C;
    // Leading dimension of the P block and of the gathered Z: = 4 (mod 16) doubles, so that the DMMA fragment loads (8
    // consecutive + 4 strided elements per half-warp) touch 16 distinct 8-byte banks
    // (never N itself: column N of the gathered Z holds z_v for the CTA that updates the state mean)
    g.LD = N + (((20 - (N & 15)) & 15) ? ((20 - (N & 15)) & 15) : 16);
    g.X = n * (l > g.LD ? l : g.LD);                        // H (n x l, ld n), later the gathered Z (n x N, ld LD)
    // tableau row [S | HP_J | v | (I)], padded to = 4 (mod 16) doubles like LD: every fragment load of the products that read the
    // tableau (8 rows x 4 consecutive columns, or 4 rows x 8 columns, per half-warp) then touches 16 distinct 8-byte banks. Round 1
    // used an odd width: 2- to 3-way conflicts, and the partial S product (A operand = the HP part of the tableau) ran at a third
    // of the tensor rate (tools/ubench_gemm.cu)
    g.W = ek2_pad4mod16(n + g.B + 1 + (joseph ? n : 0));
    g.T = (n * g.W + 1) & ~1;                               // even: the P block behind the tableau starts on a 16-byte boundary (bulk copies)
    g.PB = g.LD * g.B;                                      // own column block of P, ld LD
    const int MTn = (n + 7) >> 3;
    const int E = (64 * (MTn * (MTn + 1) / 2) + EK2_C - 1) / EK2_C;   // two-stage: a slice of the upper-triangular 8 x 8 tiles of S
    // small S: every CTA leaves its partial in RS and sums all of them itself; a large S goes through L2 and leaves RS unused
    g.oneStage = n * n <= 1024 ? 1 : 0;
    g.RS = g.oneStage ? n * n : E;                          // (E unused; dropping it would move the cluster / single-CTA boundary, untimed)
    g.EXTRA = joseph ? N * EKF_POSE + 2 * 21 * g.LD + N * g.B : 0;   // K | [G special | K] | [T1c | R K] | P'' block
    // transposition buffer of the symmetrisation: present for every op that sets `symmetrize` (position 3 rows, zero height 1,
    // orientation 4, augmentation 7), so the kernel needs no other way to reach the mirrored entries
    g.SYM = n <= 8 ? N * g.B : 0;
    return g;
}
__host__ __device__ inline size_t ek2_smem_bytes(int n, int l, int N, bool joseph)
{
    const Ek2Geom g = ek2_geom(n, l, N, joseph);
    return ((size_t)g.X + g.T + g.PB + g.RS + g.EXTRA + g.SYM) * sizeof(double);
}
// Row-chunked form of a dense visual op (EkfUpdateArgs::rowChunk): the buffers of an h-row measurement, no symmetrisation buffer
// (a visual update does not symmetrise), and EXTRA = the accumulated mean change m_cur - m_0 (N) and the whole residual v (n)
#define EK2_MIN_CHUNK 8               // one pivot block: a lower chunk height costs as much per pass
__host__ __device__ inline Ek2Geom ek2_geom_chunked(int h, int n, int l, int N)
{
    Ek2Geom g = ek2_geom(h, l, N, false);
    g.SYM = 0;
    g.EXTRA = (N + n + 1) & ~1;
    return g;
}
__host__ __device__ inline size_t ek2_smem_bytes_chunked(int h, int n, int l, int N)
{
    const Ek2Geom g = ek2_geom_chunked(h, n, l, N);
    return ((size_t)g.X + g.T + g.PB + g.RS + g.EXTRA) * sizeof(double);
}

__device__ __forceinline__ void ek2_copy8(double* __restrict__ dst, const double* __restrict__ src, int count, int tid)
{
    for (int base = 0; base < count; base += 8 * EK2_NT) {
        double r[8];
#pragma unroll
        for (int u = 0; u < 8; u++) { const int i = base + u * EK2_NT + tid; r[u] = i < count ? src[i] : 0.0; }
#pragma unroll
        for (int u = 0; u < 8; u++) { const int i = base + u * EK2_NT + tid; if (i < count) dst[i] = r[u]; }
    }
}
__device__ __forceinline__ void ek2_normalize_quat(double* q)
{
    const double z = (q[0] * q[0] + q[2] * q[2]) + (q[1] * q[1] + q[3] * q[3]);
    if (z > 0.0) { const double nrm = sqrt(z); q[0] /= nrm; q[1] /= nrm; q[2] /= nrm; q[3] /= nrm; }
}
__device__ __forceinline__ int ek2_aug_src(int i, int drop)
{
    if (i < EKF_CAM) return i;
    if (i < EKF_CAM + EKF_POSE) return -1;
    if (i < EKF_CAM + (drop + 1) * EKF_POSE) return i - EKF_POSE;
    return i;
}
__device__ __forceinline__ int ek2_special_col(int c) { return c < 3 ? EKF_POS + c : c < 7 ? EKF_ORI + c - 3 : EKF_CAM + c - 7; }
// Entry (i, j) of the shifted covariance the augmentation starts from, A P A' + visAugQ (ekf.cpp:853-857), with the deferred
// maintainPositiveSemiDefinite() (ekf.cpp:1059-1067) evaluated while the shift reads P (the mirror entries are a column apart each;
// reading them in a second, coalesced pass over the block costs a second pass). Shared by ek2_body and ek2_aug_mean_cta, which must
// see the same bits.
__device__ __forceinline__ double ek2_aug_entry(const EkfUpdateArgs& a, int i, int j)
{
    const double* const P = a.b.P;
    const int N = a.b.N;
    const int si = ek2_aug_src(i, a.dropIdx), sj = ek2_aug_src(j, a.dropIdx);
    double v = (si < 0 || sj < 0) ? 0.0 : P[si + (size_t)sj * N];
    if (a.symFirst && si >= 0 && sj >= 0 && si != sj) v = 0.5 * (v + P[sj + (size_t)si * N]);
    if (i == j && i >= EKF_CAM && i < EKF_CAM + EKF_POSE) v += (i - EKF_CAM) < 3 ? a.augNoisePos : a.augNoiseOri;
    return v;
}

// C(M x Nn) = cinit + A(M x K) B(K x Nn) on the fp64 tensor cores, 8 x 8 tiles dealt to the 16 warps, up to EK2_NI tiles
// of a warp advance together through k (independent DMMA chains, operands of step k+1 loaded while step k multiplies).
// fa(m, k) / fb(k, n) are called with indices CLAMPED into the matrix (so every load is unconditional and in bounds: no
// branches between the loads, which would serialise them behind the warp-synchronous MMAs); contributions of k >= K are
// zeroed with a select, rows / columns beyond the matrix produce values that are never stored. cinit(m, n) gives the
// initial value, store(m, n, v0, v1) receives C(m, n), C(m, n + 1) for m < M, n < Nn (n even).
#define EK2_NI 4
// Upper-triangular tile list of a symmetric matrix (column-tile major): tu = nt (nt + 1) / 2 + mt, mt <= nt
__host__ __device__ inline void ek2_upper_tile(int tu, int& mt, int& nt)
{
    nt = (int)((sqrtf(8.0f * (float)tu + 1.0f) - 1.0f) * 0.5f);
    while ((nt + 1) * (nt + 2) / 2 <= tu) nt++;
    while (nt * (nt + 1) / 2 > tu) nt--;
    mt = tu - nt * (nt + 1) / 2;
}
// UPPER: C is symmetric (M == Nn) and only its tiles on or above the diagonal are computed and stored.
// Operands are AFFINE views of shared memory, A(m, k) = A[m sAm + k sAk], B(k, n) = B[k sBk + n sBn]: a k-step of a tile is
// two loads off running pointers and one DMMA -- with only 256 FMAs per MMA the instruction count around it decides the
// speed (the first version took its operands through index-clamping lambdas: ~15 instructions per MMA, and was issue-bound
// at a third of the tensor-core rate).
// One chunk of NI tiles of one warp (NI is exact: no padded tiles -- the kernel is bound by the tensor-core rate, 64 FMA per
// clock per SM, so a padded slot costs as much as a real one)
template <int NI, bool UPPER, class FCI, class FST>
__device__ __forceinline__ void ek2_dmma_chunk(int M, int Nn, int K, int MT, int base, int stride, int lane, const double* A, int sAm, int sAk,
                                               const double* B, int sBk, int sBn, FCI cinit, FST store)
{
    const int g8 = lane >> 2, t4 = lane & 3;
    const int KF = K >> 2, tail = K & 3;                                  // full k-steps, leftover k's
    const int dA = 4 * sAk, dB = 4 * sBk;
    double c0[NI], c1[NI];
    int row[NI], col[NI];
    const double* pa[NI]; const double* pb[NI];
#pragma unroll
    for (int q = 0; q < NI; q++) {
        const int tl = base + q * stride;
        int mt, nt;
        if (UPPER) ek2_upper_tile(tl, mt, nt); else { mt = tl % MT; nt = tl / MT; }
        row[q] = mt * 8 + g8; col[q] = nt * 8 + 2 * t4;
        const int rowc = min(row[q], M - 1), colbc = min(nt * 8 + g8, Nn - 1);   // rows / columns past the matrix: clamped, never stored
        pa[q] = A + (size_t)rowc * sAm + (size_t)t4 * sAk;
        pb[q] = B + (size_t)t4 * sBk + (size_t)colbc * sBn;
        c0[q] = cinit(rowc, min(col[q], Nn - 1)); c1[q] = cinit(rowc, min(col[q] + 1, Nn - 1));
    }
    int kt = 0;
    for (; kt + 2 <= KF; kt += 2) {
        double a0[NI], b0[NI], a1[NI], b1[NI];
#pragma unroll
        for (int q = 0; q < NI; q++) { a0[q] = pa[q][0]; b0[q] = pb[q][0]; a1[q] = pa[q][dA]; b1[q] = pb[q][dB]; pa[q] += 2 * dA; pb[q] += 2 * dB; }
#pragma unroll
        for (int q = 0; q < NI; q++) hv_dmma(c0[q], c1[q], a0[q], b0[q]);
#pragma unroll
        for (int q = 0; q < NI; q++) hv_dmma(c0[q], c1[q], a1[q], b1[q]);
    }
    if (kt < KF) {
        double a0[NI], b0[NI];
#pragma unroll
        for (int q = 0; q < NI; q++) { a0[q] = pa[q][0]; b0[q] = pb[q][0]; pa[q] += dA; pb[q] += dB; }
#pragma unroll
        for (int q = 0; q < NI; q++) hv_dmma(c0[q], c1[q], a0[q], b0[q]);
    }
    if (tail) {                                                           // k = 4 KF + t4 is valid for t4 < tail: others re-read k = 4 KF, zeroed
        const bool kv = t4 < tail;
        double a0[NI], b0[NI];
#pragma unroll
        for (int q = 0; q < NI; q++) {
            const double xa = kv ? pa[q][0] : pa[q][-(ptrdiff_t)t4 * sAk];
            a0[q] = kv ? xa : 0.0;
            b0[q] = kv ? pb[q][0] : pb[q][-(ptrdiff_t)t4 * sBk];
        }
#pragma unroll
        for (int q = 0; q < NI; q++) hv_dmma(c0[q], c1[q], a0[q], b0[q]);
    }
    __syncwarp();                                     // (a product in place: lanes with clamped indices have read what other lanes store)
#pragma unroll
    for (int q = 0; q < NI; q++)
        if (row[q] < M && col[q] < Nn) store(row[q], col[q], c0[q], c1[q]);
}

template <bool UPPER = false, class FCI, class FST>
__device__ __forceinline__ void ek2_dmma_gemm(int M, int Nn, int K, int wrp, int lane, const double* A, int sAm, int sAk,
                                              const double* B, int sBk, int sBn, FCI cinit, FST store)
{
    const int MT = (M + 7) >> 3, NT = (Nn + 7) >> 3, tiles = UPPER ? MT * (MT + 1) / 2 : MT * NT;
    const int nwarps = EK2_NT / 32;
    if (M <= 0 || Nn <= 0) return;
    for (int base = wrp; base < tiles; base += nwarps * EK2_NI) {
        const int cnt = min(EK2_NI, (tiles - base + nwarps - 1) / nwarps);      // tiles of this warp in this chunk (warp-uniform)
        switch (cnt) {
            case 1: ek2_dmma_chunk<1, UPPER>(M, Nn, K, MT, base, nwarps, lane, A, sAm, sAk, B, sBk, sBn, cinit, store); break;
            case 2: ek2_dmma_chunk<2, UPPER>(M, Nn, K, MT, base, nwarps, lane, A, sAm, sAk, B, sBk, sBn, cinit, store); break;
            case 3: ek2_dmma_chunk<3, UPPER>(M, Nn, K, MT, base, nwarps, lane, A, sAm, sAk, B, sBk, sBn, cinit, store); break;
            default: ek2_dmma_chunk<4, UPPER>(M, Nn, K, MT, base, nwarps, lane, A, sAm, sAk, B, sBk, sBn, cinit, store); break;
        }
    }
}

// ---- blocked forward elimination ------------------------------------------------------------------------------------------------
// (tools/ubench_elim2.cu can substitute an experimental version: -DEK2_ELIM_OVERRIDE='"file"'; tools/elim_variants/ holds
// the alternatives)
#ifdef EK2_ELIM_OVERRIDE
#include EK2_ELIM_OVERRIDE
#else
#define EK2_LINV_DOUBLES 128
#define EK2_EB 8                      // pivots per block
// Factorisation of the 8 x 8 diagonal block D = T[r0 .. r0+nb, r0 .. r0+nb] of the current Schur complement by ONE warp with
// shuffles only: lanes 0..7 hold the columns of D (padded with the identity), lanes 8..15 those of I; the row operations
// of the factorisation applied to both leave L_jj' in the first and L_jj^-1 (lower triangular) in the second group, which
// is written to linv (8 x 8, row-major). 8 dependent pivots: the only serial part of the elimination.
// 1 / x to double precision without the slow-path division: hardware approximation + 2 Newton steps, a much shorter
// dependent chain than 1.0 / x (tools/ubench.cu measures both)
__device__ __forceinline__ double ek2_rcp(double x)
{
#ifdef HV_EMU
    return 1.0 / x;
#else
    double r;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
    r = fma(fma(-x, r, 1.0), r, r);
    r = fma(fma(-x, r, 1.0), r, r);
    return r;
#endif
}

__device__ __forceinline__ void ek2_diag_factor(const double* T, int W, int r0, int nb, int lane, double* linv, volatile int* s_bad)
{
    double v[8];
    const int cidx = lane & 7;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const double t = T[(size_t)(r0 + min(i, nb - 1)) * W + r0 + min(cidx, nb - 1)];
        double x = (i == cidx) ? 1.0 : 0.0;
        if (lane < 8 && i < nb && cidx < nb) x = t;
        if (lane >= 16) x = 0.0;
        v[i] = x;
    }
    // Cholesky row operations on [D | I]. Dependent chain per pivot: broadcast a_kk (shuffle) -> rsqrt -> scale (own entry
    // of the pivot row, and the multipliers of the rows below, whose RAW values were shuffled in beforehand: S is symmetric,
    // a_ik = entry i of row k) -> one FMA. Alternatives tools/ubench_elim2.cu can time against it: shuffling the scaled row
    // after the multiply, LDL' with rcp.approx + 2 Newton steps and a final scaling, 2 x 2 pivot blocks with one reciprocal
    // of the determinant per pair.
    bool ok = true;
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const double akk = __shfl_sync(0xffffffffu, v[k], k);
        double raw[8];
#pragma unroll
        for (int i = k + 1; i < 8; i++) raw[i] = __shfl_sync(0xffffffffu, v[k], i);
        if (!(akk > 0.0)) ok = false;
        const double r = rsqrt(akk);
        const double u = v[k] * r;                   // row k of L' (entry of this column)
        v[k] = u;
#pragma unroll
        for (int i = k + 1; i < 8; i++) v[i] = fma(-(raw[i] * r), u, v[i]);
    }
    if (lane >= 8 && lane < 16) {
#pragma unroll
        for (int i = 0; i < 8; i++) linv[i * 8 + (lane - 8)] = v[i];
    }
    if (!ok && lane == 0) *s_bad = 1;
}

// Blocked forward elimination of the tableau T = [ S | Y ] (n rows, columns 0 .. ncols-1, row-major, ld W) in shared
// memory: S = L L' (never pivoted: R > 0 makes S positive definite), Y <- L^-1 Y, by 8-row blocks j:
//   a. all warps: rows of block j <- L_jj^-1 * rows (8 x 8 x 8 DMMA per column tile);
//   b. trailing update T[i, c] -= U_j[:, i]' U_j[:, c] for the rows below, upper triangle of S and all of Y (8 x 8 x 8 DMMA
//      per tile, several tiles of a warp in flight) by warps 1..15, WHILE warp 0 updates the next diagonal tile first and
//      factors it (ek2_diag_factor: look-ahead), so that the serial pivot chain overlaps the bulk work.
// Two barriers per 8 pivots; the first generation (ekf_elim.cuh) needed one barrier per two pivots and kept the tableau
// in registers, which bounded n <= 96. Returns false (uniformly) on a non-positive pivot. s_linv: 2 x 64 doubles.
__device__ __forceinline__ bool ek2_block_eliminate(double* T, int W, int n, int ncols, int wrp, int lane, double* s_linv, volatile int* s_bad)
{
    const int g8 = lane >> 2, t4 = lane & 3;
    const int nwarps = EK2_NT / 32;
    const int MT = (n + 7) >> 3, CT = (ncols + 7) >> 3;
    EK2_ELIM_DECL
    if (wrp == 0) {
        if (lane == 0) *s_bad = 0;
        __syncwarp();
        ek2_diag_factor(T, W, 0, min(8, n), lane, s_linv, s_bad);
    }
    __syncthreads();
    for (int j = 0; j < MT; j++) {
        if (*s_bad) return false;
        const int r0 = 8 * j, nb = min(8, n - r0);
        const double* linv = s_linv + (j & 1) * 64;
        EK2_ELIM_MARK(0);
        // ---- a. rows of the block <- L_jj^-1 * rows, column tiles j .. CT-1 (loads clamped into the tableau: no branches)
        for (int ct = j + wrp; ct < CT; ct += nwarps) {
            double c0 = 0.0, c1 = 0.0;
            const int colbc = min(8 * ct + g8, ncols - 1);
            double bf[2];
#pragma unroll
            for (int kt = 0; kt < 2; kt++) {
                const int k = kt * 4 + t4;
                const double x = T[(size_t)(r0 + min(k, nb - 1)) * W + colbc];
                bf[kt] = k < nb ? x : 0.0;
            }
#pragma unroll
            for (int kt = 0; kt < 2; kt++) hv_dmma(c0, c1, linv[g8 * 8 + kt * 4 + t4], bf[kt]);
            const int col = 8 * ct + 2 * t4;
            __syncwarp();                             // in place: every lane's loads of the tile precede any lane's store (racecheck, session W)
            if (g8 < nb) { if (col < ncols) T[(size_t)(r0 + g8) * W + col] = c0; if (col + 1 < ncols) T[(size_t)(r0 + g8) * W + col + 1] = c1; }
        }
        EK2_ELIM_MARK(1);
        __syncthreads();
        EK2_ELIM_MARK(2);
        // ---- b. trailing update: row tiles mt > j, column tiles nt >= mt (row-major list; entry 0 is the next diagonal tile).
        // Warp 0 takes entry 0 and then factors it; warps 1..15 walk contiguous ranges of the rest, reloading the A
        // fragment (-U_j[:, row tile]') only when the row tile changes.
        if (j + 1 < MT) {
            const int first = j + 1;
            int total = 0;
            for (int mt = first; mt < MT; mt++) total += CT - mt;
            const bool ahead = wrp == 0;
            // Workers: the warps that do NOT share warp 0's scheduler / FP64 pipe (warp id mod 4 != 0). The pivot chain of the
            // look-ahead factorisation is a sequence of dependent fp64 operations; every DMMA a sibling warp queues on the
            // same pipe (16 cycles each) would sit in front of them.
            const int nwork = nwarps - nwarps / 4, widx = wrp - wrp / 4 - 1;           // 12 workers, index 0..11
            const bool worker = (wrp & 3) != 0;
            const int rest = total - 1;
            int lo = ahead ? 0 : worker ? 1 + (int)(((long long)rest * widx) / nwork) : 0;
            const int hi = ahead ? 1 : worker ? 1 + (int)(((long long)rest * (widx + 1)) / nwork) : 0;
            const double* rowk0 = T + (size_t)(r0 + min(t4, nb - 1)) * W;        // k = t4
            const double* rowk1 = T + (size_t)(r0 + min(4 + t4, nb - 1)) * W;    // k = 4 + t4
            const bool k0v = t4 < nb, k1v = 4 + t4 < nb;
            if (ahead) {
                // the next diagonal tile (first, first): A and B fragments are the same column block of U_j
                const int cb = 8 * first, am = min(cb + g8, ncols - 1);
                const double x0 = rowk0[am], x1 = rowk1[am];
                const int rowi = cb + g8, coli = cb + 2 * t4;
                double* crow = T + (size_t)min(rowi, n - 1) * W;
                double c0 = crow[min(coli, ncols - 1)], c1 = crow[min(coli + 1, ncols - 1)];
                hv_dmma(c0, c1, k0v ? -x0 : 0.0, x0);
                hv_dmma(c0, c1, k1v ? -x1 : 0.0, x1);
                __syncwarp();                         // lanes past the last row read CLAMPED elements that other lanes store (values unused)
                if (rowi < n) { if (coli < ncols) crow[coli] = c0; if (coli + 1 < ncols) crow[coli + 1] = c1; }
            } else if (worker) {
                int mt = first, nt, idx = min(lo, total - 1);
                while (idx >= CT - mt) { idx -= CT - mt; mt++; }
                nt = mt + idx;
                int curMt = -1;
                double a0 = 0.0, a1 = 0.0;
                for (; lo < hi; lo++) {
                    if (mt != curMt) {
                        const int am = min(8 * mt + g8, ncols - 1);
                        const double x0 = rowk0[am], x1 = rowk1[am];
                        a0 = k0v ? -x0 : 0.0; a1 = k1v ? -x1 : 0.0;                   // A[m][k] = -U_j[k][8 mt + m]
                        curMt = mt;
                    }
                    const int rowi = 8 * mt + g8, coli = 8 * nt + 2 * t4, bn = min(8 * nt + g8, ncols - 1);
                    double* crow = T + (size_t)min(rowi, n - 1) * W;
                    double c0 = crow[min(coli, ncols - 1)], c1 = crow[min(coli + 1, ncols - 1)];
                    const double b0 = rowk0[bn], b1 = rowk1[bn];                       // B[k][nn] = U_j[k][8 nt + nn]
                    hv_dmma(c0, c1, a0, b0);
                    hv_dmma(c0, c1, a1, b1);
                    __syncwarp();
                    if (rowi < n) { if (coli < ncols) crow[coli] = c0; if (coli + 1 < ncols) crow[coli + 1] = c1; }
                    if (++nt == CT) { mt++; nt = mt; }
                }
            }
            EK2_ELIM_MARK(3);
            if (ahead) {
                __syncwarp();
                ek2_diag_factor(T, W, 8 * first, min(8, n - 8 * first), lane, s_linv + (first & 1) * 64, s_bad);
            }
            EK2_ELIM_MARK(4);
            __syncthreads();
            EK2_ELIM_MARK(5);
        }
    }
    return !*s_bad;
}

#endif

// Programmatic dependent launch (sm_90+): see ek2_body. No-ops on the host emulator.
__device__ __forceinline__ void ek2_pdl_launch_dependents()
{
#ifndef HV_EMU
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
#endif
}
__device__ __forceinline__ void ek2_pdl_wait()
{
#ifndef HV_EMU
    asm volatile("griddepcontrol.wait;" ::: "memory");
#endif
}

// ---- bulk asynchronous copies (TMA, non-tensor form: cp.async.bulk) between global and shared memory, completion on an mbarrier.
// One instruction moves a whole column / row / block: no register staging, no load -> store loop per thread. Addresses and sizes must
// be multiples of 16 bytes (ek2_body checks and keeps the loops otherwise). On the host emulator: memcpy by the issuing thread.
__device__ __forceinline__ void ek2_bar_init(unsigned long long* bar, int count)
{
#ifdef HV_EMU
    *bar = 0; (void)count;
#else
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"((unsigned)__cvta_generic_to_shared(bar)), "r"(count) : "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
#endif
}
__device__ __forceinline__ void ek2_bar_expect(unsigned long long* bar, unsigned bytes)   // one arrival + the bytes it announces (0: plain arrival)
{
#ifdef HV_EMU
    (void)bar; (void)bytes;
#else
    if (bytes) asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"((unsigned)__cvta_generic_to_shared(bar)), "r"(bytes) : "memory");
    else asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"((unsigned)__cvta_generic_to_shared(bar)) : "memory");
#endif
}
__device__ __forceinline__ void ek2_bar_wait(unsigned long long* bar, unsigned phase)
{
#ifdef HV_EMU
    (void)bar; (void)phase;                           // (every use is followed by a barrier of the CTA)
#else
    unsigned done;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"((unsigned)__cvta_generic_to_shared(bar)), "r"(phase) : "memory");
    } while (!done);
#endif
}
__device__ __forceinline__ void ek2_bulk_g2s(double* dst, const double* src, unsigned bytes, unsigned long long* bar)
{
#ifdef HV_EMU
    if ((((size_t)dst) | ((size_t)src) | bytes) & 15) { fprintf(stderr, "emu: misaligned bulk copy (global -> shared)\n"); abort(); }
    memcpy(dst, src, bytes); (void)bar;
#else
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src), "r"(bytes), "r"((unsigned)__cvta_generic_to_shared(bar)) : "memory");
#endif
}
__device__ __forceinline__ void ek2_bulk_s2g(double* dst, const double* src, unsigned bytes)
{
#ifdef HV_EMU
    if ((((size_t)dst) | ((size_t)src) | bytes) & 15) { fprintf(stderr, "emu: misaligned bulk copy (shared -> global)\n"); abort(); }
    memcpy(dst, src, bytes);
#else
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" :: "l"(dst), "r"((unsigned)__cvta_generic_to_shared(src)), "r"(bytes) : "memory");
#endif
}
__device__ __forceinline__ void ek2_bulk_store_done()        // by the thread that issued the stores: committed and complete
{
#ifndef HV_EMU
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
#endif
}
__device__ __forceinline__ void ek2_fence_async_smem()       // generic-proxy writes to shared memory -> visible to the bulk-copy engine
{
#ifndef HV_EMU
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
#endif
}
__device__ __forceinline__ void ek2_fence_async_all()        // ... to global memory (a slice published for the neighbours' bulk reads)
{
#ifndef HV_EMU
    asm volatile("fence.proxy.async;" ::: "memory");
#endif
}

// `Cluster` is cooperative_groups::cluster_group (or the emulator's stand-in). CHUNKS = false compiles the body without the row-chunked
// form (a.rowChunk is ignored): the kernels of the measurements that fit whole keep their code and registers.
template <bool CHUNKS = true, class Cluster>
__device__ __forceinline__ void ek2_body(EkfUpdateArgs& a, double* sm, Cluster cluster)
{
    __shared__ double s_scalar[2];
    __shared__ double s_linv[EK2_LINV_DOUBLES];
    __shared__ int s_bad;
    __shared__ __align__(16) double s_m[EK2_MAXN];
    __shared__ __align__(8) unsigned long long s_bar[4];      // [0] staging (two arrivals: H, then P block + mean), [1] Z gather, [2] / [3] S exchange
    const int c = (int)cluster.block_rank(), C = (int)cluster.num_blocks();      // == EK2_C (as a run-time value: fewer spills)
    const int tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5, nwarps = EK2_NT / 32;
    const int N = a.b.N, n = a.n, l = a.l;
    const bool joseph = a.op == EKF_OP_AUGMENT;
    // Row-chunked form (a.rowChunk > 0, dense visual ops): the rows are processed hc at a time (the last chunk may be lower); every
    // buffer below is sized for hc rows, the P blocks stay resident across the chunks
    const bool chunked = CHUNKS && a.rowChunk > 0;
    const int hc = chunked ? min(a.rowChunk, n) : n;
    const Ek2Geom g = chunked ? ek2_geom_chunked(hc, n, l, N) : ek2_geom(n, l, N, joseph);
    double* X = sm;                 // H, later Z
    double* T = X + g.X;                                // tableau
    double* PB = T + g.T;                               // P[:, J_c]
    double* RS = PB + g.PB;         // partial S (one-stage)
    double* EX = RS + g.RS;         // Joseph-form extras; chunked: m_cur - m_0 (N), then the whole residual (n)
    double* SYMB = EX + g.EXTRA;    // symmetrisation: mirrored entries, transposed
    double* const DM = EX;
    double* const VF = EX + N;
    const int W = g.W, B = g.B, LD = g.LD;
    const int J0 = c * B, Bc = max(0, min(B, N - J0));
    const int vcol = n + B;
    const bool oneStage = g.oneStage != 0;
    // S exchange: entries of the upper-triangular 8 x 8 tiles, tile by tile (ETOT of them per chunk, below). Large S goes through L2 (bulk
    // remote shared-memory pulls run at less than half the L2 rate): a.b.cwork = [ Z (N^2) | reduced S (N^2) | C partial S (8 N^2) ].
    // Precondition: the C partial slices of ETOT entries fit into 8 N^2, C ETOT <= 8 N^2, for every two-stage n <= N <= EK2_MAXN
    // (tests/test_kalman_ref.py checks it).
    double* const Sred = a.b.cwork + (size_t)N * N;
    double* const Spart = a.b.cwork + (size_t)2 * N * N;
    double* const P = a.b.P;

    EK2_PHASE(0);
    // Programmatic dependent launch: the next kernel of the stream may start now (its launch latency and the staging of its
    // own measurement matrix overlap with this kernel); it will not touch the filter state before its own
    // griddepcontrol.wait, which returns when this grid has completed and its writes are visible.
    ek2_pdl_launch_dependents();
    // Bulk copies need 16-byte aligned addresses and sizes: an even state dimension and aligned buffers (ek2_geom keeps the shared-memory
    // side aligned); otherwise the loops below do the same work.
    const bool bulk = (N & 1) == 0 && ((((size_t)P) | ((size_t)a.b.m) | ((size_t)a.b.cwork) | ((size_t)a.specP) | ((size_t)a.specM) | ((size_t)sm)) & 15) == 0;
    const bool bulkH = bulk && !chunked && a.op == EKF_OP_DENSE && ((n * l) & 1) == 0 && (((size_t)a.H) & 15) == 0;
    if (tid == 0) { ek2_bar_init(&s_bar[0], 2); ek2_bar_init(&s_bar[1], 1); ek2_bar_init(&s_bar[2], 1); ek2_bar_init(&s_bar[3], 1); }
    if (bulk) __syncthreads();                        // the barriers exist before anybody waits on them
    // ---- the measurement matrix does not depend on earlier kernels: stage it before waiting for them
    const bool lateH = a.lateH != 0 && a.op == EKF_OP_DENSE;
    if (a.op == EKF_OP_DENSE) {
        if (!lateH && !chunked) {                     // (chunked: the rows of a chunk are staged when it starts)
            if (bulkH) { if (tid == 0) { ek2_bar_expect(&s_bar[0], (unsigned)(n * l * 8)); ek2_bulk_g2s(X, a.H, (unsigned)(n * l * 8), &s_bar[0]); } }
            else ek2_copy8(X, a.H, n * l, tid);
        }
    } else for (int i = tid; i < n * l; i += EK2_NT) X[i] = 0.0;
    ek2_pdl_wait();
    // ---- device-side control flow of a chain issued without host round trips (EkfUpdateArgs): every thread of the cluster
    // reads the same words, written by kernels that have completed
    if (a.gateI || a.gateD || a.counter) {
        bool run = true;
        if (a.gateI && *(volatile const int*)a.gateI != a.gateIExpect) run = false;
        if (a.gateD && *(volatile const double*)a.gateD != a.gateDExpect) run = false;
        if (a.counter && *(volatile const int*)a.counter >= a.counterMax) run = false;
        if (!run) {                                                                        // VuOutlierStatus::NOT_COMPUTED
            if (bulk) {                               // a bulk copy of H may be in flight: complete the staging barrier and wait for it
                const int arrived = (bulkH && !lateH) ? 1 : 0;
                if (tid == 0) for (int q = arrived; q < 2; q++) ek2_bar_expect(&s_bar[0], 0);
                ek2_bar_wait(&s_bar[0], 0);
            }
            if (c == 0 && tid == 0) ekf_report(a, 1.0, 0.0, 0.0);
            return;
        }
    }
    if (lateH && !chunked) {
        if (bulkH) { if (tid == 0) { ek2_bar_expect(&s_bar[0], (unsigned)(n * l * 8)); ek2_bulk_g2s(X, a.H, (unsigned)(n * l * 8), &s_bar[0]); } }
        else ek2_copy8(X, a.H, n * l, tid);
    }
    if (bulk && !bulkH && tid == 0) ek2_bar_expect(&s_bar[0], 0);        // the first of the two arrivals of the staging barrier
    // ---- stage the state mean and the own column block of P (augmentation: of A P A' + visAugQ, ekf.cpp:853-857)
    if (joseph) {
        const int drop = a.dropIdx;
        for (int i = tid; i < N; i += EK2_NT) { const int s = ek2_aug_src(i, drop); s_m[i] = s < 0 ? 0.0 : a.b.m[s]; }
        for (int idx = tid; idx < N * Bc; idx += EK2_NT) {
            const int i = idx % N, j = J0 + idx / N;
            PB[i + (size_t)(idx / N) * LD] = ek2_aug_entry(a, i, j);
        }
        if (bulk && tid == 0) ek2_bar_expect(&s_bar[0], 0);
    } else if (bulk) {
        // one bulk copy per column of the block (N doubles each, into the padded leading dimension) + one for the state mean
        if (wrp == 0) {
            if (lane == 0) ek2_bar_expect(&s_bar[0], (unsigned)((N * Bc + N) * 8));
            __syncwarp();
            for (int j = lane; j < Bc; j += 32) ek2_bulk_g2s(PB + (size_t)j * LD, P + (size_t)(J0 + j) * N, (unsigned)(N * 8), &s_bar[0]);
            if (lane == 31) ek2_bulk_g2s(s_m, a.b.m, (unsigned)(N * 8), &s_bar[0]);
        }
    } else {
        for (int i = tid; i < N; i += EK2_NT) s_m[i] = a.b.m[i];
        // whole columns: one contiguous block of global memory, 8 loads in flight per thread
        const double* src = P + (size_t)J0 * N;
        const int count = N * Bc;
        for (int base = 0; base < count; base += 8 * EK2_NT) {
            double r[8];
#pragma unroll
            for (int u = 0; u < 8; u++) { const int i = base + u * EK2_NT + tid; r[u] = i < count ? src[i] : 0.0; }
#pragma unroll
            for (int u = 0; u < 8; u++) { const int i = base + u * EK2_NT + tid; if (i < count) PB[(i % N) + (size_t)(i / N) * LD] = r[u]; }
        }
    }

    if (bulk) ek2_bar_wait(&s_bar[0], 0);             // H, the P block and the mean have landed
    // ---- measurement model into shared memory (ld = n)
    double hspeed = 0.0;
    if (a.op == EKF_OP_DENSE) {
        __syncthreads();
    } else {
        __syncthreads();                                                  // s_m staged, X zeroed
        if (a.op == EKF_OP_PSEUDO_VELOCITY) {
            hspeed = sqrt(s_m[EKF_VEL] * s_m[EKF_VEL] + s_m[EKF_VEL + 1] * s_m[EKF_VEL + 1]);
            if (hspeed <= 1e-7) return;                                   // ekf.cpp:635-637 (uniform; nothing exposed yet)
        }
        if (tid == 0) {
            switch (a.op) {
                case EKF_OP_ZUPT: for (int i = 0; i < 3; i++) X[i + (EKF_VEL + i) * n] = 1.0; break;
                case EKF_OP_ZRUPT: for (int i = 0; i < 3; i++) X[i + (EKF_BGA + i) * n] = 1.0; break;
                case EKF_OP_PSEUDO_VELOCITY: for (int i = 0; i < 2; i++) X[(EKF_VEL + i) * n] = s_m[EKF_VEL + i] / hspeed; break;
                case EKF_OP_POSITION: for (int i = 0; i < 3; i++) X[i + (EKF_POS + i) * n] = 1.0; break;
                case EKF_OP_ZERO_HEIGHT: X[(EKF_POS + 2) * n] = 1.0; break;
                case EKF_OP_ORIENTATION: for (int i = 0; i < 4; i++) X[i + (EKF_ORI + i) * n] = 1.0; break;
                case EKF_OP_AUGMENT:
                    for (int i = 0; i < 3; i++) { X[i + (EKF_POS + i) * n] = 1.0; X[i + (EKF_CAM + i) * n] = -1.0; }
                    for (int i = 0; i < 4; i++) { X[3 + i + (EKF_ORI + i) * n] = 1.0; X[3 + i + (EKF_CAM + 3 + i) * n] = -1.0; }
                    break;
            }
        }
        __syncthreads();
    }
    const double* Hs = X;

    // residual (identical in every CTA); chunked: all n rows, against the mean m_0 the update starts from
    const double* Hf = chunked ? a.H : Hs;            // (ld n)
    for (int i = tid; i < n; i += EK2_NT) {
        double v;
        if (a.op == EKF_OP_PSEUDO_VELOCITY) v = a.defaultSpeed - hspeed;
        else {
            const double yi = a.y ? a.y[i] : a.ysmall[i];
            double fi = 0.0;
            if (a.f) fi = a.f[i];
            else for (int k = 0; k < l; k++) fi += Hf[i + (size_t)k * n] * s_m[k];
            v = yi - fi;
        }
        if (chunked) VF[i] = v;
        else T[(size_t)i * W + vcol] = v;
    }
    if (joseph) for (int t = tid; t < n * n; t += EK2_NT) T[(size_t)(t / n) * W + vcol + 1 + (t % n)] = (t / n == t % n) ? 1.0 : 0.0;
    __syncthreads();

    const bool checking = a.mode != EKF_MODE_UPDATE;
    if (checking && a.rmseThr >= 0.0) {               // ekf.cpp:797-801
        if (tid == 0) { double ss = 0.0; for (int i = 0; i < n; i++) { const double v = chunked ? VF[i] : T[(size_t)i * W + vcol]; ss += v * v; } s_scalar[0] = sqrt(ss / n); }
        __syncthreads();
        if (s_scalar[0] > a.rmseThr) { if (c == 0 && tid == 0) ekf_report(a, 2.0, 0.0, 0.0); return; }
    }
    if (checking && a.skipChi2 && a.mode == EKF_MODE_CHECK) {
        if (c == 0 && tid == 0) ekf_report(a, 0.0, 0.0, 0.0);
        return;
    }

    if (chunked) {
        for (int i = tid; i < N; i += EK2_NT) DM[i] = 0.0;
        __syncthreads();
    }

    // Row-chunked form: the rows are eliminated hc at a time on [S_k | HP_k | v_k], chunk k formed from what the earlier chunks left in
    // shared memory -- HP_k = H_k P_cur[0:l, J_c] from the downdated blocks, v_k = v_k(m_0) - H_k (m_cur - m_0) -- which is the trailing
    // update of the whole tableau (H_2 P_1 = H_2 P - L_21 Z_1, H_2 (m_1 - m_0) = L_21 z_1): the same update in exact arithmetic. chi2
    // is summed over the chunks; the decision, the write-back and the quaternion normalisation follow the last chunk (normalising in
    // between would break the equivalence). A check with its own noise level before an update (Rdiag2) is a pass of its own; the
    // update pass restarts from P and m in global memory, which the check pass does not write. Without chunks: one iteration.
    const bool twoPass = chunked && a.Rdiag2 > 0.0 && a.mode == EKF_MODE_CHECK_UPDATE && !a.skipChi2;
    int pass = 0, r0 = 0;                             // pass (1: the update of a two-pass op), first row of the chunk
    double Rk = a.Rdiag, chi2sum = 0.0;               // noise level of the pass, chi2 of the pass so far
    unsigned zph = 0, sph = 0;                        // phases of the Z-gather / S-exchange mbarriers (one completion per chunk)
    double* const Z = X;                              // the gathered Z, once H is dead
    const int cm = (N - 1) / B;                       // the last CTA that owns columns
    for (;;) {
        const int nr = chunked ? min(hc, n - r0) : n;     // rows of this chunk
        const bool lastChunk = r0 + nr >= n;
        const bool decideOnly = chunked && checking && pass == 0 && (a.mode == EKF_MODE_CHECK || twoPass);   // nothing to write back
        const int vk = nr + B, cend = joseph ? vk + nr : vk;                  // column of v in this chunk's tableau
        const int MTs = (nr + 7) >> 3, ETOT = 64 * (MTs * (MTs + 1) / 2);
        if (chunked) {
            if (pass > 0 || r0 > 0) cluster.sync();       // the neighbours are done with this CTA's tableau (Z gather) and partial S
            for (int t = tid; t < nr * l; t += EK2_NT) { const int i = t % nr, k = t / nr; X[t] = a.H[r0 + i + (size_t)k * n]; }   // H_k, ld nr
            __syncthreads();
            for (int i = tid; i < nr; i += EK2_NT) {
                double v = VF[r0 + i];
                for (int k = 0; k < l; k++) v -= X[i + (size_t)k * nr] * DM[k];
                T[(size_t)i * W + vk] = v;
            }
            __syncthreads();
        }

        EK2_PHASE(1);
        // ---- phase A: HP[:, J_c] = H P[0:l, J_c] on the fp64 tensor cores (n x Bc x l)
        ek2_dmma_gemm(nr, Bc, l, wrp, lane, Hs, 1, nr, PB, 1, LD,
                      [](int, int) { return 0.0; },
                      [&](int i, int j, double v0, double v1) { T[(size_t)i * W + nr + j] = v0; if (j + 1 < Bc) T[(size_t)i * W + nr + j + 1] = v1; });
        __syncthreads();
        EK2_PHASE(2);
        // ---- phase B: partial S = HP[:, J_c within [0, l)] H[:, J_c]' (n x n x kc), tiles on or above the diagonal only: the
        // blocked elimination never reads S below its diagonal tiles
        {
            const int kc = max(0, min(Bc, l - J0));
            ek2_dmma_gemm<true>(nr, nr, kc, wrp, lane, T + nr, W, 1, Hs + (size_t)J0 * nr, nr, 1,
                          [](int, int) { return 0.0; },
                          [&](int i, int j, double v0, double v1) {
                              if (oneStage) { RS[i * nr + j] = v0; if (j + 1 < nr) RS[i * nr + j + 1] = v1; }      // partial stays out of the tableau
                              else {                                                                            // tile-ordered, through L2
                                  const int mt = i >> 3, nt = j >> 3;
                                  double* dst = Spart + (size_t)c * ETOT + 64 * (nt * (nt + 1) / 2 + mt) + 8 * (i & 7) + (j & 7);
                                  dst[0] = v0; dst[1] = v1;
                              }
                          });
        }
        EK2_PHASE(3);
        if (!oneStage && bulk) ek2_fence_async_all();     // the partials are read by the neighbours' bulk copies
        cluster.sync();                                   // #1: every partial S is in place (and from here on shared memory is exposed)
        // ---- reduce S through distributed shared memory, fixed order r = 0 .. C-1 (+ R on the diagonal)
        {
            auto entry = [&](int e, int& i, int& ip) { int mt, nt; ek2_upper_tile(e >> 6, mt, nt); i = 8 * mt + ((e >> 3) & 7); ip = 8 * nt + (e & 7); };
            if (oneStage) {
                for (int e = tid; e < ETOT; e += EK2_NT) {
                    int i, ip; entry(e, i, ip);
                    if (i < nr && ip < nr) {
                        double s = 0.0;
                        for (int r = 0; r < C; r++) s += cluster.map_shared_rank(RS, r)[i * nr + ip];
                        if (i == ip) s += Rk;
                        T[(size_t)i * W + ip] = s;             // the own tableau is not read by anybody else
                    }
                }
                __syncthreads();
            } else if (bulk && ETOT >= 2048 && ETOT % (2 * C) == 0 && 2 * ETOT <= g.X) {
                // Through L2 with bulk copies: the eight partial slices and, after the second barrier, the reduced S arrive in the region H
                // occupied (dead since the partial product) by ONE round trip each, instead of one dependent load per entry and turn
                // (n = 84: 5.4 -> 4.4 us; below ~57 rows the barriers of the copies cost more than they save: n = 40 measured 2.8 -> 3.6 us)
                const int E = ETOT / C, e0 = c * E;
                double* SL = X + ETOT;                        // [C][E] partial slices
                if (wrp == 0) {
                    if (lane == 0) ek2_bar_expect(&s_bar[2], (unsigned)(C * E * 8));
                    __syncwarp();
                    if (lane < C) ek2_bulk_g2s(SL + (size_t)lane * E, Spart + (size_t)lane * ETOT + e0, (unsigned)(E * 8), &s_bar[2]);
                }
                ek2_bar_wait(&s_bar[2], sph);
                __syncthreads();
                for (int q = tid; q < E; q += EK2_NT) {
                    const int e = e0 + q;
                    int i, ip; entry(e, i, ip);
                    double sacc = 0.0;
                    if (i < nr && ip < nr) {
                        for (int r = 0; r < C; r++) sacc += SL[(size_t)r * E + q];
                        if (i == ip) sacc += Rk;
                    }
                    Sred[e] = sacc;
                }
                ek2_fence_async_all();                        // the reduced slice is read by everybody's bulk copy
                cluster.sync();                               // #2
                if (tid == 0) { ek2_bar_expect(&s_bar[3], (unsigned)(ETOT * 8)); ek2_bulk_g2s(X, Sred, (unsigned)(ETOT * 8), &s_bar[3]); }
                ek2_bar_wait(&s_bar[3], sph);
                sph ^= 1;
                __syncthreads();
                for (int tu = wrp; tu < ETOT / 64; tu += nwarps) {
                    int mt, nt; ek2_upper_tile(tu, mt, nt);
#pragma unroll
                    for (int h = 0; h < 2; h++) {
                        const int q = lane + 32 * h, i = 8 * mt + (q >> 3), ip = 8 * nt + (q & 7);
                        if (i < nr && ip < nr) T[(size_t)i * W + ip] = X[64 * tu + q];
                    }
                }
                __syncthreads();
            } else {
                const int E = (ETOT + C - 1) / C, e0 = c * E, e1 = min(ETOT, e0 + E);
                for (int e = e0 + tid; e < e1; e += EK2_NT) {
                    int i, ip; entry(e, i, ip);
                    double s = 0.0;
                    if (i < nr && ip < nr) {
                        for (int r = 0; r < C; r++) s += Spart[(size_t)r * ETOT + e];
                        if (i == ip) s += Rk;
                    }
                    Sred[e] = s;
                }
                cluster.sync();                               // #2: all slices reduced
                for (int tu = wrp; tu < ETOT / 64; tu += nwarps) {            // one tile per warp and turn: the tile index is decoded once
                    int mt, nt; ek2_upper_tile(tu, mt, nt);
#pragma unroll
                    for (int h = 0; h < 2; h++) {
                        const int q = lane + 32 * h, e = 64 * tu + q, i = 8 * mt + (q >> 3), ip = 8 * nt + (q & 7);
                        if (i < nr && ip < nr) T[(size_t)i * W + ip] = Sred[e];
                    }
                }
                __syncthreads();
            }
        }

        EK2_PHASE(4);
        bool decided = false;
        if (!chunked && a.Rdiag2 > 0.0 && a.mode == EKF_MODE_CHECK_UPDATE && a.op == EKF_OP_DENSE && !a.skipChi2) {
            // ---- check and update with different R: chi2 from a small tableau [S0 + R_check | v] in the region H occupied (dead since
            // phase B, not exposed to the cluster), every CTA for itself; the big tableau gets S0 + R_update and is eliminated below
            const int W2 = min(ek2_pad4mod16(n + 1), max(l, LD));       // (fits the region H occupied: n rows of max(l, LD) doubles)
            double* Xc = X;
            for (int e = tid; e < n * n; e += EK2_NT) Xc[(size_t)(e / n) * W2 + (e % n)] = T[(size_t)(e / n) * W + (e % n)];
            for (int i = tid; i < n; i += EK2_NT) Xc[(size_t)i * W2 + n] = T[(size_t)i * W + vcol];
            __syncthreads();
            for (int i = tid; i < n; i += EK2_NT) T[(size_t)i * W + i] += a.Rdiag2 - a.Rdiag;
            const bool bad2 = !ek2_block_eliminate(Xc, W2, n, n + 1, wrp, lane, s_linv, &s_bad);
            if (bad2) {                                   // uniform over the cluster
                if (c == 0 && tid == 0) ekf_report(a, 1.0, 0.0, 1.0);
                cluster.sync();
                return;
            }
            __syncthreads();
            if (wrp == 0) {
                double t = 0.0;
                for (int k = lane; k < n; k += 32) { const double z = Xc[(size_t)k * W2 + n]; t += z * z; }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) t += __shfl_sync(0xffffffffu, t, lane ^ o);
                if (lane == 0) s_scalar[1] = a.noiseScale * t;
            }
            __syncthreads();
            const double chi2c = s_scalar[1];
            const bool outlier = chi2c > a.chi2Thr;
            if (c == 0 && tid == 0) ekf_report(a, outlier ? 3.0 : 0.0, chi2c, 0.0);
            if (outlier) { cluster.sync(); return; }
            decided = true;
            __syncthreads();                              // s_scalar / s_linv are reused below
        }
        // ---- blocked forward elimination of [S | HP_Jc | v | (I)]: the right part becomes Z = L^-1 (.)
        const bool bad = !ek2_block_eliminate(T, W, nr, cend + 1, wrp, lane, s_linv, &s_bad);
        if (bad) {                                        // uniform over the cluster
            if (c == 0 && tid == 0) ekf_report(a, 1.0, 0.0, 1.0);
            if (a.specP) {
                // results go to the second buffers, but cannot be computed: leave the UNCHANGED state there, so that adopting them equals a
                // skipped update (what the in-place path does when this elimination fails)
                for (int idx = tid; idx < N * Bc; idx += EK2_NT) a.specP[(size_t)J0 * N + idx] = P[(size_t)J0 * N + idx];
                if (c == 0) for (int i = tid; i < N; i += EK2_NT) a.specM[i] = a.b.m[i];
            }
            cluster.sync();
            return;
        }
        __syncthreads();
        EK2_PHASE(5);
        if (wrp == 0) {                                   // chi2 = noiseScale |z_v|^2 (ekf.cpp:815): lane-strided sums, fixed shuffle tree
            double t = 0.0;
            for (int k = lane; k < nr; k += 32) { const double z = T[(size_t)k * W + vk]; t += z * z; }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) t += __shfl_sync(0xffffffffu, t, lane ^ o);
            if (lane == 0) s_scalar[1] = a.noiseScale * t;
        }
        __syncthreads();
        const double chi2 = s_scalar[1];
        if (chunked) {
            chi2sum += chi2;                              // (the decision follows the last chunk)
        } else if (decided) {
            // INLIER under the check's R has been reported already; chi2 here belongs to the update's R and is not reported
        } else if (checking) {
            const bool outlier = !a.skipChi2 && chi2 > a.chi2Thr;
            if (c == 0 && tid == 0) ekf_report(a, outlier ? 3.0 : 0.0, chi2, 0.0);
            if (outlier || a.mode == EKF_MODE_CHECK) { cluster.sync(); return; }
        } else if (c == 0 && tid == 0) ekf_report(a, 0.0, chi2, 0.0);

        if (!(lastChunk && decideOnly)) {
            EK2_PHASE(6);
            // ---- gather Z (n x N, row-major) out of the neighbours' tableaus, then P[:, J_c] -= Z' Z[:, J_c] in shared memory
            if ((size_t)nr * N >= 4096) {
                // large Z: through L2 (a CTA pulls an L2-resident block faster than a remote shared-memory one); every CTA publishes its slice, cluster barrier (release / acquire covers global memory), bulk read
                double* Zg = a.b.cwork;
                for (int t = tid; t < nr * Bc; t += EK2_NT) { const int k = t / Bc, jj = t - k * Bc; Zg[(size_t)k * N + J0 + jj] = T[(size_t)k * W + nr + jj]; }
                if (bulk) ek2_fence_async_all();              // the slice is read by the neighbours' bulk copies (async proxy)
                cluster.sync();                               // #3
                if (bulk) {
                    // one bulk copy per row of Z (N doubles into the padded leading dimension), issued by warp 0
                    if (wrp == 0) {
                        if (lane == 0) ek2_bar_expect(&s_bar[1], (unsigned)(nr * N * 8));
                        __syncwarp();
                        for (int k = lane; k < nr; k += 32) ek2_bulk_g2s(Z + (size_t)k * LD, Zg + (size_t)k * N, (unsigned)(N * 8), &s_bar[1]);
                    }
                    ek2_bar_wait(&s_bar[1], zph);
                    zph ^= 1;
                } else
                for (int base = 0; base < nr * N; base += 8 * EK2_NT) {
                    double r[8];
#pragma unroll
                    for (int u = 0; u < 8; u++) { const int t = base + u * EK2_NT + tid; r[u] = t < nr * N ? Zg[t] : 0.0; }
#pragma unroll
                    for (int u = 0; u < 8; u++) { const int t = base + u * EK2_NT + tid; if (t < nr * N) Z[(size_t)(t / N) * LD + (t % N)] = r[u]; }
                }
            } else {
                cluster.sync();                               // #3: every Z slice is final
                for (int t = tid; t < nr * N; t += EK2_NT) {  // small Z: straight out of the neighbours' tableaus, one flat pass
                    const int k = t / N, col = t - k * N, r = col / B;
                    Z[(size_t)k * LD + col] = cluster.map_shared_rank(T, r)[(size_t)k * W + nr + (col - r * B)];
                }
            }
            // The state mean m += Z' z_v rides along with the downdate of the LAST column block as one more column of its right-hand side
            // (z_v parked in the padding column N of Z): no second product, no extra barrier on any CTA's path. Chunked: every CTA
            // accumulates m_cur - m_0 += Z_k' z_k itself (the residual of the next chunk needs it), below.
            if (!chunked && c == cm) for (int k = tid; k < n; k += EK2_NT) Z[(size_t)k * LD + N] = T[(size_t)k * W + vcol];
            __syncthreads();
            EK2_PHASE(7);
            // P[:, J_c] -= Z' Z[:, J_c] on the fp64 tensor cores (N x Bc x n), in place in the shared-memory block
            // (accumulated as -P + Z'Z and negated on the way out: no per-step negation of an operand)
            {
                const int own = !chunked && c == cm ? 1 : 0;  // column Bc of the product: m + Z' z_v
                ek2_dmma_gemm(N, Bc + own, nr, wrp, lane, Z, 1, LD, Z + J0, LD, 1,
                              [&](int i, int j) { return j < Bc ? -PB[i + (size_t)j * LD] : s_m[i]; },
                              [&](int i, int j, double v0, double v1) {
                                  if (j < Bc) PB[i + (size_t)j * LD] = -v0; else s_m[i] = v0;
                                  if (j + 1 < Bc) PB[i + (size_t)(j + 1) * LD] = -v1; else if (j + 1 == Bc && own) s_m[i] = v1;
                              });
            }
            if (chunked)
                for (int i = tid; i < N; i += EK2_NT) {
                    double s = DM[i];
                    for (int k = 0; k < nr; k++) s += Z[(size_t)k * LD + i] * T[(size_t)k * W + vk];
                    DM[i] = s;
                }
        }   // (gather and downdate)
        if (!chunked) break;
        if (!lastChunk) { r0 += nr; continue; }
        // ---- end of a chunked pass: the decisions the single-chunk form takes after its elimination
        if (checking && pass == 0) {
            const bool outlier = !a.skipChi2 && chi2sum > a.chi2Thr;
            if (c == 0 && tid == 0) ekf_report(a, outlier ? 3.0 : 0.0, chi2sum, 0.0);
            if (outlier || a.mode == EKF_MODE_CHECK) { cluster.sync(); return; }
            if (twoPass) {                                // INLIER under the check's R: the update pass, from P and m as they were
                const double* src = P + (size_t)J0 * N;
                for (int idx = tid; idx < N * Bc; idx += EK2_NT) PB[(idx % N) + (size_t)(idx / N) * LD] = src[idx];
                for (int i = tid; i < N; i += EK2_NT) DM[i] = 0.0;
                pass = 1; r0 = 0; chi2sum = 0.0; Rk = a.Rdiag2;
                continue;
            }
        } else if (!checking && c == 0 && tid == 0) ekf_report(a, 0.0, chi2sum, 0.0);
        break;
    }   // chunks
    // Joseph form, first step: the gain K = Z' (L^-1 I) (N x 7) needs the gathered Z and the eliminated identity columns only, so it
    // shares the barrier of the downdate
    if (joseph) {
        double* Ks = EX;
        for (int t = tid; t < N * EKF_POSE; t += EK2_NT) {
            const int i = t % N, r = t / N;
            double s = 0.0;
            for (int k = 0; k < n; k++) s += Z[(size_t)k * LD + i] * T[(size_t)k * W + vcol + 1 + r];
            Ks[t] = s;
        }
    }
    // quaternion normalisation: updateCommon normalises the current orientation only, the visual update and the augmentation all of
    // them (ekf.cpp:31, 843, 874)
    if (bulk) ek2_fence_async_smem();                 // the block just written leaves by bulk copies (below)
    __syncthreads();
    if (c == cm) {
        if (chunked) {                                // m = m_0 + the change the chunks accumulated
            for (int i = tid; i < N; i += EK2_NT) s_m[i] += DM[i];
            __syncthreads();
        }
        for (int q = tid; q < (a.normalizeAll ? a.b.trail + 1 : 1); q += EK2_NT)
            ek2_normalize_quat(q == 0 ? s_m + EKF_ORI : s_m + EKF_CAM + EKF_POSE * (q - 1) + 3);
        ek2_fence_async_smem();
        __syncthreads();
        double* const mDst = a.specM ? a.specM : a.b.m;
        if (bulk) { if (tid == 32) { ek2_bulk_s2g(mDst, s_m, (unsigned)(N * 8)); ek2_bulk_store_done(); } }
        else for (int i = tid; i < N; i += EK2_NT) mDst[i] = s_m[i];
    }
    EK2_PHASE(8);

    double* Pblk = PB;                                // block holding this CTA's final columns ...
    int ldb = LD;                                     // ... and its leading dimension
    if (joseph) {
        // ---- Joseph form (ekf.cpp:35-50): P'' = G T1' + K R K', G = T1 P' = P' - Z'Z (in PB now), T1 = I - K visAugH
        // As ONE product on the tensor cores: P''[:, J_c] = [G_special | K] (N x 21) * [T1c | R K]' (21 x Bc) + (G[:, J_c] on the
        // non-special columns): the 14 special columns of G come from the CTAs that own them (distributed shared memory).
        double* Ks = EX;                              // N x 7
        double* AS = Ks + (size_t)N * EKF_POSE;       // N x 21, ld LD: [G special columns | K]
        double* BS = AS + (size_t)21 * LD;            // N x 21, ld LD: [T1c | Rdiag K]
        double* P2 = BS + (size_t)21 * LD;            // N x B: P'' block
        EK2_PHASE(10);
        for (int t = tid; t < N * 21; t += EK2_NT) {
            const int j = t % N, cc = t / N;
            if (cc < 14) {
                const double kv = cc < 7 ? -Ks[j + cc * N] : Ks[j + (cc - 7) * N];
                BS[j + (size_t)cc * LD] = (j == ek2_special_col(cc) ? 1.0 : 0.0) + kv;          // T1 = I - K visAugH, its 14 columns
            } else {
                BS[j + (size_t)cc * LD] = a.Rdiag * Ks[j + (cc - 14) * N];
                AS[j + (size_t)cc * LD] = Ks[j + (cc - 14) * N];
            }
        }
        EK2_PHASE(11);
        cluster.sync();                               // #4: all of G is final
        EK2_PHASE(12);
        // (fetched by every CTA: letting the two owners PUSH their 7 columns each to all eight CTAs serialises the remote stores
        // on two CTAs, while the remote loads spread over all of them)
        for (int t = tid; t < N * 14; t += EK2_NT) {
            const int i = t % N, cc = t / N;
            const int col = ek2_special_col(cc), r = col / B;
            AS[i + (size_t)cc * LD] = cluster.map_shared_rank(PB, r)[i + (size_t)(col - r * B) * LD];
        }
        __syncthreads();
        EK2_PHASE(13);
        ek2_dmma_gemm(N, Bc, 21, wrp, lane, AS, 1, LD, BS + J0, LD, 1,
                      [&](int i, int jj) {
                          const int j = J0 + jj;
                          const bool jsp = j < 3 || (j >= EKF_ORI && j < EKF_ORI + 4) || (j >= EKF_CAM && j < EKF_CAM + EKF_POSE);
                          return jsp ? 0.0 : PB[i + (size_t)jj * LD];
                      },
                      [&](int i, int jj, double v0, double v1) { P2[i + (size_t)jj * N] = v0; if (jj + 1 < Bc) P2[i + (size_t)(jj + 1) * N] = v1; });
        Pblk = P2; ldb = N;
        EK2_PHASE(14);
    }
    double* const Pdst = a.specP ? a.specP : P;
    if (a.symmetrize) {
        // the mirrored entry of P(i, j) is P(j, i), held by the CTA that owns column i: every CTA SENDS the entries of its block to the
        // owners of their mirror images (row j of the own column i -> slot (i, j) of the owner of column j, the buffer g.SYM), remote
        // stores that are complete at the cluster barrier; the first version fetched them after the barrier (a dependent round trip per element)
        if (joseph) __syncthreads();                  // the Joseph product above wrote the block
        for (int idx = tid; idx < N * Bc; idx += EK2_NT) {
            const int jrow = idx % N, icol = idx / N, r = jrow / B;
            cluster.map_shared_rank(SYMB, r)[(J0 + icol) + (size_t)(jrow - r * B) * N] = Pblk[jrow + (size_t)icol * ldb];
        }
        cluster.sync();                               // #5: every final block is in shared memory, every mirror image has arrived
        EK2_PHASE(15);
        for (int idx = tid; idx < N * Bc; idx += EK2_NT) {
            const int i = idx % N, jj = idx / N, j = J0 + jj;
            double v = Pblk[i + (size_t)jj * ldb];
            const double w = SYMB[idx];
            if (i != j) v = i > j ? 0.5 * (v + w) : 0.5 * (w + v);
            Pdst[i + (size_t)j * N] = v;
        }
    } else if (bulk) {
        // (the downdate wrote the block with ordinary stores: fenced towards the bulk-copy engine right after it, a CTA barrier since)
        if (wrp == 0) {
            for (int j = lane; j < Bc; j += 32) ek2_bulk_s2g(Pdst + (size_t)(J0 + j) * N, Pblk + (size_t)j * ldb, (unsigned)(N * 8));
            ek2_bulk_store_done();
        }
    } else {
        for (int idx = tid; idx < N * Bc; idx += EK2_NT) Pdst[(size_t)J0 * N + idx] = Pblk[(idx % N) + (size_t)(idx / N) * ldb];
    }
    EK2_PHASE(9);
    if (a.bump && c == 0 && tid == 0) *a.bump = *a.bump + 1;          // one writer per grid; kernels of a chain are stream-ordered
    cluster.sync();                                   // nobody may leave while its shared memory can still be read
}

// ---- one outlier check on ONE CTA (the compact clusters of ekf_check_batch_cluster2_kernel) --------------------------------------
// A check needs chi2 only, and chi2 needs S = H P[0:l, 0:l] H' + R and v, not HP over all N columns nor the downdate. This body forms
// S from the cluster's own column blocks J_c (c = 0 .. 7), one after the other in one CTA: stage P[0:l, J_c within [0, l)], HP_c with
// the call of phase A, the partial S_c with the call of phase B, s += S_c in the order c = 0 .. 7 from +0.0 (the order of both
// reductions of ek2_body; a block at or beyond l adds +0.0 there, which cannot change a sum that starts at +0.0, so it is skipped),
// then + R on the diagonal. The elimination runs on [S | v] only: every entry of its products depends on its own row and column
// operands and the k order alone, so z_v and therefore every result word are bitwise those of ek2_body. The batch's checks carry no
// device-side gates and no second noise level (check_items). Shared memory: scratch | H (n x l, ld n) | tableau rows [S | v | HP_c]
// (ld W, as ek2_geom's) | P block (l x B, ld LDP).
struct Ek2CheckGeom { int B, W, LDP, X, T; };
#define EK2_CTA_SCRATCH (EK2_LINV_DOUBLES + 4)         // L_jj^-1 (2 x 64) | rmse, chi2 | pivot flag (+ pad: H starts 16-byte aligned)
__host__ __device__ inline Ek2CheckGeom ek2_check_geom(int n, int l, int N)
{
    Ek2CheckGeom g;
    g.B = (N + EK2_C - 1) / EK2_C;
    g.W = ek2_pad4mod16(n + 1 + g.B);
    g.LDP = ek2_pad4mod16(l);
    g.X = (n * l + 1) & ~1;
    g.T = (n * g.W + 1) & ~1;
    return g;
}
__host__ __device__ inline size_t ek2_check_cta_smem_bytes(int n, int l, int N)
{
    const Ek2CheckGeom g = ek2_check_geom(n, l, N);
    return ((size_t)EK2_CTA_SCRATCH + g.X + g.T + (size_t)g.LDP * g.B) * sizeof(double);
}

#ifdef HV_EMU
#define EK2_NOINLINE inline
#else
#define EK2_NOINLINE __noinline__             // its own register allocation: inlined beside ek2_body, the batch kernel spills
#endif
__device__ EK2_NOINLINE void ek2_check_cta(const EkfUpdateArgs& a, double* sm)
{
    const int tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5;
    const int N = a.b.N, n = a.n, l = a.l;
    const Ek2CheckGeom g = ek2_check_geom(n, l, N);
    const int W = g.W, B = g.B, LDP = g.LDP;
    double* const s_linv = sm;
    double* const s_scalar = sm + EK2_LINV_DOUBLES;
    volatile int* const s_bad = (volatile int*)(sm + EK2_LINV_DOUBLES + 2);
    double* const Hs = sm + EK2_CTA_SCRATCH;
    double* const T = Hs + g.X;
    double* const PB = T + g.T;
    ek2_pdl_launch_dependents();                      // (see ek2_body)
    if (!a.lateH) ek2_copy8(Hs, a.H, n * l, tid);
    ek2_pdl_wait();
    if (a.lateH) ek2_copy8(Hs, a.H, n * l, tid);
    __syncthreads();
    for (int i = tid; i < n; i += EK2_NT) {
        const double yi = a.y ? a.y[i] : a.ysmall[i];
        double fi = 0.0;
        if (a.f) fi = a.f[i];
        else for (int k = 0; k < l; k++) fi += Hs[i + (size_t)k * n] * a.b.m[k];
        T[(size_t)i * W + n] = yi - fi;
    }
    for (int e = tid; e < n * n; e += EK2_NT) T[(size_t)(e / n) * W + (e % n)] = 0.0;
    __syncthreads();
    if (a.rmseThr >= 0.0) {                           // ekf.cpp:797-801
        if (tid == 0) { double ss = 0.0; for (int i = 0; i < n; i++) { const double v = T[(size_t)i * W + n]; ss += v * v; } s_scalar[0] = sqrt(ss / n); }
        __syncthreads();
        if (s_scalar[0] > a.rmseThr) { if (tid == 0) ekf_report(a, 2.0, 0.0, 0.0); return; }
    }
    if (a.skipChi2) { if (tid == 0) ekf_report(a, 0.0, 0.0, 0.0); return; }

    for (int c = 0; c < EK2_C; c++) {
        const int J0 = c * B, kc = min(B, l - J0);    // (l <= N: the block's columns below l)
        if (kc <= 0) break;
        const double* src = a.b.P + (size_t)J0 * N;
        const int count = l * kc;
        for (int base = 0; base < count; base += 8 * EK2_NT) {
            double r[8];
#pragma unroll
            for (int u = 0; u < 8; u++) { const int t = base + u * EK2_NT + tid, j = t / l; r[u] = t < count ? src[(t - j * l) + (size_t)j * N] : 0.0; }
#pragma unroll
            for (int u = 0; u < 8; u++) { const int t = base + u * EK2_NT + tid, j = t / l; if (t < count) PB[(t - j * l) + (size_t)j * LDP] = r[u]; }
        }
        __syncthreads();
        ek2_dmma_gemm(n, kc, l, wrp, lane, Hs, 1, n, PB, 1, LDP,
                      [](int, int) { return 0.0; },
                      [&](int i, int j, double v0, double v1) { T[(size_t)i * W + n + 1 + j] = v0; if (j + 1 < kc) T[(size_t)i * W + n + 2 + j] = v1; });
        __syncthreads();
        ek2_dmma_gemm<true>(n, n, kc, wrp, lane, T + n + 1, W, 1, Hs + (size_t)J0 * n, n, 1,
                            [](int, int) { return 0.0; },
                            [&](int i, int j, double v0, double v1) { T[(size_t)i * W + j] += v0; if (j + 1 < n) T[(size_t)i * W + j + 1] += v1; });
        __syncthreads();
    }
    for (int i = tid; i < n; i += EK2_NT) T[(size_t)i * W + i] += a.Rdiag;
    __syncthreads();
    if (!ek2_block_eliminate(T, W, n, n + 1, wrp, lane, s_linv, s_bad)) {
        if (tid == 0) ekf_report(a, 1.0, 0.0, 1.0);
        return;
    }
    __syncthreads();
    if (wrp == 0) {                                   // as ek2_body: lane-strided sums, fixed shuffle tree
        double t = 0.0;
        for (int k = lane; k < n; k += 32) { const double z = T[(size_t)k * W + n]; t += z * z; }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_sync(0xffffffffu, t, lane ^ o);
        if (lane == 0) s_scalar[1] = a.noiseScale * t;
    }
    __syncthreads();
    const double chi2 = s_scalar[1];
    if (tid == 0) ekf_report(a, chi2 > a.chi2Thr ? 3.0 : 0.0, chi2, 0.0);
}

// ---- the state mean of the pose augmentation on ONE CTA (EKF_OP_AUGMENT, a.specM; the covariance is left to a cluster elsewhere) -----
// m' = m_shift + Z' z_v needs the eliminated [S | HP | v] only: HP = H P_shift[0:l, :] with l = EKF_CAM + EKF_POSE, S = HP[:, 0:l] H' + R,
// not the N x N downdate and Joseph product. The body stages the l rows of the shifted P (ek2_aug_entry, symmetrised when a.symFirst),
// forms HP with the call of ek2_body's phase A, the partial S of every column block J_c of the cluster with the call of phase B, summed in
// the order c = 0 .. 7 from +0.0 (blocks at or beyond l add +0.0 there, as in ek2_check_cta), eliminates with the same routine and
// forms m' with the product that carries the mean along with the cluster's downdate (a column of its own, A = Z, B = z_v, C = m_shift).
// Every entry of these products depends on its own row and column operands and the k order alone, so m' and the result words are bitwise
// those of ek2_body; a non-positive pivot leaves the unchanged mean in a.specM, as ek2_body does. Shared memory: scratch | m (N) |
// H (n x l, ld n) | tableau rows [S | v | HP] (ld W) | P_shift[0:l, :] (ld LDP).
struct Ek2AugMeanGeom { int W, LDP, M, X, T; };
__host__ __device__ inline Ek2AugMeanGeom ek2_aug_mean_geom(int n, int l, int N)
{
    Ek2AugMeanGeom g;
    g.W = ek2_pad4mod16(n + 1 + N);
    g.LDP = ek2_pad4mod16(l);
    g.M = (N + 1) & ~1;
    g.X = (n * l + 1) & ~1;
    g.T = (n * g.W + 1) & ~1;
    return g;
}
__host__ __device__ inline size_t ek2_aug_mean_smem_bytes(int n, int l, int N)
{
    const Ek2AugMeanGeom g = ek2_aug_mean_geom(n, l, N);
    return ((size_t)EK2_CTA_SCRATCH + g.M + g.X + g.T + (size_t)g.LDP * N) * sizeof(double);
}

__device__ inline void ek2_aug_mean_cta(const EkfUpdateArgs& a, double* sm)
{
    const int tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5;
    const int N = a.b.N, n = a.n, l = a.l, B = (N + EK2_C - 1) / EK2_C;
    const Ek2AugMeanGeom g = ek2_aug_mean_geom(n, l, N);
    const int W = g.W, LDP = g.LDP, hp = n + 1;      // tableau: S in columns 0 .. n-1, v in column n, HP from column hp
    double* const s_linv = sm;
    double* const s_scalar = sm + EK2_LINV_DOUBLES;
    volatile int* const s_bad = (volatile int*)(sm + EK2_LINV_DOUBLES + 2);
    double* const s_m = sm + EK2_CTA_SCRATCH;
    double* const Hs = s_m + g.M;
    double* const T = Hs + g.X;
    double* const PB = T + g.T;
    ek2_pdl_launch_dependents();                      // (see ek2_body)
    // the measurement model (ek2_body, EKF_OP_AUGMENT) depends on nothing earlier kernels write
    for (int i = tid; i < n * l; i += EK2_NT) Hs[i] = 0.0;
    __syncthreads();
    if (tid == 0) {
        for (int i = 0; i < 3; i++) { Hs[i + (EKF_POS + i) * n] = 1.0; Hs[i + (EKF_CAM + i) * n] = -1.0; }
        for (int i = 0; i < 4; i++) { Hs[3 + i + (EKF_ORI + i) * n] = 1.0; Hs[3 + i + (EKF_CAM + 3 + i) * n] = -1.0; }
    }
    ek2_pdl_wait();
    for (int i = tid; i < N; i += EK2_NT) { const int s = ek2_aug_src(i, a.dropIdx); s_m[i] = s < 0 ? 0.0 : a.b.m[s]; }
    for (int base = 0; base < l * N; base += 8 * EK2_NT) {        // rows 0 .. l-1 of the shifted P, 8 entries in flight per thread
        double r[8];
#pragma unroll
        for (int u = 0; u < 8; u++) { const int t = base + u * EK2_NT + tid, j = t / l; r[u] = t < l * N ? ek2_aug_entry(a, t - j * l, j) : 0.0; }
#pragma unroll
        for (int u = 0; u < 8; u++) { const int t = base + u * EK2_NT + tid, j = t / l; if (t < l * N) PB[(t - j * l) + (size_t)j * LDP] = r[u]; }
    }
    for (int e = tid; e < n * n; e += EK2_NT) T[(size_t)(e / n) * W + (e % n)] = 0.0;
    __syncthreads();
    for (int i = tid; i < n; i += EK2_NT) {           // residual, as ek2_body
        const double yi = a.y ? a.y[i] : a.ysmall[i];
        double fi = 0.0;
        if (a.f) fi = a.f[i];
        else for (int k = 0; k < l; k++) fi += Hs[i + (size_t)k * n] * s_m[k];
        T[(size_t)i * W + n] = yi - fi;
    }
    // HP = H P_shift[0:l, :] (phase A of ek2_body over all N columns at once)
    ek2_dmma_gemm(n, N, l, wrp, lane, Hs, 1, n, PB, 1, LDP,
                  [](int, int) { return 0.0; },
                  [&](int i, int j, double v0, double v1) { T[(size_t)i * W + hp + j] = v0; if (j + 1 < N) T[(size_t)i * W + hp + j + 1] = v1; });
    __syncthreads();
    // S = sum over the cluster's column blocks in block order of HP[:, J_c within [0, l)] H[:, J_c]' (phase B), then + R
    for (int c = 0; c < EK2_C; c++) {
        const int J0 = c * B, kc = min(B, l - J0);
        if (kc <= 0) break;
        ek2_dmma_gemm<true>(n, n, kc, wrp, lane, T + hp + J0, W, 1, Hs + (size_t)J0 * n, n, 1,
                            [](int, int) { return 0.0; },
                            [&](int i, int j, double v0, double v1) { T[(size_t)i * W + j] += v0; if (j + 1 < n) T[(size_t)i * W + j + 1] += v1; });
        __syncthreads();
    }
    for (int i = tid; i < n; i += EK2_NT) T[(size_t)i * W + i] += a.Rdiag;
    __syncthreads();
    if (!ek2_block_eliminate(T, W, n, hp + N, wrp, lane, s_linv, s_bad)) {
        if (tid == 0) ekf_report(a, 1.0, 0.0, 1.0);
        for (int i = tid; i < N; i += EK2_NT) a.specM[i] = a.b.m[i];
        return;
    }
    __syncthreads();
    if (wrp == 0) {                                   // chi2 as ek2_body reports it
        double t = 0.0;
        for (int k = lane; k < n; k += 32) { const double z = T[(size_t)k * W + n]; t += z * z; }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_sync(0xffffffffu, t, lane ^ o);
        if (lane == 0) s_scalar[1] = a.noiseScale * t;
    }
    // m' = m_shift + Z' z_v (N x 1 x n), in place: every row of s_m is read and written by the warp that owns its tile
    ek2_dmma_gemm(N, 1, n, wrp, lane, T + hp, 1, W, T + n, W, 1,
                  [&](int i, int) { return s_m[i]; },
                  [&](int i, int, double v0, double) { s_m[i] = v0; });
    __syncthreads();
    if (tid == 0) ekf_report(a, 0.0, s_scalar[1], 0.0);
    for (int q = tid; q < (a.normalizeAll ? a.b.trail + 1 : 1); q += EK2_NT)
        ek2_normalize_quat(q == 0 ? s_m + EKF_ORI : s_m + EKF_CAM + EKF_POSE * (q - 1) + 3);
    __syncthreads();
    for (int i = tid; i < N; i += EK2_NT) a.specM[i] = s_m[i];
}

// Cluster `inst` of a group launch (ekf_group_cluster2_kernel): its own argument block, fully resolved by the host (filter buffers,
// exchange area, result words, second buffers), read from device memory. Clusters of one launch share nothing.
template <class Cluster>
__device__ __forceinline__ void ek2_group_body(const EkfUpdateArgs* __restrict__ args, int inst, double* sm, Cluster cluster)
{
    EkfUpdateArgs a = args[inst];
    ek2_body<false>(a, sm, cluster);
}
