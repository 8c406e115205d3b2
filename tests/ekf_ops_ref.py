"""Plain extended-precision reference of the EKF's non-visual operations (src/odometry/ekf.cpp, conventions as restated in
oracle/hv_oracle_ekf.c): the pose augmentation (848-885 with the Joseph form 35-50), the fixed-H updates (update() 57-82 and 573-677),
transformTo (704-758), conditionOnLastPose (928-942) and normalizeQuaternions (1024-1032), each with a componentwise error bound for
an fp64 implementation, and fp64 restatements of the operations that are pure permutations, zeroings or one rounding per entry
(unaugment, lockBiases, insertMapPoint, translateTo, maintainPositiveSemiDefinite, the augmentation's shift), which the
implementations must reproduce bit for bit.

The reference works in np.longdouble (80-bit on x86-64) from the equations: HP = H P[0:l, :], S = HP[:, 0:l] H' + R I, a Cholesky
factor of S, K = (S^-1 HP)', m += K v, P -= K HP. It never uses the kernels' algebra (no elimination tableau, no Z = L^-1 HP). The
augmentation is computed two ways: the literal Joseph form T1 P+ T1' + K R K' with T1 = I - K visAugH (augment(form="joseph"), dense
N x N x N, small N only), and the cancellation-free closed form that uses that the new slot c has no prior cross-covariance. With a the
current pose (position, orientation), Q the augmentation noise of slot c and S = P_aa + Q + R:
    P'_cc = Q S^-1 (P_aa + R),   P'_co = Q S^-1 P_ao,   P'_oo' = P_oo' - P_oa S^-1 P_ao',   m'_c = Q S^-1 m_a,
    m'_o = m_o - P_oa S^-1 m_a
(form="closed", O(7 N^2)). Inputs the host computes in fp64 (noiseScale = noise_scale^2, R = r noiseScale, the augmentation noise)
are taken as the same fp64 numbers; init_zupt_r noiseScale exp(0.5 t) is formed in longdouble and its fp64 error (4u relative)
enters the bound as eR R |K| |K|'.

Error bound. Every computed entry gets C u (absolute-value evaluation of the operation), u = 2^-53, where the absolute-value
evaluation of a product replaces every sum by the sum of the absolute values of its terms:
  * update (UPDATE):        C_UPD kappa(S) (|P| + |K| |H| |P_l|),     m: C_UPD kappa(S) (|m| + |K| (|v| + l u (|H| |m_l| + |y|))),
                            |K| = |P_l|' |H|' |S^-1| (H of the pseudo-velocity update is formed from the fp64 mean)
  * augmentation (AUGMENT): C_AUG kappa(S) (|T1| (|P+| + |K| |H| |P+|) |T1|' + |K| R |K|'),  P+ = A P A' + Q
  * transform:              C_XF |A| |P| |A|',  |A| the absolute-value evaluation of the block rotations
  * conditioning:           C_COND kappa(B) (|P_aa| + |P_ab| |B^-1| |P_ba|)
  * normalisation of q:     2 sum(B_q) / |q| + C_NORM u |q / |q||
An entry whose evaluation has no rounding (every product term 0 apart from a copy) gets the bound 0 and must be exact: structural
zeros, untouched blocks, the 1e6 blocks of insertMapPoint / conditionOnLastPose.

Tally of C (standard inner-product bounds gamma_k ~ k u, Higham, Accuracy and Stability of Numerical Algorithms 3.1; only the
nonzero terms of the sparse products count, zero products add exactly):
  * UPDATE, n <= 4 rows, selector or 2-column H: HP 2 terms (2u), S 2 terms + R (3u), elimination / Cholesky of n rows ((n + 1)u,
    carried through kappa(S)), Z = D^-1/2 L^-1 HP (n terms, sqrt and division: (n + 3)u), the n-term Z'Z and the subtraction
    ((n + 1)u), symmetrisation (1u): at n = 4 2 + 3 + 5 + 7 + 5 + 1 = 23u. The augmentation's own update (n = 7) is 32u by the same
    count. C_UPD = 64 (the next power of two, doubled for the split S sums of the cluster kernel).
  * AUGMENT: the n = 7 downdate G = P+ - K HP (32u), the gain K = Z'M (7 terms, 8u), T1's special columns (1u), G T1' (the 14
    special columns plus the copy: 15u), K R K' (8u), the final sum and the symmetrisation (2u): 66u. C_AUG = 128.
  * transform: qc (4-term products, 4u) and the entries of R(qc) / Omega(qc) from it (2u products, 2-term sums: 4u more), so A is
    within 8u of |A|; the inner 4-term and outer 4-term sums (8u) and A twice (16u): 24u. C_XF = 32.
  * conditioning: B^-1 by Gauss-Jordan on 7 rows (7u, through kappa(B)), P_ab B^-1 (7 terms), its product with P_ba (7 terms), the
    subtraction (1u): 22u. C_COND = 32.
  * normalisation: 4 squares in two pairs (3u), sqrt (1u), division (1u): 5u. C_NORM = 8."""
import numpy as np

import ekf_script
import predict_ref as PR

LD = np.longdouble
U = 2.0 ** -53
C_UPD, C_AUG, C_XF, C_COND, C_NORM = 64.0, 128.0, 32.0, 32.0, 8.0
POS, VEL, ORI, BGA, BAA, BAT, SFT, CAM, INER, POSE, MAPPT = 0, 3, 6, 10, 13, 16, 19, 20, 20, 7, 3
CUR = np.array([POS, POS + 1, POS + 2, ORI, ORI + 1, ORI + 2, ORI + 3])          # the current pose a of visAugH
NEW = np.arange(CAM, CAM + POSE)                                                # the new slot c
SPECIAL = np.concatenate([CUR, NEW])                                            # the 14 columns visAugH touches


def state_dim(trail, map_size):
    return INER + POSE * trail + MAPPT * map_size


# ------------------------------------------------------------------------------------------------ results and comparison
class Result:
    """(m, P) in longdouble with their componentwise bounds."""

    def __init__(self, m, P, Bm, BP):
        self.m, self.P, self.Bm, self.BP = m, P, Bm, BP

    def ratios(self, m, P):
        return {"m": bound_ratio(m, self.m, self.Bm), "P": bound_ratio(P, self.P, self.BP)}

    def worst_entry(self, P):
        """(ratio, i, j) of the worst entry of P; ratio inf where an entry with bound 0 is not exact."""
        d = np.abs(np.asarray(P, dtype=LD) - self.P)
        zero = self.BP == 0
        r = np.where(zero, np.where(d > 0, LD(np.inf), LD(0)), d / np.where(zero, LD(1), self.BP))
        i, j = np.unravel_index(int(np.argmax(r)), r.shape)
        return float(r[i, j]), int(i), int(j)


def bound_ratio(got, ref, bound):
    """max |got - ref| / bound over the entries with a nonzero bound; inf if an entry with a zero bound is not exact."""
    got, ref, bound = np.asarray(got, dtype=LD), np.asarray(ref, dtype=LD), np.asarray(bound, dtype=LD)
    d = np.abs(got - ref)
    zero = bound == 0
    if (d[zero] != 0).any():
        return float("inf")
    return float((d[~zero] / bound[~zero]).max()) if (~zero).any() else 0.0


def block_of(i, trail, map_size):
    """Which part of the state index i lies in: inertial / new slot / trail / map."""
    if i < INER:
        return "inertial"
    if i < CAM + POSE:
        return "new slot"
    return "trail" if i < CAM + POSE * trail else "map"


# ------------------------------------------------------------------------------------------------ linear algebra (longdouble)
def _chol(S):
    n = S.shape[0]
    L = np.zeros_like(S)
    for j in range(n):
        d = S[j, j] - L[j, :j] @ L[j, :j]
        if not d > 0:
            raise ValueError("S is not positive definite")
        L[j, j] = np.sqrt(d)
        L[j + 1:, j] = (S[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
    return L


def _solve(S, B):
    """S^-1 B for symmetric positive definite S (Cholesky)."""
    L = _chol(S)
    X = np.array(B, dtype=LD, copy=True)
    for i in range(L.shape[0]):
        X[i] = (X[i] - L[i, :i] @ X[:i]) / L[i, i]
    for i in range(L.shape[0] - 1, -1, -1):
        X[i] = (X[i] - L[i + 1:, i] @ X[i + 1:]) / L[i, i]
    return X


def _inv(B):
    """Inverse of a general square matrix (Gauss-Jordan with partial pivoting in longdouble)."""
    n = B.shape[0]
    M = np.concatenate([np.array(B, dtype=LD), np.eye(n, dtype=LD)], axis=1)
    for c in range(n):
        p = c + int(np.argmax(np.abs(M[c:, c])))
        M[[c, p]] = M[[p, c]]
        M[c] /= M[c, c]
        for r in range(n):
            if r != c:
                M[r] -= M[r, c] * M[c]
    return M[:, n:]


def _cond(S):
    return float(np.linalg.cond(np.asarray(S, dtype=np.float64)))


def _sym(P):
    return 0.5 * (P + P.T)


def _normalize(m, Bm, offsets):
    """normalizeQuaternions at the given offsets (zero slots stay zero) and the bound of the result."""
    for o in offsets:
        q = m[o:o + 4]
        z = q @ q
        if z > 0:
            nrm = np.sqrt(z)
            qn = q / nrm
            Bm[o:o + 4] = 2 * Bm[o:o + 4].sum() / nrm + C_NORM * U * np.abs(qn)
            m[o:o + 4] = qn


def quaternion_offsets(trail, only_current):
    return [ORI] if only_current else [ORI] + [CAM + POSE * i + 3 for i in range(trail)]


# ------------------------------------------------------------------------------------------------ the reference
def noise_scale(params):
    return np.float64(params.noise_scale) * np.float64(params.noise_scale)


def aug_src(N, drop):
    """Source index of every row of the augmentation shift A (ekf.cpp:230-248); -1: zero row."""
    i = np.arange(N)
    return np.where(i < CAM, i, np.where(i < CAM + POSE, -1, np.where(i < CAM + (drop + 1) * POSE, i - POSE, i)))


def shift_fp64(m, P, src):
    """A m and A P A' for a 0/1 selection A given by src (-1: zero): a copy, exact in fp64."""
    ok = src >= 0
    s = np.where(ok, src, 0)
    m2 = np.where(ok, np.asarray(m, np.float64)[s], 0.0)
    P2 = np.asarray(P, np.float64)[np.ix_(s, s)] * (ok[:, None] & ok[None, :])
    return m2, np.where(ok[:, None] & ok[None, :], P2, 0.0)


def symmetrize_fp64(P):
    """maintainPositiveSemiDefinite (ekf.cpp:1059-1067): 0.5 (P_ij + P_ji), one rounding per entry."""
    P = np.asarray(P, np.float64)
    return 0.5 * (P + P.T)


class Ops:
    """The reference of one filter layout. `params` has the fields of hv_ekf_params."""

    def __init__(self, params):
        self.p = params
        self.trail, self.map_size = params.camera_trail_length, params.hybrid_map_size
        self.N = state_dim(self.trail, self.map_size)
        self.ns = noise_scale(params)

    # ---- update() (ekf.cpp:57-82): a generic update with its bound
    def _update(self, m, P, H, y=None, v=None, R=0.0, eR=0.0):
        m, P = np.array(m, dtype=LD), np.array(P, dtype=LD)
        H = np.asarray(H, dtype=LD)
        n, l = H.shape
        R = LD(R)
        HP = H @ P[:l]
        S = _sym(HP[:, :l] @ H.T) + R * np.eye(n, dtype=LD)
        W = _solve(S, HP)                                   # S^-1 HP = K'
        if v is None:
            v = np.asarray(y, dtype=LD) - H @ m[:l]
        m1 = m + W.T @ v
        P1 = P - HP.T @ W
        kap = _cond(S)
        aHP = np.abs(H) @ np.abs(P[:l])
        aK = aHP.T @ np.abs(_inv(S))                        # absolute-value evaluation of K = HP' S^-1
        X = aK @ aHP
        BP = np.where(X != 0, C_UPD * U * kap * (np.abs(P) + X), LD(0))
        av = np.abs(v) + l * U * (np.abs(H) @ np.abs(m[:l]) + (np.abs(np.asarray(y, dtype=LD)) if y is not None else 0))
        Xm = aK @ av
        Bm = np.where(Xm != 0, C_UPD * U * kap * (np.abs(m) + Xm), LD(0))
        if eR:
            BP = BP + LD(eR) * R * (aK @ aK.T)
            Bm = Bm + LD(eR) * R * (aK @ np.abs(_solve(S, v[:, None])[:, 0]))
        return Result(m1, P1, Bm, _sym(BP))

    def _post(self, r, only_current, symmetrize):
        _normalize(r.m, r.Bm, quaternion_offsets(self.trail, only_current))
        if symmetrize:
            r.P = _sym(r.P)
        return r

    @staticmethod
    def _selector(n, l, cols):
        H = np.zeros((n, l), dtype=LD)
        H[np.arange(n), cols] = 1
        return H

    # ---- the fixed-H updates (ekf.cpp:573-677). R as the host forms it; normalisation / symmetrisation as update() / the op does.
    def zupt(self, m, P, r):
        r_ = self._update(m, P, self._selector(3, VEL + 3, [VEL, VEL + 1, VEL + 2]), y=np.zeros(3), R=np.float64(r) * self.ns)
        return self._post(r_, True, False)

    def zupt_initialization(self, m, P, time, fault=None):
        R = LD(self.p.init_zupt_r) * LD(self.ns)
        if fault != "no_exp":
            R = R * np.exp(LD(0.5) * LD(time))
        r_ = self._update(m, P, self._selector(3, VEL + 3, [VEL, VEL + 1, VEL + 2]), y=np.zeros(3), R=R, eR=4 * U)
        return self._post(r_, True, False)

    def zrupt(self, m, P, xg):
        r_ = self._update(m, P, self._selector(3, BGA + 3, [BGA, BGA + 1, BGA + 2]), y=xg, R=np.float64(self.p.rotation_zupt_r) * self.ns)
        return self._post(r_, True, False)

    def pseudo_velocity(self, m, P, speed, r, fault=None):
        """None where the horizontal speed is <= 1e-7 (no-op, ekf.cpp:635-637)."""
        mv = np.asarray(m, dtype=LD)[VEL:VEL + 3]
        k = 3 if fault == "speed_3d" else 2
        h = np.sqrt(mv[:k] @ mv[:k])
        if h <= 1e-7:
            return None
        H = np.zeros((1, VEL + k), dtype=LD)
        H[0, VEL:VEL + k] = mv[:k] / h
        r_ = self._update(m, P, H, v=np.array([LD(speed) - h]), R=np.float64(r) * self.ns)
        # H and v come from the fp64 mean: |H| and h are within 2u of the exact ones; that is in l u |H| |m_l| of the mean bound and,
        # for P, in kappa(S) |K| |H| |P_l| with the 64u of C_UPD (the 2u of H are one more term of the HP product)
        return self._post(r_, True, False)

    def position(self, m, P, y, r):
        r_ = self._update(m, P, self._selector(3, POS + 3, [POS, POS + 1, POS + 2]), y=y, R=np.float64(r) * self.ns)
        return self._post(r_, True, True)

    def zero_height(self, m, P, r):
        r_ = self._update(m, P, self._selector(1, POS + 3, [POS + 2]), y=np.zeros(1), R=np.float64(r) * self.ns)
        return self._post(r_, True, True)

    def orientation(self, m, P, q, r):
        r_ = self._update(m, P, self._selector(4, ORI + 4, [ORI, ORI + 1, ORI + 2, ORI + 3]), y=q, R=np.float64(r) * self.ns)
        return self._post(r_, False, True)

    def normalize_quaternions(self, m, P, only_current):
        r_ = Result(np.array(m, dtype=LD), np.array(P, dtype=LD), np.zeros(self.N, dtype=LD), np.zeros((self.N, self.N), dtype=LD))
        return self._post(r_, only_current, False)

    # ---- the pose augmentation (ekf.cpp:848-885, 35-50)
    def augment_noise(self):
        """visAugQ's diagonal as the host forms it (fp64)."""
        p = self.p
        qp = np.float64(p.noise_initial_pos_trail) * np.float64(p.noise_initial_pos_trail) * self.ns
        qo = np.float64(p.noise_initial_ori_trail) * np.float64(p.noise_initial_ori_trail) * self.ns
        return np.array([qp] * 3 + [qo] * 4)

    def augment_prior(self, m, P, drop, sym_first=False, fault=None):
        """(m+, P+) = (A m, A P A' + visAugQ) in fp64 (exact: a copy and an addition to zero), after the deferred symmetrisation."""
        drop = self.trail - 1 if drop == -1 else drop
        if fault == "drop_off_by_one":
            drop = drop + 1 if drop + 1 < self.trail else drop - 1
        P = np.asarray(P, np.float64)
        if sym_first and fault != "sym_first_skipped":
            P = symmetrize_fp64(P)
        m2, P2 = shift_fp64(m, P, aug_src(self.N, drop))
        q = self.augment_noise()
        slot = NEW + (POSE if fault == "noise_wrong_slot" else 0)
        for k in range(POSE):
            if fault == "noise_position_only" and k >= 3:
                continue
            P2[slot[k], slot[k]] += q[k]
        return m2, P2

    def augment(self, m, P, drop=-1, sym_first=False, form="closed", fault=None):
        mp, Pp = self.augment_prior(m, P, drop, sym_first, fault)
        N = self.N
        R = LD(np.float64(self.p.augment_r) * self.ns)
        m_, P_ = np.array(mp, dtype=LD), np.array(Pp, dtype=LD)
        HP = P_[CUR] - P_[NEW]                                              # visAugH P+
        S = _sym(HP[:, CUR] - HP[:, NEW]) + R * np.eye(POSE, dtype=LD)
        W = _solve(S, HP)                                                   # K'
        K = W.T
        v = -(m_[CUR] - m_[NEW])
        if form == "joseph":
            H = np.zeros((POSE, N), dtype=LD)
            H[np.arange(POSE), CUR] = 1
            H[np.arange(POSE), NEW] = -1
            T1 = np.eye(N, dtype=LD) - K @ H
            P1 = T1 @ P_ @ T1.T + R * (K @ K.T)
            m1 = m_ + K @ v
        else:
            # the closed form rests on P+ = P+' and on the new slot having no prior cross-covariance (the Joseph form of an asymmetric P+
            # differs from it by the asymmetry)
            Qd = np.diag(P_[NEW, NEW])
            if (P_[NEW] != 0).sum() != POSE or (P_[np.ix_(NEW, NEW)] != Qd).any() or (P_ != P_.T).any():
                raise AssertionError("the closed form needs a symmetric P+ without prior cross-covariance of the new slot")
            SinvPa = _solve(S, P_[CUR])
            P1 = P_ - P_[:, CUR] @ SinvPa
            QS = Qd @ _inv(S)
            P1[np.ix_(NEW, NEW)] = QS @ (P_[np.ix_(CUR, CUR)] + R * np.eye(POSE, dtype=LD))
            other = np.setdiff1d(np.arange(N), NEW)
            P1[np.ix_(NEW, other)] = QS @ P_[np.ix_(CUR, other)]
            P1[np.ix_(other, NEW)] = P1[np.ix_(NEW, other)].T
            Sm = _solve(S, m_[CUR][:, None])[:, 0]
            m1 = m_ - P_[:, CUR] @ Sm
            m1[NEW] = QS @ m_[CUR]
        P1 = _sym(P1)
        # bound: kappa(S) (|T1| (|P+| + |K| |H| |P+|) |T1|' + |K| R |K|'), |T1| = I except in the 14 special columns (F)
        kap = _cond(S)
        aK = np.abs(K)
        X = np.abs(P_) + aK @ (np.abs(P_[CUR]) + np.abs(P_[NEW]))
        F = np.abs(np.eye(N, dtype=LD)[:, SPECIAL] - np.concatenate([K, -K], axis=1))   # |T1[:, special]|
        E1 = F @ X[SPECIAL]
        Y = X.copy()
        Y[SPECIAL] = 0
        Y = Y + E1
        YF = Y[:, SPECIAL] @ F.T
        M = Y.copy()
        M[:, SPECIAL] = 0
        M = M + YF
        KRK = R * (aK @ aK.T)
        touched = (E1 + YF + aK @ (np.abs(P_[CUR]) + np.abs(P_[NEW])) + KRK) != 0
        BP = np.where(touched, C_AUG * U * kap * (M + KRK), LD(0))
        Xm = aK @ np.abs(v)
        Bm = np.where(Xm != 0, C_AUG * U * kap * (np.abs(m_) + Xm), LD(0))
        r_ = Result(m1, P1, Bm, _sym(BP))
        return self._post(r_, False, True)

    def augment_plain_fp64(self, m, P, drop=-1, sym_first=False):
        """Fault: the augmentation with the plain downdate P+ - K HP instead of the Joseph form, in fp64."""
        mp, Pp = self.augment_prior(m, P, drop, sym_first)
        R = np.float64(self.p.augment_r) * self.ns
        HP = Pp[CUR] - Pp[NEW]
        S = HP[:, CUR] - HP[:, NEW] + R * np.eye(POSE)
        W = np.linalg.solve(S, HP)
        m1 = mp + W.T @ (-(mp[CUR] - mp[NEW]))
        P1 = symmetrize_fp64(Pp - HP.T @ W)
        for o in quaternion_offsets(self.trail, False):
            z = m1[o:o + 4] @ m1[o:o + 4]
            if z > 0:
                m1[o:o + 4] /= np.sqrt(z)
        return m1, P1

    # ---- structural operations
    def transform_to(self, m, P, pos, q1, pi, fault=None):
        """transformTo (ekf.cpp:704-758): block rotations A (trailRotationA) on P and m, then translateTo(position + t)."""
        m0, P0 = np.array(m, dtype=LD), np.array(P, dtype=LD)
        q1 = np.asarray(q1, dtype=LD)
        o = ORI if pi < 0 else CAM + POSE * pi + 3
        p = POS if pi < 0 else CAM + POSE * pi
        q0, rp = m0[o:o + 4], m0[p:p + 3]

        def hamilton(a, b, absolute=False):
            aw, ax, ay, az = a
            bw, bx, by, bz = b
            if absolute:
                return np.array([aw * bw + ax * bx + ay * by + az * bz, aw * bx + ax * bw + ay * bz + az * by,
                                 aw * by + ay * bw + az * bx + ax * bz, aw * bz + az * bw + ax * by + ay * bx], dtype=LD)
            return np.array([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                             aw * by + ay * bw + az * bx - ax * bz, aw * bz + az * bw + ax * by - ay * bx], dtype=LD)

        def blocks(qc, absolute=False):
            s = 1 if absolute else -1
            p1, p2, p3, p4 = qc
            Qm = np.array([[p1, s * p2, s * p3, s * p4], [p2, p1, p4, s * p3], [p3, s * p4, p1, p2], [p4, p3, s * p2, p1]], dtype=LD)
            tx, ty, tz = 2 * qc[1], 2 * qc[2], 2 * qc[3]
            twx, twy, twz, txx, txy, txz = tx * qc[0], ty * qc[0], tz * qc[0], tx * qc[1], ty * qc[1], tz * qc[1]
            tyy, tyz, tzz = ty * qc[2], tz * qc[2], tz * qc[3]
            R = np.array([[1 + s * (tyy + tzz), txy + s * twz, txz + twy], [txy + twz, 1 + s * (txx + tzz), tyz + s * twx],
                          [txz + s * twy, tyz + twx, 1 + s * (txx + tyy)]], dtype=LD)
            return Qm, (R if fault == "transposed_rotation" and not absolute else R.T)

        conj = np.array([q0[0], -q0[1], -q0[2], -q0[3]], dtype=LD)
        Qm, Pc = blocks(hamilton(conj, q1))
        Qa, Pa = blocks(hamilton(np.abs(conj), np.abs(q1), absolute=True), absolute=True)
        starts = [(POS, 0), (VEL, 0), (ORI, 1)] + [(CAM + POSE * k + d, kind) for k in range(self.trail) for d, kind in ((0, 0), (3, 1))]
        mats = [(Pc, Qm), (Pa, Qa)]

        def apply(X, absolute, side):
            Y = X.copy()
            for s, kind in starts:
                Mx = mats[absolute][0] if kind == 0 else mats[absolute][1]
                k = Mx.shape[0]
                if side == "left":
                    Y[s:s + k] = Mx @ X[s:s + k]
                else:
                    Y[:, s:s + k] = X[:, s:s + k] @ Mx.T
            return Y

        P1 = apply(apply(P0, 0, "left"), 0, "right")
        m1 = apply(m0[:, None], 0, "left")[:, 0]
        aP = apply(apply(np.abs(P0), 1, "left"), 1, "right")
        am = apply(np.abs(m0)[:, None], 1, "left")[:, 0]
        rot = np.zeros(self.N, dtype=bool)
        for s, kind in starts:
            rot[s:s + (3 if kind == 0 else 4)] = True
        BP = np.where(rot[:, None] | rot[None, :], C_XF * U * aP, LD(0))
        Bm = np.where(rot, C_XF * U * am, LD(0))
        t = np.asarray(pos, dtype=LD) - Pc @ rp
        bt = C_XF * U * (np.abs(np.asarray(pos, dtype=LD)) + Pa @ np.abs(rp) + np.abs(m1[POS:POS + 3]))
        for s in [POS] + [CAM + POSE * k for k in range(self.trail)]:
            m1[s:s + 3] += t
            Bm[s:s + 3] += bt + C_XF * U * np.abs(m1[s:s + 3])
        return Result(m1, P1, Bm, _sym(BP))

    def condition_on_last_pose(self, m, P, fault=None):
        """conditionOnLastPose (ekf.cpp:928-942)."""
        P0 = np.array(P, dtype=LD)
        N, mm = self.N, self.N - POSE
        B = P0[mm:, mm:]
        Binv = np.diag(1 / np.diag(B)) if fault == "diag_binv" else _inv(B)
        Pab, Pba = P0[:mm, mm:], P0[mm:, :mm]
        P1 = np.zeros_like(P0)
        P1[:mm, :mm] = P0[:mm, :mm] - (Pab @ Binv) @ Pba
        P1[mm:, mm:] = LD(1e6) * np.eye(POSE, dtype=LD)
        X = np.abs(Pab) @ np.abs(_inv(B)) @ np.abs(Pba)
        BP = np.zeros_like(P0)
        BP[:mm, :mm] = np.where(X != 0, C_COND * U * _cond(B) * (np.abs(P0[:mm, :mm]) + X), LD(0))
        return Result(np.array(m, dtype=LD), P1, np.zeros(N, dtype=LD), _sym(BP))

    # ---- the operations an fp64 implementation reproduces bit for bit
    def unaugment_fp64(self, m, P):
        """updateUndoAugmentation (ekf.cpp:888-903): the trail moves up one slot, the last one becomes zero."""
        i = np.arange(self.N)
        ptd = self.N - MAPPT * self.map_size
        src = np.where(i < CAM, i, np.where(i >= ptd, i, np.where(i + POSE < ptd, i + POSE, -1)))
        return shift_fp64(m, P, src)

    def lock_biases_fp64(self, m, P):
        P = np.array(P, np.float64)
        P[BGA:BGA + 9] = 0
        P[:, BGA:BGA + 9] = 0
        return np.array(m, np.float64), P

    def insert_map_point_fp64(self, m, P, idx, pf):
        off = self.N - MAPPT * self.map_size + idx * MAPPT
        m, P = np.array(m, np.float64), np.array(P, np.float64)
        P[off:off + 3] = 0
        P[:, off:off + 3] = 0
        for k in range(3):
            P[off + k, off + k] = 1e3 * 1e3
            m[off + k] = pf[k]
        return m, P

    def translate_to_fp64(self, m, pos):
        m = np.array(m, np.float64)
        d = np.asarray(pos, np.float64) - m[POS:POS + 3]
        for s in [POS] + [CAM + POSE * k for k in range(self.trail)]:
            m[s:s + 3] += d
        return m


# ------------------------------------------------------------------------------------------------ states and operations of the tests
Q_ORI = np.array([0.9, 0.1, -0.2, 0.3]) / np.linalg.norm([0.9, 0.1, -0.2, 0.3])
Q_XF = np.array([0.7, -0.1, 0.2, 0.6]) / np.linalg.norm([0.7, -0.1, 0.2, 0.6])



def start_state(backend, kind):
    """(m, P, time) of a starting state, exactly symmetric, uploaded into the back end (oracle or CUDA):
    fresh: initialize_orientation and six predicts (the 1e8 trail priors, the cancellation case of the augmentation);
    filled: the trail filled by tests/ekf_script.run_frames; dense: predict_ref.dense_state (every entry O(1) relative to its
    variables, quaternion of norm 1.05)."""
    t = 0.0
    if kind == "fresh":
        backend.initialize_orientation(PR.ACC0)
        rng = np.random.RandomState(4)
        for k in range(7):
            t = 0.005 * (k + 1)
            backend.predict(t, *ekf_script.imu_sample(rng, k))
        backend.normalize_quaternions(True)
        m, P = backend.download()
        t -= 0.005
    elif kind == "filled":
        frames = backend.params.camera_trail_length + 2
        t = ekf_script.run_frames(backend, frames=frames, n_list=(8, 20)) - 0.005
        m, P = backend.download()
    else:
        m, P = PR.dense_state(backend.N)
    P = symmetrize_fp64(P)
    backend.upload(m, P)
    return m, P, t



def fixed_h_ops(ops, m, P, time):
    """(name, backend call, reference) of the fixed-H updates and the structural ops with a bound."""
    g = np.array([0.01, -0.02, 0.2])
    out = [("zupt_initialization", lambda b: b.update_zupt_initialization(), lambda: ops.zupt_initialization(m, P, time)),
           ("zupt", lambda b: b.update_zupt(1e-2), lambda: ops.zupt(m, P, 1e-2)),
           ("zrupt", lambda b: b.update_zrupt(g), lambda: ops.zrupt(m, P, g)),
           ("position", lambda b: b.update_position([0.1, -0.2, 0.05], 1e-3), lambda: ops.position(m, P, [0.1, -0.2, 0.05], 1e-3)),
           ("zero_height", lambda b: b.update_zero_height(1e-3), lambda: ops.zero_height(m, P, 1e-3)),
           ("orientation", lambda b: b.update_orientation(Q_ORI, 1e-2), lambda: ops.orientation(m, P, Q_ORI, 1e-2)),
           ("normalize_all", lambda b: b.normalize_quaternions(False), lambda: ops.normalize_quaternions(m, P, False))]
    if np.hypot(m[VEL], m[VEL + 1]) > 1e-7:
        out.append(("pseudo_velocity", lambda b: b.update_pseudo_velocity(0.7, 1.0), lambda: ops.pseudo_velocity(m, P, 0.7, 1.0)))
    for pi in sorted({-1, 0, ops.trail - 1}):
        out.append((f"transform_to[{pi}]", lambda b, pi=pi: b.transform_to([0.5, -0.5, 0.25], Q_XF, pi),
                    lambda pi=pi: ops.transform_to(m, P, [0.5, -0.5, 0.25], Q_XF, pi)))
    if ops.map_size == 0:
        # (an augmentation first: the filter needs an augmented pose; the upload restores the state)
        out.append(("condition_on_last_pose", lambda b: (b.augment(-1), b.upload(m, P), b.condition_on_last_pose()),
                    lambda: ops.condition_on_last_pose(m, P)))
    return out



# ------------------------------------------------------------------------------------------------ kernel paths
FIXED_H = {"zupt": (3, 6), "zrupt": (3, 13), "pseudo_velocity": (1, 5), "position": (3, 3), "zero_height": (1, 3), "orientation": (4, 10)}


def update_kernel(op, N):
    """The kernel a fixed-H update (FIXED_H: n rows, l columns) or the augmentation (op == "augment", n = 7, l = 27, Joseph form)
    launches on an N-dimensional state (kalman_ref.cluster_fits, the launcher's predicate)."""
    import kalman_ref as K
    n, l = (7, 27) if op == "augment" else FIXED_H[op]
    joseph = op == "augment"
    return "ekf_update_cluster2_kernel" if K.cluster_fits(n, l, N, joseph) else "ekf_update_kernel"
