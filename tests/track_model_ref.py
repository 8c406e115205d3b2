"""Plain extended-precision reference of the per-track measurement model (hybvio_b200/csrc/track_model.cuh), with a per-entry
tolerance that the reference measures itself, and the track sweep the tests around it run.

The model is restated in np.longdouble (80-bit on x86-64: 64-bit mantissa) from the equations oracle/hv_oracle_tri.c cites:
  pose trail of the observing cameras          extractCameraPoseTrail, triangulation.cpp:65-103
  two-view start                               triangulateWithTwoCameras, triangulation.cpp:610-710: pinv of the 3x2 ray matrix
                                               (triangulation.cpp:1000-1004) from a re-orthogonalised QR, dpinv (Golub & Pereyra 1973,
                                               eq. 4.12; triangulation.cpp:32-51)
  Gauss-Newton in inverse depth                Triangulator::triangulate, triangulation.cpp:120-407, with the FULL product rule of the
                                               residual block per (observation, derivative column), as the reference writes it
                                               (triangulation.cpp:216-318). The kernel instead splits every column into a generic part
                                               and an explicit part; comparing against the full rule checks that restructuring too.
  3x3 solves                                   Eigen's pivoted LDL^T (Eigen/src/Cholesky/LDLT.h) and the Hager / Higham rcond estimate
                                               (Eigen/src/Core/ConditionEstimator.h), so that BAD_COND is decided on the same number
  convergence                                  |dJ / J| < convergence_threshold, J = 0.5 |e|^2 / convergence_r^2 (:337-345)
  back from inverse depth                      triangulation.cpp:359-395. Like the reference, it leaves out the dependence of the first
                                               camera's position on the first pose's quaternion through the lever arm (-dR0' baseline);
                                               tests/test_oracle_tri.py documents that omission.
  behind test                                  isBehind, triangulation.cpp:53-59
  stereo sum                                   backend.cpp:1105-1116
  prepareVisualUpdate (truncated)              triangulation.cpp:897-987: H (2 n_obs x l), f, rows, cols

All six camera-model parameters (gauss_newton_iterations, convergence_threshold, convergence_r, rcond_threshold, min_dist,
max_dist), the trail length and the state dimension N are arguments.

The depth gate (backend.cpp:1095-1098). The reading implemented here: depth = |pf - p_0| is computed from whatever pf holds after
triangulate() returns, and depth < min_dist or depth > max_dist sets BAD_DEPTH whatever status triangulate() returned. The gate sits
between the triangulation and the block that drops the derivatives of a failed track (backend.cpp:1100-1104), so it sees every
status, and the reference's own shim (oracle/ref_build/ref_tri_shim.cpp) computes the depth the same way for every status. On
failure pf is the two-view point, in the camera frame of observation 0, while p_0 is that camera's position in the world frame;
the "depth" of a failed track is therefore not a distance, but it is what the gate reads. The kernel applies the gate in the same
way (track_model.cuh, after the behind test). The statuses it replaces are recorded in the decision trace.

Tolerance: a rounding-perturbation ensemble. A closed-form componentwise bound carried through ten Gauss-Newton iterations grows
like (1 + kappa)^iterations, while the actual error does not (the Gauss-Newton map and the derivative recurrence contract). So the
reference evaluates itself K_RUNS more times, seeded; in each run every stored intermediate (each matrix or vector a formula step
produces: products, sums, quotients, the factor and the solves) is multiplied by (1 + delta) with delta uniform in [-2^-53, 2^-53],
one fresh delta per entry. sigma_ij = max over the runs of |r_k - r_0| measures how much one fp64 rounding per stored intermediate
moves entry ij, through every cancellation the formulas contain. The tolerance is C_TOL * sigma_ij.

C_TOL = 64, fixed before any kernel result was looked at:
  * an fp64 evaluation rounds every intermediate once or, inside an inner product of k terms, up to k times (the kernel's sums over
    n_obs <= 42 observations, taken in a different order: a factor of up to ~6 in the typical sqrt(k) growth of independent roundings);
  * the kernel stores intermediates the reference does not (the generic / explicit split of every derivative column, the merged
    solve of the derivative update): their roundings enter the result through the same cancellations, with a gain that can exceed
    the reference's by a small factor (~4 allowed);
  * with K_RUNS = 8 independent draws the maximum of |r_k - r_0| falls below the largest response to deltas of the same size by at
    most a factor of ~2 on a single entry; C_TOL covers the product 6 * 4 * 2 ~ 48, rounded up to a power of two.
The injected faults the tests require (1e-8 and 1e-6 relative on single columns, structural ones) are 1e4 and more above this
level. Where sigma is 0 the entry must be exact: structural zeros of H and dpf (poses a track does not touch, the time-shift column
with the time shift off) and entries copied through unchanged. The reference's own error (u = 2^-64 per operation) is 2^-11 of
sigma for the same sensitivity.

Decision trace. Each run records (iterations, converged, BAD_COND, behind, UNKNOWN_PROBLEM, BAD_DEPTH, prepareVisualUpdate status).
LDL^T pivot choices are not part of it: a flip only moves rounding. A case is decided when every run's trace equals the unperturbed
one. The sweep's cases must be decided. A boundary case (a threshold placed at the reference's own number) may be undecided: the
kernel's status must then be one of the ensemble's, and its values must lie within the tolerance of an ensemble forced to follow a
trace with that status (Reference.forced)."""
import numpy as np

import tri_common

LD = np.longdouble
assert np.finfo(LD).nmant >= 63, "track_model_ref needs an extended-precision long double (x86-64 80-bit or wider)"
U = 2.0 ** -53                  # unit roundoff of the fp64 implementations under test
DBL_EPS = np.finfo(np.float64).eps
DBL_MIN = np.finfo(np.float64).tiny
K_RUNS = 8
C_TOL = 64.0
POS, ORI, SFT, CAM, POSE = 0, 6, 19, 20, 7
MAXPOSE = 21                    # TM_MAXPOSE: cameraTrailLength 20 + the current pose
MAXN = 20 + 7 * (MAXPOSE - 1)   # TM_MAXN: the widest H a track can have
OK, HYBRID, BEHIND, BAD_COND, NO_CONVERGENCE, BAD_DEPTH, UNKNOWN_PROBLEM = range(7)
VU_OK, VU_ZERO_DEPTH, VU_BEHIND, VU_NOT_RUN = 0, 1, 2, -1
DEFAULTS = dict(gauss_newton_iterations=10, convergence_threshold=1e-2, convergence_r=11.0, rcond_threshold=1e-8, min_dist=0.0,
                max_dist=1e300)
OUTPUTS = ("pf", "depth", "dpf", "H", "f")
FAULTS = ("dpf_pose0_position", "H_time_column", "H_smallest_column", "skip_converging_derivative_update", "drop_obs_32_up",
          "camera1_own_quaternion_with_camera0_baseline")


# ------------------------------------------------------------------------------------------------ rounding perturbation
class _Rounding:
    """x -> x (1 + delta), delta uniform in [-U, U] per entry; the identity for the unperturbed run."""

    def __init__(self, rng):
        self.rng = rng

    def __call__(self, x):
        x = np.asarray(x, dtype=LD)
        if self.rng is None:
            return x
        return x + x * (self.rng.random(x.shape) * (2 * U) - U)


def _quat(q):
    """R(q) and dR / dq_a (src/odometry/util.cpp:10-47), row-major."""
    q0, q1, q2, q3 = q
    R = np.array([[q0 * q0 + q1 * q1 - q2 * q2 - q3 * q3, 2 * q1 * q2 - 2 * q0 * q3, 2 * q1 * q3 + 2 * q0 * q2],
                  [2 * q1 * q2 + 2 * q0 * q3, q0 * q0 - q1 * q1 + q2 * q2 - q3 * q3, 2 * q2 * q3 - 2 * q0 * q1],
                  [2 * q1 * q3 - 2 * q0 * q2, 2 * q2 * q3 + 2 * q0 * q1, q0 * q0 - q1 * q1 - q2 * q2 + q3 * q3]], dtype=LD)
    a, b, c, d = 2 * q0, 2 * q1, 2 * q2, 2 * q3
    dR = np.array([[[a, -d, c], [d, a, -b], [-c, b, a]], [[b, c, d], [c, -b, -a], [d, a, -b]],
                   [[-c, b, a], [b, c, d], [-a, d, -c]], [[-d, -a, b], [a, -d, c], [b, c, d]]], dtype=LD)
    return R, dR


def _inverse_depth(p, rd):
    """(x, y, z) -> (x, y, 1) / z and its Jacobian (triangulation.cpp:1006-1030); p (..., 3)."""
    z = p[..., 2]
    ip = rd(np.stack([p[..., 0] / z, p[..., 1] / z, LD(1) / z], axis=-1))
    dip = np.zeros(p.shape[:-1] + (3, 3), dtype=LD)
    dip[..., 0, 0] = LD(1) / z
    dip[..., 1, 1] = LD(1) / z
    for i in range(3):
        dip[..., i, 2] = -ip[..., i] / z
    return ip, rd(dip)


def _norm(x):
    return np.sqrt(np.sum(x * x, axis=-1))


def _pinv32(A, rd):
    """Moore-Penrose inverse of a 3 x 2 matrix from a column-pivoted, re-orthogonalised QR (rank threshold 2 eps, as Eigen's
    completeOrthogonalDecomposition); A (3, 2) -> (2, 3)."""
    c = [A[:, 0], A[:, 1]]
    a = 1 if _norm(c[1]) > _norm(c[0]) else 0
    b = 1 - a
    r11 = _norm(c[a])
    q1 = c[a] / r11
    r12 = q1 @ c[b]
    u = c[b] - r12 * q1
    r12b = q1 @ u
    u = u - r12b * q1
    r12 = r12 + r12b
    r22 = _norm(u)
    iA = np.zeros((2, 3), dtype=LD)
    if r22 <= 2 * DBL_EPS * r11:
        s = r11 * r11 + r12 * r12
        iA[a] = r11 * q1 / s
        iA[b] = r12 * q1 / s
        return rd(iA)
    q2 = u / r22
    iA[b] = q2 / r22
    iA[a] = (q1 - r12 * q2 / r22) / r11
    return rd(iA)


def _dpinv32(A, iA, dA, rd):
    """d pinv(A) for dA (J, 3, 2): -iA dA iA + (iA iA') dA' (I - A iA) + (I - iA A) dA' (iA' iA)."""
    dAT = np.swapaxes(dA, -1, -2)
    t1 = rd(rd(iA @ dA) @ iA)
    P3 = rd(np.eye(3, dtype=LD) - rd(A @ iA))
    G2 = rd(iA @ iA.T)
    t2 = rd(rd(G2 @ dAT) @ P3)
    P2 = rd(np.eye(2, dtype=LD) - rd(iA @ A))
    G3 = rd(iA.T @ iA)
    w = rd(rd(P2 @ dAT) @ G3)
    return rd(-t1 + t2 + w)


# ------------------------------------------------------------------------------------------------ LDL^T and rcond
class _Ldlt:
    """Eigen's LDLT (lower, unblocked, diagonal pivoting on the remaining ORIGINAL diagonal) of a 3 x 3 self-adjoint matrix."""

    def __init__(self, A, rd):
        M = np.array(A, dtype=LD)
        self.l1 = max(sum(abs(M[r, c]) for r in range(c, 3)) + sum(abs(M[c, k]) for k in range(c)) for c in range(3))
        tp = [0, 1, 2]
        stop = False
        for k in range(3):
            big = k
            for i in range(k + 1, 3):
                if abs(M[i, i]) > abs(M[big, big]):
                    big = i
            tp[k] = big
            if big != k:
                for c in range(k):
                    M[k, c], M[big, c] = M[big, c], M[k, c]
                for r in range(big + 1, 3):
                    M[r, k], M[r, big] = M[r, big], M[r, k]
                M[k, k], M[big, big] = M[big, big], M[k, k]
                for i in range(k + 1, big):
                    M[i, k], M[big, i] = M[big, i], M[i, k]
            temp = [M[c, c] * M[k, c] for c in range(k)]
            for c in range(k):
                M[k, k] -= M[k, c] * temp[c]
            for r in range(k + 1, 3):
                for c in range(k):
                    M[r, k] -= M[r, c] * temp[c]
            akk = M[k, k]
            if k == 0 and not abs(akk) > 0:
                tp = [0, 1, 2]
                stop = True
                break
            if abs(akk) > 0:
                for r in range(k + 1, 3):
                    M[r, k] /= akk
        if not stop:
            M = rd(M)
        self.M, self.tp, self.rd = M, tp, rd

    def solve(self, rhs):
        """rhs (3,) or (3, J)."""
        M, tp = self.M, self.tp
        v = np.array(rhs, dtype=LD)
        for k in range(3):
            if tp[k] != k:
                v[[k, tp[k]]] = v[[tp[k], k]]
        for r in range(1, 3):
            for c in range(r):
                v[r] = v[r] - M[r, c] * v[c]
        for i in range(3):
            v[i] = v[i] / M[i, i] if abs(M[i, i]) > DBL_MIN else LD(0) * v[i]
        for r in (1, 0):
            for c in range(r + 1, 3):
                v[r] = v[r] - M[c, r] * v[c]
        for k in (2, 1, 0):
            if tp[k] != k:
                v[[k, tp[k]]] = v[[tp[k], k]]
        return self.rd(v)

    def rcond(self):
        """Hager's 1-norm estimate of the inverse with Higham's alternating-sign safeguard (Eigen's LDLT::rcond)."""
        if self.l1 == 0:
            return LD(0)
        v = self.solve(np.full(3, LD(1) / 3))
        lower = np.sum(np.abs(v))
        old_lower, jmax, old_jmax, old_sgn = lower, -1, -1, None
        for k in range(4):
            sgn = np.where(v < 0, LD(-1), LD(1))
            if k > 0 and np.array_equal(sgn, old_sgn):
                break
            v = self.solve(sgn)
            jmax = int(np.argmax(np.abs(v)))
            if jmax == old_jmax:
                break
            e = np.zeros(3, dtype=LD)
            e[jmax] = 1
            v = self.solve(e)
            lower = np.sum(np.abs(v))
            if lower <= old_lower:
                break
            old_sgn, old_jmax, old_lower = sgn, jmax, lower
        a = self.solve(np.array([1.0, -1.5, 2.0], dtype=LD))
        alt = 2 * np.sum(np.abs(a)) / 9
        inv = lower if lower > alt else alt
        return LD(0) if inv == 0 else self.rd((LD(1) / inv) / self.l1)


# ------------------------------------------------------------------------------------------------ the model
def pose_offsets(i):
    """getPosOriIndices (triangulation.cpp:989-998): state offsets of pose-trail index i (0 = current pose)."""
    return (POS, ORI) if i == 0 else (CAM + POSE * (i - 1), CAM + POSE * (i - 1) + 3)


def truncation(idx):
    """The column count l of prepareVisualUpdate(truncated) (triangulation.cpp:909-921)."""
    return max(max(p + 3, o + 4) for p, o in (pose_offsets(int(i)) for i in idx))


class Track:
    """One track and the state it is modelled against: m (N), trail, stereo, idx (npose), T1 / T2 (4 x 4 imuToCamera, row-major
    numpy), ip / vel (n_obs x 2: camera 0 poses, then camera 1), time_shift, params (DEFAULTS overridden)."""

    def __init__(self, m, trail, stereo, idx, T1, T2, ip, vel, time_shift=True, params=None, label=""):
        self.m = np.asarray(m, np.float64)
        self.trail, self.stereo, self.time_shift, self.label = int(trail), bool(stereo), bool(time_shift), label
        self.idx = np.asarray(idx, np.int32)
        self.T1, self.T2 = np.asarray(T1, np.float64), np.asarray(T2 if T2 is not None else T1, np.float64)
        self.ip = np.asarray(ip, np.float64).reshape(-1, 2)
        self.vel = np.asarray(vel, np.float64).reshape(-1, 2)
        self.params = dict(DEFAULTS, **(params or {}))
        self.N = len(self.m)
        self.npose = len(self.idx)
        self.nobs = self.npose * (2 if self.stereo else 1)
        assert 2 <= self.npose <= MAXPOSE and self.idx[0] == 0 and self.N >= 20 + POSE * self.trail
        assert self.idx.max() <= min(self.trail, MAXPOSE - 1) and len(set(self.idx.tolist())) == self.npose
        assert self.ip.shape == (self.nobs, 2) and self.vel.shape == (self.nobs, 2)

    @property
    def rows(self):
        return 2 * self.nobs


def _pose_trail(t, rd):
    """R (n, 3, 3), dR (n, 4, 3, 3), p (n, 3), base (n, 3): camera 0 poses for every index, then camera 1."""
    R, dR, p, base = [], [], [], []
    for T in ([t.T1, t.T2] if t.stereo else [t.T1]):
        Rc, b = T[:3, :3].astype(LD), T[:3, 3].astype(LD)
        for i in t.idx:
            po, oo = pose_offsets(int(i))
            Rq, dRq = _quat(t.m[oo:oo + 4].astype(LD))
            Ri = rd(Rc @ rd(Rq))
            R.append(Ri)
            dR.append(rd(Rc @ dRq))
            p.append(rd(t.m[po:po + 3].astype(LD) - rd(Ri.T @ b)))
            base.append(b)
    return np.array(R), np.array(dR), np.array(p), np.array(base)


def _two_cameras(R, dR, p, ip0, ip1, vel0, vel1, ind1, time_shift, rd):
    """triangulateWithTwoCameras: pf (3, frame of observation 0) and its 15 derivative columns p0, q0, p1, q1, t."""
    R0, R1 = R[0], R[ind1]
    R1T = R1.T
    C = rd(R0 @ R1T)
    d = rd(p[ind1] - p[0])
    b = rd(R0 @ d)
    v0, v1 = np.array([ip0[0], ip0[1], 1.0], dtype=LD), np.array([ip1[0], ip1[1], 1.0], dtype=LD)
    n0, n1 = rd(_norm(v0)), rd(_norm(v1))
    vn0, vn1 = rd(v0 / n0), rd(v1 / n1)
    Cv = rd(C @ vn1)
    A = np.stack([vn0, -Cv], axis=1)
    iA = _pinv32(A, rd)
    s = rd(iA @ b)
    pf = rd(s[0] * vn0)
    dA = np.zeros((15, 3, 2), dtype=LD)
    db = np.zeros((15, 3), dtype=LD)
    for i in range(4):
        dA[3 + i, :, 1] = -rd(rd(dR[0, i] @ R1T) @ vn1)
        dA[10 + i, :, 1] = -rd(rd(R0 @ dR[ind1, i].T) @ vn1)
        db[3 + i] = rd(dR[0, i] @ d)
        if i < 3:
            db[i] = -R0[:, i]
            db[7 + i] = R0[:, i]
    diA = _dpinv32(A, iA, dA[:14], rd)
    x = rd(np.einsum("k,jk->j", iA[0], db[:14]))
    y = rd(diA[:, 0, :] @ b)
    dpf = np.zeros((15, 3), dtype=LD)
    dpf[:14] = rd(rd(x + y)[:, None] * vn0[None, :])
    if time_shift:
        w0, w1 = np.array([vel0[0], vel0[1], 0.0], dtype=LD), np.array([vel1[0], vel1[1], 0.0], dtype=LD)
        B0 = rd((np.eye(3, dtype=LD) - rd(np.outer(vn0, vn0))) / n0)
        B1 = rd((np.eye(3, dtype=LD) - rd(np.outer(vn1, vn1))) / n1)
        xs, ys = rd(B0 @ w0), rd(B1 @ w1)
        Cy = rd(C @ ys)
        dA14 = np.stack([xs, -Cy], axis=1)[None]
        ds = rd(_dpinv32(A, iA, dA14, rd)[0] @ b)
        dpf[14] = rd(rd(s[0] * xs) + rd(vn0 * ds[0]))
    return pf, dpf


def _explicit_columns(R, dR, p, base, n, rd):
    """dC (n, J, 3, 3) and dt (n, J, 3) of every (observation i, column j) for j < 7 n: the derivatives of C_i = R_i R_0' and
    t_i = R_i (p_0 - p_i) with respect to component j % 7 of pose j // 7 (non-zero only for i's own pose and for pose 0)."""
    J = POSE * n
    dC = np.zeros((n, J + 1, 3, 3), dtype=LD)
    dt = np.zeros((n, J + 1, 3), dtype=LD)
    R0T = R[0].T
    for i in range(n):
        dp = rd(p[0] - p[i])
        for pose in {i, 0}:
            for comp in range(POSE):
                j = POSE * pose + comp
                dRi = dR[i, comp - 3] if (pose == i and comp >= 3) else None
                dR0 = dR[0, comp - 3] if (pose == 0 and comp >= 3) else None
                dpi, dp0 = np.zeros(3, dtype=LD), np.zeros(3, dtype=LD)
                if comp < 3:
                    if pose == i:
                        dpi[comp] = 1
                    if pose == 0:
                        dp0[comp] = 1
                else:
                    if dRi is not None:
                        dpi = -rd(dRi.T @ base[i])
                    if dR0 is not None:
                        dp0 = -rd(dR0.T @ base[0])
                c = np.zeros((3, 3), dtype=LD)
                if dRi is not None:
                    c = c + rd(dRi @ R0T)
                if dR0 is not None:
                    c = c + rd(R[i] @ dR0.T)
                dC[i, j] = rd(c)
                tt = rd(R[i] @ rd(dp0 - dpi))
                if dRi is not None:
                    tt = rd(rd(dRi @ dp) + tt)
                dt[i, j] = tt
    return dC, dt


def evaluate(t, rng=None, force=None, fault=None):
    """One evaluation of the model (rng: the rounding perturbation, None for the unperturbed run). force: a decision trace to
    follow instead of deciding (Reference.forced). fault: one of FAULTS, for the comparator tests. Returns a dict with the outputs
    (status, vu_status, rows, cols, pf, depth, dpf (3 x (7 npose + 1)), H (rows x cols), f) and the decision trace."""
    rd = _Rounding(rng)
    prm = t.params
    npose, n = t.npose, t.nobs
    dDim = POSE * n
    R, dR, p, base = _pose_trail(t, rd)
    ip = t.ip.astype(LD)
    vel = t.vel.astype(LD)
    ind1 = n // 2 - 1 if t.stereo else n - 1

    # ---- two-view start, in inverse depth
    pf, d2 = _two_cameras(R, dR, p, ip[0], ip[ind1], vel[0], vel[ind1], ind1, t.time_shift, rd)
    pf2view = pf
    pfi, dpfi_dpf = _inverse_depth(pf, rd)
    dpfi = np.zeros((dDim + 1, 3), dtype=LD)
    cols2 = rd(d2 @ dpfi_dpf.T)
    dpfi[0:POSE] = cols2[0:POSE]
    dpfi[POSE * ind1:POSE * ind1 + POSE] = cols2[POSE:2 * POSE]
    dpfi[dDim] = cols2[14]

    # ---- Gauss-Newton with derivatives
    R0 = R[0]
    C = rd(R @ R0.T)                                                # C_i = R_i R_0'
    t_ = rd(np.einsum("irc,ic->ir", R, rd(p[0][None, :] - p)))      # t_i = R_i (p_0 - p_i)
    dC, dtc = _explicit_columns(R, dR, p, base, n, rd)
    extra = np.zeros((n, dDim + 1, 2), dtype=LD)
    if t.time_shift:
        extra[:, dDim, :] = vel
    conv_r = LD(prm["convergence_r"])
    Jprev = LD(1e10)
    converged, iters, rcond, X = False, 0, LD(0), None
    Jds = []
    n_iter = int(prm["gauss_newton_iterations"]) if force is None else force[0]
    keep = np.ones(n, bool)
    if fault == "drop_obs_32_up":
        keep[32:] = False
    for it in range(n_iter):
        iters = it + 1
        pfiab = np.array([pfi[0], pfi[1], 1.0], dtype=LD)
        h = rd(rd(C @ pfiab) + rd(pfi[2] * t_))
        h2 = h[:, 2]
        ih2sq = rd(LD(1) / rd(h2 * h2))
        err = rd(ip - rd(h[:, :2] / h2[:, None]))
        E = np.empty((n, 2, 3), dtype=LD)
        for r in range(2):
            E[:, r, :2] = rd(rd((-LD(1) / h2)[:, None] * C[:, r, :2]) + rd((h[:, r] * ih2sq)[:, None] * C[:, 2, :2]))
            E[:, r, 2] = rd(rd(-t_[:, r] / h2) + rd(h[:, r] * ih2sq * t_[:, 2]))
        ETE = rd(np.einsum("iac,iad->cd", E[keep], E[keep]))
        Eerror = rd(np.einsum("iac,ia->c", E[keep], err[keep]))
        error2 = rd(np.sum(err * err))
        # the full product rule per (observation, column) (triangulation.cpp:216-318)
        dq = dpfi                                                   # (J, 3)
        dpfiab = np.concatenate([dq[:, :2], np.zeros((dDim + 1, 1), dtype=LD)], axis=1)
        a_ = rd(np.einsum("ijrc,c->ijr", dC, pfiab))
        b_ = rd(np.einsum("irc,jc->ijr", C, dpfiab))
        dh = rd(a_ + b_ + rd(dq[None, :, 2, None] * t_[:, None, :]) + rd(pfi[2] * dtc))
        H2 = h2[:, None]
        dih2 = rd(-dh[..., 2] / rd(H2 * H2))
        dih2sq = rd(-2 * dh[..., 2] * ih2sq[:, None] / H2)
        dErr = rd(extra - rd(dh[..., :2] / H2[..., None]) - rd(dih2[..., None] * h[:, None, :2]))
        dE = np.empty((n, dDim + 1, 2, 3), dtype=LD)
        for r in range(2):
            k1 = rd(rd(dh[..., r] * ih2sq[:, None]) + rd(dih2sq * h[:, None, r]))
            hr = (h[:, r] * ih2sq)[:, None]
            dE[..., r, :2] = rd(rd(-dih2[..., None] * C[:, None, r, :2]) + rd((-LD(1) / H2)[..., None] * dC[:, :, r, :2])
                                + rd(k1[..., None] * C[:, None, 2, :2]) + rd(hr[..., None] * dC[:, :, 2, :2]))
            dE[..., r, 2] = rd(rd(-dtc[..., r] / H2) - rd(t_[:, None, r] * dih2) + rd(dh[..., r] * ih2sq[:, None] * t_[:, None, 2])
                               + rd(h[:, None, r] * dih2sq * t_[:, None, 2]) + rd(hr * dtc[..., 2]))
        if not t.time_shift:
            dErr[:, dDim] = 0
            dE[:, dDim] = 0
        dEerror = rd(np.sum(rd(np.einsum("ijac,ia->ijc", dE, err) + np.einsum("iac,ija->ijc", E, dErr)), axis=0))
        dETE = rd(np.sum(rd(np.einsum("ijac,iad->ijcd", dE, E) + np.einsum("iac,ijad->ijcd", E, dE)), axis=0))
        X = _Ldlt(ETE, rd)
        step = X.solve(Eerror)
        pfi_new = rd(pfi - step)
        w = rd(dETE @ step)                                         # (J, 3)
        u = X.solve(w.T).T
        g = X.solve(dEerror.T).T
        dpfi_new = rd(dpfi - g + u)
        J = rd(LD(0.5) * error2 / (conv_r * conv_r))
        Jd = rd(abs((J - Jprev) / J))
        Jds.append(Jd)
        Jprev = J
        conv = (Jd < prm["convergence_threshold"]) if force is None else (it + 1 == force[0] and force[1])
        pfi = pfi_new
        if not (conv and fault == "skip_converging_derivative_update"):
            dpfi = dpfi_new
        if conv:
            converged = True
            break
    rcond = X.rcond()
    bad_cond = None
    status = OK
    if not converged:
        status = NO_CONVERGENCE
    else:
        bad_cond = bool(rcond < prm["rcond_threshold"]) if force is None else force[2]
        if bad_cond:
            status = BAD_COND
    pf = pf2view
    behind = unknown = None
    dpf_all = None
    if status == OK:
        pf0, dpf0 = _inverse_depth(pfi, rd)
        pf = rd(rd(R0.T @ pf0) + p[0])
        unknown = bool(np.array_equal(pf.astype(np.float64), p[0].astype(np.float64)))
        if unknown:
            status = UNKNOWN_PROBLEM
        else:
            M = rd(R0.T @ dpf0)
            dpf_all = rd(dpfi @ M.T)
            for j in range(3, 7):
                dpf_all[j] = rd(rd(dR[0, j - 3].T @ pf0) + dpf_all[j])
            for r in range(3):
                dpf_all[r, r] = rd(dpf_all[r, r] + 1)
            cz = np.einsum("ic,ic->i", R[:, 2, :], rd(pf[None, :] - p))
            behind = bool((cz < 0).any())
            if behind:
                status = BEHIND
    depth = rd(_norm(rd(pf - p[0])))
    bad_depth = bool(depth < prm["min_dist"] or depth > prm["max_dist"]) if force is None else force[5]
    if bad_depth:
        status = BAD_DEPTH
    out = dict(status=status, vu_status=VU_NOT_RUN, rows=0, cols=0, pf=pf, depth=depth, Jds=Jds, rcond=rcond, iterations=iters,
               dpf=np.zeros((3, POSE * npose + 1), dtype=LD), H=np.zeros((0, 0), dtype=LD), f=np.zeros(0, dtype=LD))
    vu = VU_NOT_RUN
    if status == OK:
        # ---- stereo sum (backend.cpp:1105-1116)
        dpf = np.zeros((POSE * npose + 1, 3), dtype=LD)
        dpf[:POSE * npose] = dpf_all[:POSE * npose]
        if t.stereo:
            dpf[:POSE * npose] = rd(dpf[:POSE * npose] + dpf_all[POSE * npose:dDim])
        dpf[POSE * npose] = dpf_all[dDim]
        if fault == "dpf_pose0_position":
            dpf[0:3] = dpf[0:3] * LD(1 + 1e-8)
        out["dpf"] = dpf.T.copy()
        vu, H, f = _prepare_visual_update(t, R, dR, p, base, pf, dpf, vel, rd, fault)
        out.update(H=H, f=f, rows=H.shape[0], cols=H.shape[1])
        if vu != VU_OK:
            out.update(H=np.zeros((0, 0), dtype=LD), f=np.zeros(0, dtype=LD))
    out["vu_status"] = vu
    out["trace"] = (iters, converged, bad_cond, behind, unknown, bad_depth, vu)
    return out


def _prepare_visual_update(t, R, dR, p, base, pf, dpf, vel, rd, fault):
    """triangulation.cpp:897-987 with truncated = true. dpf ((7 npose + 1), 3) after the stereo sum."""
    npose, n = t.npose, t.nobs
    end = truncation(t.idx)
    H = np.zeros((2 * n, end), dtype=LD)
    f = np.zeros(2 * n, dtype=LD)
    pt = rd(pf[None, :] - p)
    pfc = rd(np.einsum("irc,ic->ir", R, pt))
    for i in range(n):
        if pfc[i, 2] == 0:
            return VU_ZERO_DEPTH, H, f
        if pfc[i, 2] < 0:
            return VU_BEHIND, H, f
    ipH, dipH = _inverse_depth(pfc, rd)
    f[:] = ipH[:, :2].reshape(-1)
    dipR = rd(dipH[:, :2, :] @ R)                                   # (n, 2, 3)
    cols = rd(np.einsum("irc,jc->irj", dipR, dpf))                  # (n, 2, 7 npose + 1): dipR d pf_j
    for i in range(n):
        k = i % npose
        po, oo = pose_offsets(int(t.idx[k]))
        bi = base[0] if (fault == "camera1_own_quaternion_with_camera0_baseline" and i >= npose) else base[i]
        own = np.zeros((2, POSE), dtype=LD)
        own[:, :3] = -dipR[i]
        for j in range(4):
            col = rd(rd(dR[i, j] @ pt[i]) + rd(R[i] @ rd(dR[i, j].T @ bi)))
            own[:, 3 + j] = rd(dipH[i, :2, :] @ col)
        for jj in range(npose):
            pj, oj = pose_offsets(int(t.idx[jj]))
            for c in range(POSE):
                dst = pj + c if c < 3 else oj + c - 3
                v = cols[i, :, POSE * jj + c]
                H[2 * i:2 * i + 2, dst] = rd(own[:, c] + v) if jj == k else v
        if t.time_shift:
            H[2 * i:2 * i + 2, SFT] = rd(cols[i, :, POSE * npose] - vel[i])
    if fault == "H_time_column":
        H[:, SFT] = H[:, SFT] * LD(1 + 1e-8)
    if fault == "H_smallest_column":
        mx = np.abs(H).max(axis=0)
        c = int(np.argmin(np.where(mx > 0, mx, np.inf)))
        H[:, c] = H[:, c] * LD(1 + 1e-6)
    return VU_OK, H, f


# ------------------------------------------------------------------------------------------------ the ensemble
def _arrays(o):
    return {k: np.atleast_1d(np.asarray(o[k], dtype=LD)) for k in OUTPUTS}


def status_of(trace):
    """(TriangulatorStatus, PrepareVuStatus) a decision trace leads to."""
    iters, conv, bad_cond, behind, unknown, bad_depth, vu = trace
    if bad_depth:
        return BAD_DEPTH, VU_NOT_RUN
    if not conv:
        return NO_CONVERGENCE, VU_NOT_RUN
    if bad_cond:
        return BAD_COND, VU_NOT_RUN
    if unknown:
        return UNKNOWN_PROBLEM, VU_NOT_RUN
    if behind:
        return BEHIND, VU_NOT_RUN
    return OK, vu


class Reference:
    """The unperturbed evaluation (out), the K_RUNS perturbed ones, sigma per output entry and the decision traces."""

    def __init__(self, t, seed=0, runs=K_RUNS, force=None):
        self.t, self.seed, self.force = t, seed, force
        self.out = evaluate(t, force=force)
        self.runs = [evaluate(t, rng=np.random.default_rng([seed, k]), force=force) for k in range(runs)]
        self.traces = [r["trace"] for r in self.runs]
        self.decided = all(tr == self.out["trace"] for tr in self.traces)
        self.statuses = {status_of(tr) for tr in [self.out["trace"]] + self.traces}
        base = _arrays(self.out)
        self.sigma = {k: np.zeros(v.shape, dtype=LD) for k, v in base.items()}
        for r in self.runs:
            if r["trace"] != self.out["trace"]:
                continue
            for k, v in _arrays(r).items():
                self.sigma[k] = np.maximum(self.sigma[k], np.abs(v - base[k]))

    @property
    def status(self):
        return self.out["status"], self.out["vu_status"]

    def forced(self, trace):
        """The ensemble made to follow `trace` in every run (for undecided boundary cases)."""
        return Reference(self.t, self.seed, len(self.runs), force=trace)

    def tol(self, k):
        return C_TOL * self.sigma[k]


def ratios_against(ref_out, sigma, dev, keys=OUTPUTS):
    """{output: worst |dev - ref| / (C_TOL sigma)} with sigma = 0 entries required exact (inf otherwise)."""
    out = {}
    base = _arrays(ref_out)
    for k in keys:
        d = np.atleast_1d(np.asarray(dev[k], dtype=np.float64))
        r = base[k]
        if d.shape != r.shape:
            out[k] = np.inf
            continue
        if not r.size:
            out[k] = 0.0
            continue
        err = np.abs(d.astype(LD) - r)
        tol = C_TOL * sigma[k]
        zero = tol == 0
        if (err[zero] != 0).any():
            out[k] = np.inf
            continue
        out[k] = float((err[~zero] / tol[~zero]).max()) if (~zero).any() else 0.0
    return out


def ratios(ref, dev, keys=OUTPUTS):
    """Worst |error| / tolerance per output of one device (or oracle) result against a decided Reference."""
    return ratios_against(ref.out, ref.sigma, dev, keys)


def compare(ref, dev, keys=OUTPUTS):
    """(ok, ratios, note) of one result: status, vu status, rows and cols equal and every output in `keys` within the tolerance.
    For an undecided reference the status must be one of the ensemble's and the values within the tolerance of an ensemble forced
    to follow a trace with that status."""
    st = (dev["tri_status"], dev["vu_status"])
    if ref.decided:
        r = ratios(ref, dev, keys)
        ok = st == ref.status and (dev.get("rows", ref.out["rows"]), dev.get("cols", ref.out["cols"])) == (ref.out["rows"], ref.out["cols"])
        return ok and max(r.values()) <= 1.0, r, "decided"
    if st not in ref.statuses:
        return False, {}, f"status {st} not among the ensemble's {sorted(ref.statuses)}"
    best = None
    for tr in sorted({tr for tr in [ref.out["trace"]] + ref.traces if status_of(tr) == st}, key=str):
        f = ref.forced(tr)
        r = ratios_against(f.out, f.sigma, dev, keys)
        if (dev.get("rows", f.out["rows"]), dev.get("cols", f.out["cols"])) != (f.out["rows"], f.out["cols"]):
            r = dict(r, rows=np.inf)
        if best is None or max(r.values()) < max(best[1].values()):
            best = (tr, r)
    return max(best[1].values()) <= 1.0, best[1], f"undecided, matched trace {best[0]}"


def oracle_result(o):
    """An oracle / golden-vector dict in the comparison's form (the oracle has no depth gate and reports vu -1 on failure)."""
    return dict(tri_status=o["tri_status"], vu_status=o["vu_status"], pf=o["pf"], depth=o["depth"], dpf=o["dpf"], H=o["H"],
                f=o["f"], rows=o["H"].shape[0], cols=o["H"].shape[1])


def old_gate_accepts(ref_out, dev):
    """The gate test_gpu_track_model.py applies: max|dev - ref| / max|ref| < 1e-9 per array (1e-6 once max|dpf| >= 1e6)."""
    def rel(a, b):
        a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
        return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)) if b.size else 0.0
    tol = 1e-9 if np.abs(np.asarray(ref_out["dpf"], np.float64)).max() < 1e6 else 1e-6
    return all(rel(dev[k], ref_out[k]) < tol for k in ("pf", "dpf", "H", "f"))


# ------------------------------------------------------------------------------------------------ the sweep
class Group:
    """Tracks that share one state, rig and parameter set: one launch of hv_ekf_track_models."""

    def __init__(self, name, base, trail, map_size, stereo, time_shift, params, tracks):
        self.name, self.base, self.trail, self.map_size = name, base, trail, map_size
        self.stereo, self.time_shift, self.params, self.tracks = stereo, time_shift, dict(DEFAULTS, **(params or {})), tracks

    @property
    def default_params(self):
        return self.params == DEFAULTS


def _state(seed, trail, map_size, stereo, static=False):
    base = tri_common.make_track(seed, trail=trail, npose=2, stereo=stereo)
    if static:
        tri_common.corrupt(base, "static", seed)
    if map_size:
        rng = np.random.RandomState(seed + 77)
        base["m"] = np.concatenate([base["m"], rng.normal(0, 3.0, 3 * map_size)])
    return base


def _track(base, npose, stereo, time_shift, params, rng, depth_scale=1.0, noise=1e-3, kind="none", label=""):
    """A new point seen from npose poses of base's state (indices up to min(trail, 20))."""
    top = min(base["trail"], MAXPOSE - 1)
    idx = np.concatenate([[0], np.sort(rng.choice(np.arange(1, top + 1), npose - 1, replace=False))]).astype(np.int32)
    T1, T2 = base["T1"], base["T2"]
    R0 = T1[:3, :3] @ tri_common.quat2rmat(base["m"][6:10])
    c0 = base["m"][0:3] - R0.T @ T1[:3, 3]
    pf = c0 + (base["pf_true"] - c0) * depth_scale + rng.normal(0, 0.05 * depth_scale, 3)
    ip = tri_common.project(base["m"], idx, T1, T2, stereo, pf) + rng.normal(0, noise, (len(idx) * (2 if stereo else 1), 2))
    vel = rng.normal(0, 0.05, ip.shape)
    d = dict(ip=ip, m=base["m"], trail=base["trail"])
    if kind != "none":
        tri_common.corrupt_observations(d, kind, int(rng.randint(1 << 20)))
    return Track(base["m"], base["trail"], stereo, idx, T1, T2, d["ip"], vel, time_shift, params, label or f"{npose}p-{kind}")


def _group(name, seed, trail=20, map_size=0, stereo=True, time_shift=True, params=None, nposes=(4, 9, 14), kinds=None,
           depths=(1.0,), static=False):
    base = _state(seed, trail, map_size, stereo, static)
    rng = np.random.RandomState(seed + 1)
    kinds = kinds or ["none"] * len(nposes)
    tracks = [_track(base, k, stereo, time_shift, params, rng, depths[i % len(depths)], kind=kinds[i]) for i, k in enumerate(nposes)]
    return Group(name, base, trail, map_size, stereo, time_shift, params, tracks)


def sweep_cases():
    """Groups of tracks (one state, rig and parameter set each) covering every pose count 2..21 mono and stereo with the time shift on
    and off, n_obs > 32 (rows > 64), every status the model returns except UNKNOWN_PROBLEM, trails 4, 8, 20, 30, a hybrid-map layout
    (N > TM_MAXN) and every camera-model parameter away from its default."""
    g = []
    everything = list(range(2, MAXPOSE + 1))
    for stereo in (True, False):
        for ts in (True, False):
            sfx = ("stereo" if stereo else "mono") + ("-ts" if ts else "-nots")
            kinds = ["none"] * len(everything) + ["outlier", "flip", "garbage"]
            g.append(_group(f"trail20-{sfx}", 11 + 2 * stereo + ts, stereo=stereo, time_shift=ts, nposes=everything + [6, 7, 8],
                            kinds=kinds, depths=(0.5, 1.0, 3.0, 8.0)))
    g.append(_group("trail4-stereo-ts", 21, trail=4, nposes=(2, 3, 4, 5), depths=(0.6, 2.0)))
    g.append(_group("trail8-mono-ts", 22, trail=8, stereo=False, nposes=(2, 5, 9, 9), kinds=["none", "none", "none", "flip"]))
    g.append(_group("trail30-stereo-ts", 23, trail=30, nposes=(3, 12, 21)))
    g.append(_group("trail20-map8-stereo-ts", 24, map_size=8, nposes=(2, 11, 21)))
    g.append(_group("static-stereo-ts", 25, stereo=True, nposes=(3, 6), static=True))
    g.append(_group("static-mono-nots", 26, stereo=False, time_shift=False, nposes=(4, 8), static=True))
    for it in (1, 2, 3, 25):
        g.append(_group(f"gn{it}", 30 + it, params=dict(gauss_newton_iterations=it), nposes=(3, 8, 17), kinds=["none", "none", "garbage"]))
    for thr in (1e-1, 1e-4):
        g.append(_group(f"conv{thr:g}", 60 + int(thr < 1e-2), params=dict(convergence_threshold=thr), nposes=(3, 8, 17)))
    g.append(_group("convR1", 62, params=dict(convergence_r=1.0), nposes=(3, 8, 17)))
    g.append(_group("convR11-mono", 63, stereo=False, params=dict(convergence_r=11.0), nposes=(5, 12)))
    for i, thr in enumerate((1e-8, 1e-4, 1e-2)):
        g.append(_group(f"rcond{thr:g}", 70 + i, params=dict(rcond_threshold=thr), nposes=(3, 8, 17), depths=(0.5, 3.0, 8.0)))
    g.append(_group("dist-bracket", 80, params=dict(min_dist=3.0, max_dist=20.0), nposes=(3, 6, 9, 12, 5, 4),
                    kinds=["none"] * 5 + ["flip"], depths=(0.3, 1.0, 2.0, 6.0)))
    return g
