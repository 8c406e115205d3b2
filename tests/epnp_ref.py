"""Extended-precision reference for the EPnP pose that solvePnPRansac returns (tests/test_epnp_ref.py, tests/test_gpu_epnp_ref.py):
OpenCV's epnp::compute_pose restated in mpmath at 60 digits, sharing no code or linear algebra with the solver (oracle/hv_oracle_pnp.c,
csrc/pnp.cu), which uses fixed-sweep Jacobi SVDs, OpenCV's QR and sums in the CTA's order.

- Control points: the centroid c0 and c0 + sqrt(lambda_i / n) e_i along the covariance's eigenvectors (mp.eigsy), largest first. The sign
  of each e_i is a convention of OpenCV's Jacobi SVD that no formulation derives, and on noisy points it moves the pose by about 1e-3,
  so it is the one thing taken from the solver: each e_i is turned to agree with the solver's axis (`axes`).
- Barycentric coordinates: exact, through the inverse of [c1 - c0, c2 - c0, c3 - c0] = [e_i sqrt(lambda_i / n)]. An axis whose
  length is at or below 2 DBL_EPSILON times their sum (OpenCV's cvInvert(CV_SVD) cut-off) is dropped, as the pseudo-inverse drops it;
  at 60 digits that happens only where the covariance is exactly singular (points on a plane of constant coordinate).
- M^T M summed in mp from the two rows per point; its four eigenvectors of smallest eigenvalue (v0 the smallest). Columns of M that are
  exactly zero (a dropped control point) are exact null vectors e_k; they come first, the highest index first, as OpenCV's SVD leaves
  them.
- L (6 x 10) and rho; the three beta approximations as exact least squares (mp.svd_r, OpenCV's cut-off), with OpenCV's sign branches;
  5 Gauss-Newton steps, each an exact least-squares step (or, where the Jacobian has an exactly zero column, OpenCV's qr_solve's
  early return: the previous step again).
- For each approximation: the control points in the camera, their sign chosen so that the first point is in front, and Procrustes
  from mp.svd_r with OpenCV's last-row flip when det R < 0. Where sigma3 <= 1e-8 sigma1 (points on a plane) u3 is not determined by the
  data and is taken as det(V) (u1 x u2), so that R is the nearest rotation.
- The approximation of least mean reprojection error, the first on a tie.

fp64-determined: the reference is run 8 more times, with the inputs perturbed by up to 4 ulp and the covariance, M^T M, L and rho by
up to u relative to each one's norm. Entries that are exactly zero stay zero: they are exact in double as well (the differences from
the centroid along a plane's constant coordinate), and a coordinate shared exactly by all points stays shared, for the same reason.
A scene is fp64-determined when every discrete decision (the dropped axes and least-squares cut-offs, the beta sign branches, the
first point's sign, the sigma3 branch, the det < 0 flip and the chosen approximation) is the same in all runs. Its tolerance on each
entry x of R, t and rvec is 16 spread + 64 u max(|x|, 1), spread the largest departure of a perturbed run; rvec's adds the
conditioning of Rodrigues on the tolerance of R (see reference)."""
import mpmath as mp
import numpy as np

mp.mp.dps = 60
U = mp.mpf(2) ** -53
EPS2 = 2 * mp.mpf(2) ** -52             # OpenCV's SVD cut-off, relative to the sum of the singular values


def _dot(a, b):
    return mp.fdot(a, b)


def _perturb_rows(P, rng, ulps=4):
    """each entry times (1 + ulps u r), r in [-1, 1]; a column whose entries are all equal keeps them equal"""
    shared = [all(r[k] == P[0][k] for r in P) for k in range(len(P[0]))]
    f = [1 + ulps * U * rng.uniform(-1, 1) for _ in P[0]]
    return [[x * (f[k] if shared[k] else 1 + ulps * U * rng.uniform(-1, 1)) for k, x in enumerate(r)] for r in P]


def _perturb(A, rng, sym=False):
    """A (mp.matrix) plus up to u times its Frobenius norm on each non-zero entry (symmetrically if sym)"""
    nrm = mp.mnorm(A, "f")
    B = A.copy()
    for i in range(A.rows):
        for j in range(i if sym else 0, A.cols):
            if A[i, j] != 0:
                B[i, j] = A[i, j] + U * nrm * rng.uniform(-1, 1)
                if sym:
                    B[j, i] = B[i, j]
    return B


def _lsq(A, b, dec):
    """min-norm least squares through the SVD, singular values at or below EPS2 times their sum dropped (recorded in dec)"""
    Us, S, Vt = mp.svd_r(A)
    thr = EPS2 * sum(S)
    x = [mp.mpf(0)] * A.cols
    for j in range(len(S)):
        keep = S[j] > thr
        dec.append(("cut", keep))
        if not keep:
            continue
        f = mp.fsum(Us[r, j] * b[r] for r in range(A.rows)) / S[j]
        x = [x[i] + Vt[j, i] * f for i in range(A.cols)]
    return x


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _det3(M):
    return mp.det(mp.matrix(M))


def axis_angle(R):
    """the rotation vector of the rotation R (3 x 3 mp.matrix) and sin(theta): theta = atan2(s, c), the axis from the skew part, or
    near theta = pi from the symmetric part (R + R^T) / 2 - c I = (1 - c) n n^T with the skew part's sign"""
    sk = [R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]]
    s = mp.sqrt(_dot(sk, sk)) / 2
    c = (R[0, 0] + R[1, 1] + R[2, 2] - 1) / 2
    th = mp.atan2(s, c)
    if s == 0 and c > 0:
        return [mp.mpf(0)] * 3, s
    if c > 0:
        return [x * th / (2 * s) for x in sk], s
    B = [[(R[i, j] + R[j, i]) / 2 - (c if i == j else 0) for j in range(3)] for i in range(3)]
    k = max(range(3), key=lambda i: B[i][i])
    col = [B[i][k] for i in range(3)]
    nrm = mp.sqrt(_dot(col, col))
    n = [x / nrm for x in col]
    if _dot(n, sk) < 0:
        n = [-x for x in n]
    return [x * th for x in n], s


def _betas(L, rho, dec):
    """the three approximations of epnp::find_betas_approx_1/2/3"""
    def cols(idx):
        return mp.matrix([[L[i, k] for k in idx] for i in range(6)])
    out = []
    b = _lsq(cols((0, 1, 3, 6)), rho, dec)
    dec.append(("b0<0", b[0] < 0))
    if b[0] < 0:
        b0 = mp.sqrt(-b[0])
        out.append([b0, -b[1] / b0, -b[2] / b0, -b[3] / b0])
    else:
        b0 = mp.sqrt(b[0])
        out.append([b0, b[1] / b0, b[2] / b0, b[3] / b0])
    for idx in ((0, 1, 2), (0, 1, 2, 3, 4)):
        b = _lsq(cols(idx), rho, dec)
        dec.append(("b02", b[0] < 0, b[2] < 0, b[2] > 0, b[1] < 0))
        if b[0] < 0:
            be = [mp.sqrt(-b[0]), mp.sqrt(-b[2]) if b[2] < 0 else mp.mpf(0)]
        else:
            be = [mp.sqrt(b[0]), mp.sqrt(b[2]) if b[2] > 0 else mp.mpf(0)]
        if b[1] < 0:
            be[0] = -be[0]
        be += [b[3] / be[0] if len(idx) == 5 else mp.mpf(0), mp.mpf(0)]
        out.append(be)
    return out


def _gauss_newton(L, rho, be, dec):
    """5 steps, each the exact least-squares step. Where the Jacobian has an exactly zero column (a beta that points on a plane
    leave free), OpenCV's qr_solve returns without writing the step, and the previous step (none on the first) is applied again."""
    be = list(be)
    dx = [mp.mpf(0)] * 4
    for _ in range(5):
        A = mp.matrix(6, 4)
        r = []
        for i in range(6):
            l = [L[i, k] for k in range(10)]
            A[i, 0] = 2 * l[0] * be[0] + l[1] * be[1] + l[3] * be[2] + l[6] * be[3]
            A[i, 1] = l[1] * be[0] + 2 * l[2] * be[1] + l[4] * be[2] + l[7] * be[3]
            A[i, 2] = l[3] * be[0] + l[4] * be[1] + 2 * l[5] * be[2] + l[8] * be[3]
            A[i, 3] = l[6] * be[0] + l[7] * be[1] + l[8] * be[2] + 2 * l[9] * be[3]
            q = [be[0] * be[0], be[0] * be[1], be[1] * be[1], be[0] * be[2], be[1] * be[2], be[2] * be[2], be[0] * be[3], be[1] * be[3],
                 be[2] * be[3], be[3] * be[3]]
            r.append(rho[i] - _dot(l, q))
        zero_col = any(all(A[i, k] == 0 for i in range(6)) for k in range(4))
        dec.append(("qr", zero_col))
        if not zero_col:
            dx = _lsq(A, r, dec)
        be = [be[k] + dx[k] for k in range(4)]
    return be


def _pose(be, v, al, pw, c0, us, fu, fv, uc, vc, dec):
    """compute_R_and_t of one beta vector: (R, t, mean reprojection error)"""
    ccs = [[_dot(be, [v[i][3 * j + k] for i in range(4)]) for k in range(3)] for j in range(4)]
    pcs = [[_dot(a, [ccs[j][k] for j in range(4)]) for k in range(3)] for a in al]
    flip = pcs[0][2] < 0
    dec.append(("z0<0", flip))
    if flip:
        pcs = [[-x for x in p] for p in pcs]
    n = len(pw)
    pc0 = [mp.fsum(p[k] for p in pcs) / n for k in range(3)]
    dc = [[p[k] - pc0[k] for p in pcs] for k in range(3)]
    dw = [[p[k] - c0[k] for p in pw] for k in range(3)]
    abt = mp.matrix([[_dot(dc[a], dw[b]) for b in range(3)] for a in range(3)])
    Us, S, Vt = mp.svd_r(abt)
    branch = not (S[2] > mp.mpf("1e-8") * S[0])
    dec.append(("sigma3", branch))
    if branch:
        u3 = _cross([Us[i, 0] for i in range(3)], [Us[i, 1] for i in range(3)])
        sg = 1 if _det3(Vt) > 0 else -1
        for i in range(3):
            Us[i, 2] = sg * u3[i]
    R = Us * Vt
    neg = _det3(R) < 0
    dec.append(("det<0", neg))
    if neg:
        for j in range(3):
            R[2, j] = -R[2, j]
    t = [pc0[i] - _dot([R[i, j] for j in range(3)], c0) for i in range(3)]
    err = []
    for p, u in zip(pw, us):
        Xc = [_dot([R[i, j] for j in range(3)], p) + t[i] for i in range(3)]
        if Xc[2] == 0:                  # a degenerate approximation (all points at the camera centre): never chosen
            return R, t, mp.nan
        ue, ve = uc + fu * Xc[0] / Xc[2], vc + fv * Xc[1] / Xc[2]
        err.append(mp.sqrt((u[0] - ue) ** 2 + (u[1] - ve) ** 2))
    return R, t, mp.fsum(err) / n


def compute_pose(pw, us, fu, fv, uc, vc, axes, rng=None):
    """one run of epnp::compute_pose on pw (n lists of 3 mpf) and us (n lists of 2 mpf); axes (3 x 3) the directions the principal
    axes are turned to agree with; rng perturbs as the module docstring says. Returns (R, t, rvec, sin theta, decisions, signed axes,
    eigenvalues descending)."""
    dec = []
    if rng is not None:
        pw, us = _perturb_rows(pw, rng), _perturb_rows(us, rng)
    n = len(pw)
    c0 = [mp.fsum(p[k] for p in pw) / n for k in range(3)]
    d = [[p[k] - c0[k] for p in pw] for k in range(3)]
    cov = mp.matrix([[_dot(d[i], d[j]) for j in range(3)] for i in range(3)])
    if rng is not None:
        cov = _perturb(cov, rng, sym=True)
    E, Q = mp.eigsy(cov)
    lam, ax = [], []
    for k in (2, 1, 0):
        e = [Q[i, k] for i in range(3)]
        if _dot(e, axes[len(ax)]) < 0:
            e = [-x for x in e]
        lam.append(E[k])
        ax.append(e)
    kk = [mp.sqrt(max(x, 0) / n) for x in lam]
    cws = [c0] + [[c0[j] + kk[i] * ax[i][j] for j in range(3)] for i in range(3)]
    keep = [k > EPS2 * sum(kk) for k in kk]
    dec.append(("axes", tuple(keep)))
    al = []
    for j in range(n):
        a = [_dot([d[k][j] for k in range(3)], ax[i]) / kk[i] if keep[i] else mp.mpf(0) for i in range(3)]
        al.append([1 - a[0] - a[1] - a[2]] + a)
    # M^T M from the point's two rows [a_k fu, 0, a_k (uc - u)] and [0, a_k fv, a_k (vc - v)], k the control point
    g = [uc - u[0] for u in us]
    h = [vc - u[1] for u in us]
    gh = [x * x + y * y for x, y in zip(g, h)]
    MtM = mp.matrix(12, 12)
    for k in range(4):
        for l in range(k, 4):
            aa = [a[k] * a[l] for a in al]
            s0, sg, sh, sgh = mp.fsum(aa), _dot(aa, g), _dot(aa, h), _dot(aa, gh)
            blk = [[fu * fu * s0, 0, fu * sg], [0, fv * fv * s0, fv * sh], [fu * sg, fv * sh, sgh]]
            for p in range(3):
                for q in range(3):
                    MtM[3 * k + p, 3 * l + q] = blk[p][q]
                    MtM[3 * l + q, 3 * k + p] = blk[p][q]
    if rng is not None:
        MtM = _perturb(MtM, rng, sym=True)
    zero = [k for k in range(12) if all(MtM[k, j] == 0 for j in range(12))]
    act = [k for k in range(12) if k not in zero]
    v = []
    for k in reversed(zero):
        v.append([mp.mpf(1) if j == k else mp.mpf(0) for j in range(12)])
    Ea, Qa = mp.eigsy(mp.matrix([[MtM[i, j] for j in act] for i in act]))
    for c in range(4 - len(v)):
        e = [mp.mpf(0)] * 12
        for i, k in enumerate(act):
            e[k] = Qa[i, c]
        v.append(e)
    v = v[:4]
    pairs = ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3))
    L = mp.matrix(6, 10)
    rho = mp.matrix(6, 1)
    for r, (a, b) in enumerate(pairs):
        dv = [[v[i][3 * a + k] - v[i][3 * b + k] for k in range(3)] for i in range(4)]
        row = [_dot(dv[0], dv[0]), 2 * _dot(dv[0], dv[1]), _dot(dv[1], dv[1]), 2 * _dot(dv[0], dv[2]), 2 * _dot(dv[1], dv[2]),
               _dot(dv[2], dv[2]), 2 * _dot(dv[0], dv[3]), 2 * _dot(dv[1], dv[3]), 2 * _dot(dv[2], dv[3]), _dot(dv[3], dv[3])]
        for k in range(10):
            L[r, k] = row[k]
        dw = [cws[a][k] - cws[b][k] for k in range(3)]
        rho[r] = _dot(dw, dw)
    if rng is not None:
        L, rho = _perturb(L, rng), _perturb(rho, rng)
    rho = [rho[i] for i in range(6)]
    poses = [_pose(_gauss_newton(L, rho, be, dec), v, al, pw, c0, us, fu, fv, uc, vc, dec) for be in _betas(L, rho, dec)]
    N = 0                               # OpenCV's order of comparison, so a NaN error is never chosen after the first
    if poses[1][2] < poses[0][2]:
        N = 1
    if poses[2][2] < poses[N][2]:
        N = 2
    R, t, _ = poses[N]
    dec.append(("N", N))
    r, s = axis_angle(R)
    return R, t, r, s, dec, ax, lam


def undistort_round_trip(x, fx, fy, cx, cy):
    """the double image points OpenCV's undistortPoints round trip gives for float32 pixels (n, 2), as the solver forms them"""
    x = np.asarray(x, np.float64).reshape(-1, 2)
    return np.c_[((x[:, 0] - cx) * (1.0 / fx)) * fx + cx, ((x[:, 1] - cy) * (1.0 / fy)) * fy + cy]


def reference(X, x, fx, fy, cx, cy, axes, runs=8, seed=0):
    """EPnP of the world points X (n, 3) at the float32 pixels x (n, 2), the principal axes turned to agree with `axes` (3, 3).
    Returns a dict: R (3, 3), t, rvec, sin_theta (floats); tol_R, tol_t, tol_rvec (per entry); determined; undetermined_by (the first
    decision that differed); axes (3, 3) and eigenvalues (3,) of the covariance, largest first."""
    pw = [[mp.mpf(float(c)) for c in p] for p in np.asarray(X, np.float64).reshape(-1, 3)]
    us = [[mp.mpf(float(c)) for c in p] for p in undistort_round_trip(x, fx, fy, cx, cy)]
    k = [mp.mpf(float(v)) for v in (fx, fy, cx, cy)]
    R, t, r, s, dec, ax, lam = compute_pose(pw, us, *k, np.asarray(axes, np.float64).tolist())
    flat = lambda R_, t_, r_: np.array([float(R_[i, j]) for i in range(3) for j in range(3)] + [float(c) for c in t_] + [float(c) for c in r_])
    base = [R[i, j] for i in range(3) for j in range(3)] + list(t) + list(r)
    rng = np.random.default_rng(seed)
    spread = np.zeros(15)
    determined, why = True, None
    for _ in range(runs):
        Rp, tp, rp, _, dp, _, _ = compute_pose(pw, us, *k, [[float(c) for c in e] for e in ax], rng)
        if dp != dec:
            determined = False
            why = next((a for a, b in zip(dec, dp) if a != b), "count")
            break
        pert = [Rp[i, j] for i in range(3) for j in range(3)] + list(tp) + list(rp)
        spread = np.maximum(spread, [float(abs(a - b)) for a, b in zip(pert, base)])
    val = flat(R, t, r)
    tol = 16 * spread + 64 * float(U) * np.maximum(np.abs(val), 1.0)
    # rvec is read from the solver's rounded R, which its error in R reaches amplified: by 1 / (2 s) through the skew part, or near
    # theta = pi (s < 1e-5, OpenCV's branch) through the diagonal, whose axis is off by about s^2 / 8 besides
    s, eR, nmin = float(s), tol[:9].max(), max(float(min(abs(c) for c in r)) / max(float(mp.norm(r)), 1e-300), 1e-3)
    tol[12:] += np.pi * eR / (2 * s) if s >= 1e-5 else np.pi * (s * s + 64 * eR) / nmin
    return {"R": val[:9].reshape(3, 3), "t": val[9:12], "rvec": val[12:], "sin_theta": s, "tol_R": tol[:9].reshape(3, 3),
            "tol_t": tol[9:12], "tol_rvec": tol[12:], "determined": determined, "undetermined_by": why,
            "axes": np.array([[float(c) for c in e] for e in ax]), "eigenvalues": np.array([float(x) for x in lam]), "decisions": dec}


def check(ref, R, t, rvec, name):
    """gate a solver's (R, t, rvec) on an fp64-determined reference (R None: t and rvec only); returns the worst error / tolerance. Where sin(theta) < 1e-5,
    OpenCV's Rodrigues takes the axis from the diagonal with its first component non-negative, so rvec is compared up to its sign
    there: at theta = pi - delta the two stand for rotations 2 delta apart, a property of that branch, not of EPnP."""
    worst = 0.0
    got = {"R": np.asarray(R), "t": np.asarray(t), "rvec": np.asarray(rvec)}
    for key in ("R", "t", "rvec") if R is not None else ("t", "rvec"):
        err = np.abs(got[key] - ref[key])
        if key == "rvec" and ref["sin_theta"] < 1e-5:
            err = min(err, np.abs(got[key] + ref[key]), key=lambda e: e.max())
        ratio = (err / ref["tol_" + key]).max()
        worst = max(worst, ratio)
        assert ratio <= 1.0, f"{name}: {key} {got[key].ravel()} against the reference {ref[key].ravel()} (tolerance {ref['tol_' + key].ravel()})"
    return worst
