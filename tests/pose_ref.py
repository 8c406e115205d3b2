"""Extended-precision reference for cv::recoverPose (tests/test_pose_ref.py): mpmath at 50 digits, sharing no code or order of operations
with the oracle (oracle/hv_oracle_pose.c) or the kernel.

- decomposeEssentialMat: mp.svd_r of E, U and V^T negated where their determinant is negative; R1 = U W V^T, R2 = U W^T V^T, t = U[:, 2].
- Per candidate and point, the DLT null vector is the last right singular vector of mp.svd_r of the 4 x 4 system.
- The componentwise condition number of R and t with respect to E, kappa = max over entries of sum_ab |dX/dE_ab| |E_ab|, from forward
  differences at 50 digits (each perturbed decomposition's candidates matched to the unperturbed ones, so that SVD sign conventions
  cannot swap them). For t it is of the order of |E| / (sigma2 - sigma3).
- A decision is determined at double precision when its value lies further from the threshold (0 or dist) than a first-order bound
  on the error of a double computation: the null vector's angle error
      theta = 64 u (sigma1(A) + |dA|) / (sigma3(A) - sigma4(A)),  |dA| = 2 e_P (|x2| + |y2| + 1),  e_P = 64 u max(kappa_R, kappa_t, 1),
  carried to Z = Q2 / Q3 as theta (1 + |Z|) / |Q3| and to the second camera's depth through its row of P. A point is determined
  when, under every candidate, either some decision is determined false or all four are determined true.
"""
import mpmath as mp
import numpy as np

DPS = 50
U64 = 2.0 ** -52
W = [[0, 1, 0], [-1, 0, 0], [0, 0, 1]]


def _mat(a):
    return mp.matrix([[mp.mpf(float(x)) for x in row] for row in np.asarray(a, np.float64)])


def _candidates(Em):
    """the four candidates [(R, t)] of an mp 3 x 3 E, and its singular values"""
    U, S, Vt = mp.svd_r(Em)
    if mp.det(U) < 0:
        U = -U
    if mp.det(Vt) < 0:
        Vt = -Vt
    Wm = mp.matrix(W)
    R1, R2 = U * Wm * Vt, U * Wm.T * Vt
    t = U[:, 2]
    return [(R1, t), (R2, t), (R1, -t), (R2, -t)], S


def _flat(R, t):
    return [R[i, j] for i in range(3) for j in range(3)] + [t[i] for i in range(3)]


def decompose(E):
    """(candidates as lists of 12 mpf (R row-major, t), condition numbers kappa (4,) as floats: max over R and t entries, singular
    values (3,) as floats) of a float64 E (3, 3) row-major"""
    with mp.workdps(DPS):
        Em = _mat(E)
        cands, S = _candidates(Em)
        base = [_flat(R, t) for R, t in cands]
        kap = [[mp.mpf(0)] * 12 for _ in range(4)]
        for a in range(3):
            for b in range(3):
                if Em[a, b] == 0:
                    continue
                h = abs(Em[a, b]) * mp.mpf(10) ** -25
                Ep = Em.copy()
                Ep[a, b] += h
                pc, _ = _candidates(Ep)
                pf = [_flat(R, t) for R, t in pc]
                for k in range(4):
                    # the perturbed candidate nearest to candidate k
                    j = min(range(4), key=lambda j: max(abs(x - y) for x, y in zip(pf[j], base[k])))
                    for e in range(12):
                        kap[k][e] += abs(pf[j][e] - base[k][e]) / h * abs(Em[a, b])
        kappa = np.array([float(max(k)) for k in kap])
        return base, kappa, np.array([float(s) for s in S])


def point_values(P, q, eP):
    """(Z, z, dZ, dz) of one normalised correspondence q (x1, y1, x2, y2) under one candidate P (12 mpf: R row-major, t): the depths in
    the first and second camera and the bounds on their double-precision error; None where the null vector's last entry is 0"""
    x1, y1, x2, y2 = (mp.mpf(float(v)) for v in q)
    Pm = [[P[0], P[1], P[2], P[9]], [P[3], P[4], P[5], P[10]], [P[6], P[7], P[8], P[11]]]
    A = mp.matrix([[-1, 0, x1, 0], [0, -1, y1, 0], [x2 * Pm[2][k] - Pm[0][k] for k in range(4)], [y2 * Pm[2][k] - Pm[1][k] for k in range(4)]])
    _, S, Vt = mp.svd_r(A)
    Q = [Vt[3, k] for k in range(4)]
    if Q[3] == 0:
        return None
    X, Y, Z = Q[0] / Q[3], Q[1] / Q[3], Q[2] / Q[3]
    z = Pm[2][0] * X + Pm[2][1] * Y + Pm[2][2] * Z + Pm[2][3]
    dA = 2 * eP * (abs(x2) + abs(y2) + 1)
    gap = S[2] - S[3]
    theta = mp.inf if gap == 0 else 64 * U64 * (S[0] + dA) / gap
    dX, dY, dZ = (theta * (1 + abs(v)) / abs(Q[3]) for v in (X, Y, Z))
    dz = 2 * (abs(Pm[2][0]) * dX + abs(Pm[2][1]) * dY + abs(Pm[2][2]) * dZ + eP * (abs(X) + abs(Y) + abs(Z) + 1))
    return Z, z, dZ, dz


def decide(v, dist):
    """(good, determined) from point_values: Z > 0, Z < dist, z > 0, z < dist"""
    if v is None:
        return False, False
    if np.isnan(dist) or dist == -np.inf:
        return False, True
    Z, z, dZ, dz = v
    tests = [(Z > 0, abs(Z) > dZ), (z > 0, abs(z) > dz)]
    if np.isfinite(dist):
        tests += [(Z < dist, abs(Z - dist) > dZ), (z < dist, abs(z - dist) > dz)]
    good = all(g for g, _ in tests)
    return good, any(d and not g for g, d in tests) or all(d for _, d in tests)


def recover_pose(E, q, dists):
    """The reference call on a float64 E (3, 3) and normalised points q (n, 4) at each distance threshold: ({dist: (flags (n, 4) bool,
    determined (n,) bool)}, candidates, kappa (4,), singular values of E)"""
    with mp.workdps(DPS):
        cands, kappa, S = decompose(E)
        n = len(q)
        vals = [[point_values(cands[k], q[i], mp.mpf(64 * U64 * max(kappa[k], 1.0))) for k in range(4)] for i in range(n)]
        out = {}
        for dist in dists:
            flags = np.zeros((n, 4), bool)
            det = np.ones(n, bool)
            for i in range(n):
                for k in range(4):
                    flags[i, k], d = decide(vals[i][k], dist)
                    det[i] &= d
            out[dist] = (flags, det)
        return out, cands, kappa, S


def winner(flags, use):
    """OpenCV's choice from the per-candidate flags and the used points: (index, counts, tied candidates)"""
    cnt = (flags & use[:, None]).sum(0)
    for k in range(4):
        if all(cnt[k] >= cnt[j] for j in range(4)):
            return k, cnt, [j for j in range(4) if cnt[j] == cnt[k]]
    raise AssertionError("unreachable")
