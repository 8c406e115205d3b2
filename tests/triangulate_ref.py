"""TEST INFRASTRUCTURE: a 50-digit mpmath reference for cv::triangulatePoints. It shares no code with the oracle: the DLT matrix A of a
correspondence is formed exactly (mp) from the float32 points and the fp64 projection matrices, and its null vector is the eigenvector
of AᵀA for the smallest eigenvalue (mp.eigsy), its singular values the square roots of the eigenvalues."""
import mpmath as mp

DPS = 50


def dlt(P1, P2, x1, x2):
    """The 4 x 4 DLT matrix in mp: rows x P[2,:] - P[0,:], y P[2,:] - P[1,:] of both views"""
    rows = []
    for P, (x, y) in ((P1, x1), (P2, x2)):
        for r, c in ((0, x), (1, y)):
            rows.append([mp.mpf(float(c)) * mp.mpf(float(P[2][k])) - mp.mpf(float(P[r][k])) for k in range(4)])
    return mp.matrix(rows)


def null_vector(P1, P2, x1, x2):
    """(the unit null vector (4 mpf), singular values descending (4 mpf))"""
    with mp.workdps(DPS):
        A = dlt(P1, P2, x1, x2)
        E, Q = mp.eigsy(A.T * A)
        order = sorted(range(4), key=lambda i: E[i])
        sig = [mp.sqrt(max(E[i], mp.mpf(0))) for i in reversed(order)]
        v = [Q[k, order[0]] for k in range(4)]
        nv = mp.sqrt(mp.fsum(c * c for c in v))
        return [c / nv for c in v], sig


def sin_angle(q, v):
    """sin of the angle between the line of q (4 floats, not all zero) and the unit vector v, in mp"""
    with mp.workdps(DPS):
        qm = [mp.mpf(float(c)) for c in q]
        nq = mp.sqrt(mp.fsum(c * c for c in qm))
        qm = [c / nq for c in qm]
        d = mp.fsum(a * b for a, b in zip(qm, v))
        return mp.sqrt(mp.fsum((a - d * b) ** 2 for a, b in zip(qm, v)))
