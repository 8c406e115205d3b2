"""Seeded two-view scenes for the cv::triangulatePoints tests (oracle, reference, emulator and GPU).

A scene is (name, family, P1, P2, xy1, xy2): P1, P2 row-major (3, 4) float64, xy1, xy2 (n, 2) float32. family "general" holds the
scenes a running tracker produces (rectified stereo with pixel noise, a general relative pose); "degenerate" the near-degenerate ones
(zero and negative disparity, a 1e-6 baseline, points on the epipoles, P1 == P2, a zero row or column in P, pixel coordinates of 1e5)."""
import numpy as np

F, CX, CY, B = 450.0, 370.0, 240.0, 0.11          # a rectified stereo rig: focal length, principal point, baseline (m)
K = np.array([[F, 0.0, CX], [0.0, F, CY], [0.0, 0.0, 1.0]])
NONE = np.float32(-1.0e6)                           # HV_CORNER_NONE


def rodrigues(r):
    th = float(np.linalg.norm(r))
    if th == 0.0:
        return np.eye(3)
    k = np.asarray(r, np.float64) / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def projection(R=np.eye(3), t=np.zeros(3), k=K):
    return k @ np.c_[R, np.asarray(t, np.float64).reshape(3, 1)]


def stereo_pair(baseline=B, k=K):
    """P1 = K [I | 0] (left), P2 = K [I | (-baseline, 0, 0)] (the right camera at +baseline: a point at depth Z moves f B / Z to the
    left)"""
    return projection(k=k), projection(t=(-baseline, 0.0, 0.0), k=k)


def project(P, X, rng=None, noise=0.0):
    x = (P @ np.c_[X, np.ones(len(X))].T).T
    x = x[:, :2] / x[:, 2:]
    if noise:
        x = x + rng.normal(0, noise, x.shape)
    return x.astype(np.float32)


def cloud(rng, n, zlo=0.5, zhi=30.0):
    Z = rng.uniform(zlo, zhi, n)
    u, v = rng.uniform(0, 2 * CX, n), rng.uniform(0, 2 * CY, n)
    return np.c_[(u - CX) / F * Z, (v - CY) / F * Z, Z]


def rectified(seed, n=250, noise=0.5):
    rng = np.random.default_rng(seed)
    P1, P2 = stereo_pair()
    X = cloud(rng, n)
    return P1, P2, project(P1, X, rng, noise), project(P2, X, rng, noise)


def general(seed, n=250, noise=0.5):
    """Both cameras posed in a world frame away from them (random R, t of a few metres), as when a map's frame is the world's"""
    rng = np.random.default_rng(seed)
    R1, t1 = rodrigues(rng.normal(0, 0.3, 3)), rng.normal(0, 3.0, 3)
    R = rodrigues(rng.normal(0, 0.3, 3))
    t = rng.normal(0, 1.0, 3)
    P1, P2 = projection(R1, t1), projection(R @ R1, R @ t1 + t)
    X = (R1.T @ (cloud(rng, n, 1.0, 20.0) - t1).T).T
    return P1, P2, project(P1, X, rng, noise), project(P2, X, rng, noise)


def degenerate(seed, n=60):
    """(name, P1, P2, xy1, xy2) of every near-degenerate family"""
    rng = np.random.default_rng(seed)
    P1, P2 = stereo_pair()
    out = []
    X = cloud(rng, n)
    x1 = project(P1, X, rng, 0.3)
    out.append(("zero disparity", P1, P2, x1, x1.copy()))                                   # w ~ 0: at infinity
    d = rng.uniform(0.5, 20.0, (n, 1)) * np.array([[1.0, 0.0]])
    out.append(("negative disparity", P1, P2, x1, (x1 + d).astype(np.float32)))              # behind the cameras
    Q1, Q2 = stereo_pair(1e-6)
    out.append(("baseline 1e-6", Q1, Q2, project(Q1, X, rng, 0.0), project(Q2, X, rng, 0.0)))
    R, t = rodrigues(rng.normal(0, 0.2, 3)), np.array([0.3, -0.1, 1.0])
    G1, G2 = projection(), projection(R, t)
    C2 = -R.T @ t                                                                            # camera 2's centre in camera 1
    e1 = G1 @ np.r_[C2, 1.0]
    e2 = G2 @ np.array([0.0, 0.0, 0.0, 1.0])
    e1, e2 = e1[:2] / e1[2], e2[:2] / e2[2]
    jit = rng.normal(0, 1e-3, (n, 2))
    out.append(("on the epipoles", G1, G2, (e1 + jit).astype(np.float32), (e2 - jit).astype(np.float32)))
    out.append(("P1 == P2", P1, P1.copy(), x1, x1.copy()))                                  # rank deficient
    out.append(("P1 == P2, other points", P1, P1.copy(), x1, project(P2, X, rng, 0.3)))
    Z2 = P2.copy()
    Z2[1] = 0.0
    out.append(("zero row in P2", P1, Z2, x1, project(P2, X, rng, 0.3)))
    Z1 = P1.copy()
    Z1[2] = 0.0
    out.append(("zero last row in P1", Z1, P2, x1, project(P2, X, rng, 0.3)))
    C1, C2 = P1.copy(), P2.copy()
    C1[:, 0] = 0.0
    C2[:, 0] = 0.0
    out.append(("zero first column in P1 and P2", C1, C2, x1, project(P2, X, rng, 0.3)))   # null vector e1 at row 0 before the sort
    big = rng.uniform(-1e5, 1e5, (n, 2)).astype(np.float32)
    out.append(("pixels of 1e5", P1, P2, big, (big + rng.normal(0, 5.0, (n, 2))).astype(np.float32)))
    return out


def scenes():
    """Every scene: (name, family, P1, P2, xy1, xy2)"""
    out = []
    for s in range(4):
        out.append((f"rectified stereo {s}", "general") + rectified(100 + s))
    for s in range(4):
        out.append((f"general two-view {s}", "general") + general(200 + s))
    for name, P1, P2, a, b in degenerate(300):
        out.append((name, "degenerate", P1, P2, a, b))
    return out


def padded(xy, cap):
    """xy (n, 2) in a (cap, 2) buffer filled with HV_CORNER_NONE behind the n points"""
    out = np.full((cap, 2), NONE, np.float32)
    out[:len(xy)] = xy
    return out
