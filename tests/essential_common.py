"""Seeded two-view scenes for the essential-matrix RANSAC tests (oracle, emulator-free CPU checks and GPU)."""
import numpy as np

# EuRoC cam0's pinhole intrinsics: a realistic K with fx != fy
FX, FY, CX, CY = 458.654, 457.296, 367.215, 248.375
K = np.array([[FX, 0.0, CX], [0.0, FY, CY], [0.0, 0.0, 1.0]])
W, H = 752, 480

M_VALUES = (6, 8, 20, 150, 300, 600, 2000)
OUTLIERS = (0.0, 0.1, 0.3, 0.5, 0.7)
NOISE = (0.0, 0.3, 1.0)
THRESHOLDS = (0.5, 1.0, 2.0)
PROBS = (0.99, 0.999)
MAX_ITERS = (1, 3, 1000)


def _rodrigues(w):
    th = float(np.linalg.norm(w))
    if th == 0.0:
        return np.eye(3)
    k = w / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def scene(rng, m, outliers=0.0, noise=0.0, motion="side", rot=0.05):
    """m correspondences (p1, p2) float32 of a random point cloud seen from two poses; `outliers` of them (at random positions in the
    list) replaced by uniform points in the second image; `noise` pixels of Gaussian noise on both. motion: "side" (mostly x),
    "forward" (mostly z), "rotation" (no translation), "static" (identity pose), "plane" (every point on z = 5)."""
    X = np.c_[rng.uniform(-3, 3, m), rng.uniform(-2, 2, m), rng.uniform(3, 8, m)]
    if motion == "plane":
        X[:, 2] = 5.0
    R = _rodrigues(rng.normal(0, rot, 3)) if motion not in ("static",) else np.eye(3)
    t = {"side": np.array([0.3, 0.02, 0.05]), "forward": np.array([0.02, 0.03, 0.5]), "rotation": np.zeros(3), "static": np.zeros(3),
         "plane": np.array([0.3, 0.02, 0.05])}[motion]
    p1 = (K @ X.T).T
    p1 = p1[:, :2] / p1[:, 2:]
    X2 = (R @ X.T).T + t
    p2 = (K @ X2.T).T
    p2 = p2[:, :2] / p2[:, 2:]
    p1 = p1 + rng.normal(0, noise, p1.shape)
    p2 = p2 + rng.normal(0, noise, p2.shape)
    k = int(round(m * outliers))
    if k:
        sel = rng.choice(m, k, replace=False)
        p2[sel] = np.c_[rng.uniform(0, W, k), rng.uniform(0, H, k)]
    return p1.astype(np.float32), p2.astype(np.float32)


def cases():
    """The parameter grid of the whole-call checks: every m x outlier ratio x motion, with noise, threshold, prob and max_iters
    cycling so that every value of each meets every m. Yields (name, seed, m, outliers, noise, motion, prob, threshold, max_iters)."""
    i = 0
    for m in M_VALUES:
        for outl in OUTLIERS:
            for motion in ("side", "forward"):
                for mi in MAX_ITERS:
                    noise = NOISE[i % len(NOISE)]
                    thr = THRESHOLDS[(i // 3) % len(THRESHOLDS)]
                    prob = PROBS[(i // 2) % len(PROBS)]
                    yield (f"m{m}-o{outl}-{motion}-it{mi}-n{noise}-t{thr}-p{prob}", 1000 + i, m, outl, noise, motion, prob, thr, mi)
                    i += 1


def case_points(case):
    _, seed, m, outl, noise, motion, _, _, _ = case
    return scene(np.random.default_rng(seed), m, outl, noise, motion)


def degenerate_scenes():
    """(name, p1, p2) of the degenerate configurations whose result is recorded, not gated."""
    out = []
    for k, motion in enumerate(("static", "rotation", "plane")):
        for noise in (0.0, 0.5):
            p1, p2 = scene(np.random.default_rng(50 + 2 * k + int(noise > 0)), 150, 0.2, noise, motion)
            out.append((f"{motion}-n{noise}", p1, p2))
    p1, p2 = scene(np.random.default_rng(60), 40, 0.0, 0.3)
    out.append(("repeated", np.repeat(p1, 4, axis=0), np.repeat(p2, 4, axis=0)))
    return out
