"""Seeded absolute-pose scenes for the solvePnPRansac tests (oracle, emulator, reference and GPU)."""
import numpy as np

from essential_common import CX, CY, FX, FY, H, W, _rodrigues

K = np.array([[FX, 0.0, CX], [0.0, FY, CY], [0.0, 0.0, 1.0]])

M_VALUES = (4, 5, 6, 8, 20, 150, 300, 600, 4096)
OUTLIERS = (0.0, 0.1, 0.3, 0.5, 0.7)
NOISE = (0.0, 0.5, 1.0)
THRESHOLDS = (1.0, 2.0, 8.0)
MOTIONS = ("side", "forward", "rotation")
DEPTHS = ("near", "far")


def scene(rng, m, outliers=0.0, noise=0.0, motion="side", depth="near"):
    """m world points (float32 (m, 3)) and their pixels (float32 (m, 2)) in a camera at (R, t); `outliers` of them (at random positions)
    replaced by uniform pixels; `noise` pixels of Gaussian noise. motion: the camera's pose relative to the points' frame -- "side"
    (mostly x), "forward" (mostly z), "rotation" (a larger rotation, no translation); depth "near" (2-6 m) or "far" (20-60 m).
    Returns (X, x, R, t)."""
    zlo, zhi = (2.0, 6.0) if depth == "near" else (20.0, 60.0)
    Z = rng.uniform(zlo, zhi, m)
    u = rng.uniform(20, W - 20, m)
    v = rng.uniform(20, H - 20, m)
    Xc = np.c_[(u - CX) / FX * Z, (v - CY) / FY * Z, Z]          # in the camera, visible
    rot = {"side": 0.05, "forward": 0.05, "rotation": 0.4}[motion]
    R = _rodrigues(rng.normal(0, rot, 3))
    t = {"side": np.array([0.5, 0.05, 0.1]), "forward": np.array([0.05, 0.03, 0.8]), "rotation": np.zeros(3)}[motion]
    X = (R.T @ (Xc - t).T).T                                     # world points: Xc = R X + t
    x = np.c_[u, v] + rng.normal(0, noise, (m, 2))
    k = int(round(m * outliers))
    if k:
        sel = rng.choice(m, k, replace=False)
        x[sel] = np.c_[rng.uniform(0, W, k), rng.uniform(0, H, k)]
    return np.ascontiguousarray(X, np.float32), np.ascontiguousarray(x, np.float32), R, t


def cases():
    """The parameter grid of the whole-call checks: every m x outlier ratio x motion, with noise, threshold, depth and iterations cycling.
    Yields (name, seed, m, outliers, noise, motion, depth, threshold, iterations, confidence)."""
    i = 0
    for m in M_VALUES:
        for outl in OUTLIERS:
            for motion in MOTIONS:
                noise = NOISE[i % len(NOISE)]
                thr = THRESHOLDS[(i // 3) % len(THRESHOLDS)]
                depth = DEPTHS[(i // 2) % len(DEPTHS)]
                iters = (100, 1, 1000)[(i // 5) % 3]
                conf = (0.99, 0.999)[i % 2]
                yield (f"m{m}_o{outl}_{motion}_{depth}_n{noise}_t{thr}_i{iters}", 1000 + i, m, outl, noise, motion, depth, thr, iters, conf)
                i += 1
