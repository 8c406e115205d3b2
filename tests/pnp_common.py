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


# ---------------------------------------------------------------------------------------------------- EPnP reference scenes
EPNP_SLAB_SEEDS = (14, 23, 98, 191)      # near-planar scenes on which a mirrored rotation was once returned
EPNP_SLABS = (0.0, 1e-6, 1e-4, 1e-2)


def _project(X, R, t, rng, noise):
    """float32 pixels of the float32 world points X under (R, t), exact but for the rounding, plus `noise` pixels of Gaussian noise"""
    Xc = (R @ X.astype(np.float64).T).T + t
    u = (K @ Xc.T).T
    return np.ascontiguousarray(u[:, :2] / u[:, 2:] + rng.normal(0, noise, (X.shape[0], 2)), np.float32)


def slab(seed, m, thick, noise):
    """pc.scene(m, "near") with the world's z replaced by 4 + thick N(0, 1): points on a plane (thick = 0) or in a slab, as a floor
    or a wall is; the motion cycles with the seed. Returns (X, x, R, t)."""
    rng = np.random.default_rng(seed)
    X, _, R, t = scene(rng, m, 0.0, 0.0, MOTIONS[seed % 3], "near")
    X = X.astype(np.float64)
    X[:, 2] = 4.0 + thick * rng.normal(size=m)
    X = X.astype(np.float32)
    return X, _project(X, R, t, rng, noise), R, t


def far(seed, m, scale, noise):
    """pc.scene(m, depth "far") with the world and the translation scaled by `scale` (the pixels of a scene do not change with its
    scale): 20 scale to 60 scale metres away. Returns (X, x, R, t)."""
    rng = np.random.default_rng(seed)
    X, _, R, t = scene(rng, m, 0.0, 0.0, MOTIONS[seed % 3], "far")
    X = (X.astype(np.float64) * scale).astype(np.float32)
    return X, _project(X, R, t * scale, rng, noise), R, t * scale


def near_pi(seed, m, delta, noise):
    """points 2-6 m in front of a camera whose rotation is pi - delta about a random axis. Returns (X, x, R, t)."""
    rng = np.random.default_rng(seed)
    Z = rng.uniform(2.0, 6.0, m)
    u, v = rng.uniform(20, W - 20, m), rng.uniform(20, H - 20, m)
    Xc = np.c_[(u - CX) / FX * Z, (v - CY) / FY * Z, Z]
    n = rng.normal(size=3)
    R = _rodrigues((np.pi - delta) * n / np.linalg.norm(n))
    t = rng.normal(0, 0.2, 3)
    X = (R.T @ (Xc - t).T).T.astype(np.float32)
    return X, _project(X, R, t, rng, noise), R, t


def epnp_families():
    """{family: [(name, X, x), ...]} of the EPnP reference checks: general clouds at every motion and both depths, m = 6 to 600 with
    noise 0 / 0.5 / 1 cycling; m = 4096; slabs (the seeds above at every thickness, noise-free, and two of them with 0.5 px noise);
    far depths; rotations near pi."""
    fam = {"general": [], "m4096": [], "slab": [], "far": [], "near_pi": []}
    i = 0
    for m, k in ((6, 4), (8, 4), (20, 4), (150, 6), (600, 3)):
        for j in range(k):
            motion, depth, noise = MOTIONS[(i + j) % 3], DEPTHS[j % 2], NOISE[i % 3]
            X, x, _, _ = scene(np.random.default_rng(500 + i), m, 0.0, noise, motion, depth)
            fam["general"].append((f"m{m}_{motion}_{depth}_n{noise}", X, x))
            i += 1
    for seed, noise in ((601, 0.5), (602, 0.0)):
        X, x, _, _ = scene(np.random.default_rng(seed), 4096, 0.0, noise, MOTIONS[seed % 3], DEPTHS[seed % 2])
        fam["m4096"].append((f"m4096_n{noise}", X, x))
    for seed in EPNP_SLAB_SEEDS:
        for thick in EPNP_SLABS:
            for noise in ((0.0, 0.5) if seed in (14, 191) else (0.0,)):
                fam["slab"].append((f"slab_{seed}_{thick}_n{noise}", *slab(seed, 150, thick, noise)[:2]))
    for seed, scale, noise in ((700, 10.0, 0.0), (701, 10.0, 0.5), (702, 100.0, 0.0), (703, 100.0, 0.5)):
        fam["far"].append((f"far_x{scale}_n{noise}", *far(seed, 150, scale, noise)[:2]))
    for k, delta in enumerate((1e-2, 1e-4, 1e-6, 0.0)):
        for noise in (0.0, 0.5):
            fam["near_pi"].append((f"pi-{delta}_n{noise}", *near_pi(800 + 2 * k + (noise > 0), 150, delta, noise)[:2]))
    return fam
