"""CPU: the P3P solver of the solvePnPRansac oracle (oracle/hv_oracle_pnp.c, which the device matches bit for bit) against the
extended-precision reference of tests/pnp_ref.py. The families are general triples from the seeded scenes, nearly collinear world
points, and cameras on or near the danger cylinder (the cylinder through the triangle's circumcircle, perpendicular to its plane),
where two solutions merge into a double root.

The gates apply to every fp64-determined triple (the reference's count unchanged under 4-ulp perturbations of the inputs):
- the oracle's count equals the reference's, so no root is lost and none is spurious;
- each reference solution (s1, s2, s3), the distances along the rays, has an oracle solution within (64 u max(kappa, 1) + 1024 u) of it,
  relatively. kappa is the solution's componentwise condition number. The absolute term covers the solver's own rounding of the
  rays and of the pose it returns, from which the distances are recomputed here.
Triples that are not fp64-determined are counted and not gated. On them, a different count is a property of the input, not of the
solver."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import pnp_common as pc  # noqa: E402
import pnp_ref  # noqa: E402

U = 2.0 ** -53
KK = (pc.FX, pc.FY, pc.CX, pc.CY)


@pytest.fixture(scope="module")
def orc():
    import subprocess
    from oracle import pnp_oracle
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if not os.path.exists(pnp_oracle.ORACLE_SO):
        subprocess.check_call(["make", "-C", root, "oracle"])
    return pnp_oracle.OraclePnp()


def _project(X, C, target):
    """pixels (float32) of X (3, 3) in a camera at C looking at target"""
    z = (target - C) / np.linalg.norm(target - C)
    x = np.cross([0.0, 1.0, 0.0], z)
    x /= np.linalg.norm(x)
    R = np.stack([x, np.cross(z, x), z])
    Xc = (R @ (X - C).T).T
    return (pc.K @ Xc.T).T[:, :2] / Xc[:, 2:]


def general(n):
    rng = np.random.default_rng(71)
    for k in range(n):
        X, x, _, _ = pc.scene(rng, 3, 0.0, 0.0, pc.MOTIONS[k % 3], pc.DEPTHS[k % 2])
        yield f"general-{k}", X.astype(np.float64), x


def collinear():
    rng = np.random.default_rng(72)
    for k, eps in enumerate([1e-2, 1e-3, 1e-4, 1e-6] * 10):
        A, B = rng.uniform(-2, 2, 3), rng.uniform(-2, 2, 3)
        perp = np.cross(B - A, rng.normal(size=3))
        X = np.stack([A, B, 0.5 * (A + B) + eps * perp / np.linalg.norm(perp)])
        C = 0.5 * (A + B) + np.array([0.3, -0.2, -6.0])
        yield f"collinear-{eps}-{k}", X, _project(X, C, X.mean(0)).astype(np.float32)


def danger_cylinder():
    rng = np.random.default_rng(73)
    for k, d in enumerate([0.0, 1e-6, 1e-4, 1e-2, 0.1] * 8):
        X = np.c_[rng.uniform(-2, 2, (3, 2)), np.zeros(3)]                      # the triangle in z = 0
        a, b, c = X
        A = 2 * np.array([[b[0] - a[0], b[1] - a[1]], [c[0] - a[0], c[1] - a[1]]])
        rhs = np.array([b[:2] @ b[:2] - a[:2] @ a[:2], c[:2] @ c[:2] - a[:2] @ a[:2]])
        o = np.linalg.solve(A, rhs)
        r = np.linalg.norm(a[:2] - o)
        th = rng.uniform(0, 2 * np.pi)
        C = np.r_[o + r * (1 + d) * np.array([np.cos(th), np.sin(th)]), rng.uniform(2, 6)]
        yield f"cylinder-{d}-{k}", X, _project(X, C, X.mean(0)).astype(np.float32)


def _distances(sols, X):
    return [np.linalg.norm((R @ X.T).T + t, axis=1) for R, t in sols]


def _check(orc, family):
    gated = undetermined = 0
    worst = 0.0
    for name, X, x in family:
        ref, sturm, determined, kappas = pnp_ref.reference(X, x, *KK)
        assert sturm >= len(ref), name
        got = _distances(orc.p3p(X, x, *KK), X)
        if not determined:
            undetermined += 1
            continue
        gated += 1
        assert len(got) == len(ref), f"{name}: {len(got)} solutions, the reference has {len(ref)}"
        for s, kap in zip(ref, kappas):
            s = np.array(s)
            err = min(np.abs(g - s).max() / np.abs(s).max() for g in got)
            tol = 64 * U * max(kap, 1.0) + 1024 * U
            worst = max(worst, err / tol)
            assert err <= tol, f"{name}: solution {s} off by {err:.2e} (tolerance {tol:.2e}, kappa {kap:.2e})"
    print(f"gated {gated}, undetermined {undetermined}, worst error / tolerance {worst:.3f}")
    return gated


def test_general_triples(orc):
    assert _check(orc, general(120)) >= 100


def test_nearly_collinear_triples(orc):
    _check(orc, collinear())


def test_near_the_danger_cylinder(orc):
    _check(orc, danger_cylinder())
