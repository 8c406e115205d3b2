"""CPU: the EPnP pose of the solvePnPRansac oracle (oracle/hv_oracle_pnp.c, which the device matches bit for bit) against the
extended-precision reference of tests/epnp_ref.py, on general clouds (m = 6 to 4096, noise 0 to 1 px, both depths), points on a plane
or in a thin slab (a floor or a wall), far depths and rotations near pi; and the library's trigonometry of + - * / and sqrt, with
Rodrigues near theta = pi, against mpmath.

Every fp64-determined scene (each discrete decision of EPnP the same under the reference's perturbations) is gated: R, t and rvec
within 16 spread + 64 u max(|x|, 1) per entry. The reference takes the sign of each control-point axis from the oracle; the axes
themselves must agree with the covariance's eigenvectors within 64 u max(1, lambda_1 / gap), plus the rounding of the control
points they are read from. Undetermined scenes are counted and not gated. EPnP on 4 or 5 points is not checked: its null space has more than one dimension, and any basis of it is valid."""
import os
import sys

import mpmath as mp
import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import epnp_ref  # noqa: E402
import pnp_common as pc  # noqa: E402

U = 2.0 ** -53
KK = (pc.FX, pc.FY, pc.CX, pc.CY)
FAMILIES = pc.epnp_families()
MIN_GATED = {"general": 18, "m4096": 2, "slab": 20, "far": 4, "near_pi": 7}


@pytest.fixture(scope="module")
def orc():
    import subprocess
    from oracle import pnp_oracle
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if not os.path.exists(pnp_oracle.ORACLE_SO):
        subprocess.check_call(["make", "-C", root, "oracle"])
    return pnp_oracle.OraclePnp()


def reference_of(orc, X, x):
    """the reference with the oracle's control-point axis signs, after checking the oracle's axes against it"""
    cws = orc.control_points(X)
    axes = cws[1:] - cws[0]
    ref = epnp_ref.reference(X, x, *KK, axes)
    lam = ref["eigenvalues"]
    keep = [d for d in ref["decisions"] if d[0] == "axes"][0][1]
    for i in range(3):
        if not keep[i]:
            assert np.abs(axes[i]).max() <= 4 * U * np.abs(axes).max(), f"axis {i} of a singular covariance: {axes[i]}"
            continue
        gap = min(abs(lam[i] - lam[j]) for j in range(3) if j != i)
        tol = 64 * U * max(1.0, lam[0] / gap) + 4 * U * np.abs(cws).max() / np.linalg.norm(axes[i])     # c0 + axis, rounded
        err = np.abs(axes[i] / np.linalg.norm(axes[i]) - ref["axes"][i]).max()
        assert err <= tol, f"control-point axis {i}: {axes[i]} against {ref['axes'][i]} ({err:.2e} > {tol:.2e})"
    return ref


@pytest.mark.parametrize("family", list(FAMILIES))
def test_epnp_matches_the_reference(orc, family):
    gated = undetermined = 0
    worst = 0.0
    for name, X, x in FAMILIES[family]:
        ref = reference_of(orc, X, x)
        if not ref["determined"]:
            undetermined += 1
            print(f"{name}: undetermined by {ref['undetermined_by']}")
            continue
        r, t, R = orc.epnp(X, x, *KK, rotation=True)
        worst = max(worst, epnp_ref.check(ref, R, t, r, name))
        gated += 1
    print(f"{family}: gated {gated}, undetermined {undetermined}, worst error / tolerance {worst:.3f}")
    assert gated >= MIN_GATED[family]


def test_sincos_and_atan2_against_mpmath(orc):
    for th in np.linspace(0.0, 4.0, 401):
        s, c = orc.sincos(th)
        ms, mc = mp.sin(mp.mpf(th)), mp.cos(mp.mpf(th))
        assert abs(s - float(ms)) <= 16 * U and abs(c - float(mc)) <= 16 * U, th      # three angle doublings multiply the series' rounding
    for th in np.r_[np.linspace(0.0, np.pi, 193), np.pi - np.logspace(-12, -1, 12)]:
        for rad in (1.0, 1e-3, 1e3):
            y, x = rad * np.sin(th), rad * np.cos(th)
            want = mp.atan2(mp.mpf(y), mp.mpf(x))
            assert abs(orc.atan2(y, x) - float(want)) <= 2 * U * max(1.0, float(want)), (y, x)


def _mp_rotation(n, th):
    n = [mp.mpf(float(c)) for c in n]
    nn = mp.sqrt(sum(c * c for c in n))
    n = [c / nn for c in n]
    c, s = mp.cos(th), mp.sin(th)
    K = mp.matrix([[0, -n[2], n[1]], [n[2], 0, -n[0]], [-n[1], n[0], 0]])
    return c * mp.eye(3) + (1 - c) * mp.matrix([[n[i] * n[j] for j in range(3)] for i in range(3)]) + s * K


@pytest.mark.parametrize("delta", [1e-2, 1e-4, 1e-6, 0.0])
def test_rodrigues_near_pi(orc, delta):
    """rvec of R (an mp rotation of angle pi - delta, rounded to double) against the mp axis-angle of that rotation. Where s >= 1e-5
    the tolerance is the rounding of R over sin(theta); where s < 1e-5 OpenCV's branch takes the axis from the diagonal, exact at
    theta = pi and off by about delta^2 / (8 |n_k|) otherwise, with the sign of its first component non-negative (compared up to sign). theta
    comes from atan2(s, c); OpenCV's acos(c) would lose half the digits here."""
    rng = np.random.default_rng(17)
    th = mp.pi - mp.mpf(delta)
    for _ in range(24):
        n = rng.normal(size=3)
        Rm = _mp_rotation(n, th)
        R = np.array([[float(Rm[i, j]) for j in range(3)] for i in range(3)])
        want, s = epnp_ref.axis_angle(Rm)
        want = np.array([float(c) for c in want])
        got = orc.rodrigues(R)
        if float(s) >= 1e-5:
            err, tol = np.abs(got - want).max(), 16 * U * np.pi / float(s)
        else:
            err = min(np.abs(got - want).max(), np.abs(got + want).max())
            tol = (64 * U + np.pi * delta * delta) / np.abs(want / np.linalg.norm(want)).min()
        assert err <= tol, (delta, n, got, want, err, tol)
        assert abs(np.linalg.norm(got) - float(th)) <= 64 * U + np.pi * delta * delta, (delta, np.linalg.norm(got), float(th))
