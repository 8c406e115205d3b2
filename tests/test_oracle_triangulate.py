"""CPU test: the plain-C restatement of cv::triangulatePoints + cv::convertPointsFromHomogeneous (oracle/hv_oracle_triangulate.c)
against cv2 4.13 on the seeded scenes of tests/triangulate_common.py.

- General scenes (rectified stereo with pixel noise, general two-view): X4 and xyz bit-identical to cv2's. The restatement sums in index
  order and cv2 in SIMD lanes, so a departure of at most 1 float32 ulp is tolerated -- counted and reported with the scene's name.
- Every scene: every column points the way cv2's does (positive dot product), and the sign of w equals cv2's except where w is rounding
  noise (|w| at most 64 u |Q|: the point is at infinity, and no sign is meaningful), which the test names.
- The checks have teeth: numpy's SVD (LAPACK's sign convention) and the restatement without OpenCV's final sort each fail them."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
import triangulate_common as tc  # noqa: E402

cv2 = pytest.importorskip("cv2")
U64 = np.finfo(np.float64).eps / 2


@pytest.fixture(scope="module")
def orc():
    from oracle import triangulate_oracle
    if not os.path.exists(triangulate_oracle.ORACLE_SO):
        subprocess.check_call(["make", "-C", ROOT, "oracle"])
    return triangulate_oracle.OracleTriangulate()


def _cv2(P1, P2, a, b):
    X4 = cv2.triangulatePoints(P1, P2, np.ascontiguousarray(a.T), np.ascontiguousarray(b.T))
    return X4, cv2.convertPointsFromHomogeneous(np.ascontiguousarray(X4.T)).reshape(-1, 3)


def _ulps(a, b):
    """float32 ulp distance per element (the ordered-integer difference; +0 and -0 are 0 apart)"""
    def ordered(x):
        i = np.ascontiguousarray(x, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(ordered(a) - ordered(b))


def _sign_check(X4, want):
    """(columns pointing against cv2's, w signs that differ where w is not rounding noise, w signs that differ where it is)"""
    q, r = X4.astype(np.float64), want.astype(np.float64)
    against = int(np.sum((q * r).sum(0) <= 0.0))
    noise = np.abs(r[3]) <= 64 * U64 * np.linalg.norm(r, axis=0)
    flip = np.sign(q[3]) != np.sign(r[3])
    return against, int(np.sum(flip & ~noise)), int(np.sum(flip & noise))


def test_general_scenes_are_cv2s_bits(orc):
    departures = []
    total = 0
    for name, fam, P1, P2, a, b in tc.scenes():
        if fam != "general":
            continue
        X4, xyz, used = orc.triangulate(P1, P2, a, b)
        want, wxyz = _cv2(P1, P2, a, b)
        assert X4.shape == want.shape and X4.dtype == want.dtype == np.float32 and used.all()
        u4, u3 = _ulps(X4, want), _ulps(xyz, wxyz)
        assert u4.max() <= 1 and u3.max() <= 1, f"{name}: {u4.max()} / {u3.max()} ulps from cv2"
        n = int(np.sum(u4.max(0) > 0) + np.sum(u3.max(1) > 0))
        if n:
            departures.append(f"{name}: {n}")
        total += a.shape[0]
        assert _sign_check(X4, want)[:2] == (0, 0), name
    print(f"{total} general points; columns 1 ulp from cv2: {departures or 'none'}")


def test_every_scene_has_cv2s_signs(orc):
    noise = []
    for name, fam, P1, P2, a, b in tc.scenes():
        X4, xyz, _ = orc.triangulate(P1, P2, a, b)
        want, wxyz = _cv2(P1, P2, a, b)
        against, flips, noisy = _sign_check(X4, want)
        assert against == 0 and flips == 0, f"{name}: {against} columns against cv2's, {flips} signs of w differ"
        if noisy:
            noise.append(f"{name}: {noisy}")
        if fam == "degenerate":
            bits = np.all(X4.view(np.uint32) == want.view(np.uint32), axis=0)
            print(f"{name}: {int(bits.sum())}/{bits.size} columns bit-identical to cv2")
    print(f"w signs that differ where w is rounding noise (a point at infinity): {noise or 'none'}")


def test_rank_deficient_and_zero_status_columns(orc):
    """P1 == P2 with equal points: rank 2, cv2 returns (0, 0, 0, 1) (its V^T's last row is e4); unused points give zero columns"""
    P1, _ = tc.stereo_pair()
    x = np.array([[100.0, 50.0], [370.0, 240.0], [-3.0, 7.5]], np.float32)
    X4, xyz, used = orc.triangulate(P1, P1, x, x)
    want, _ = _cv2(P1, P1, x, x)
    assert np.array_equal(X4, want)
    assert np.array_equal(np.abs(want), np.tile(np.array([[0], [0], [0], [1]], np.float32), (1, 3)))
    st = np.array([1, 0, 5], np.uint8)
    X4s, xyzs, useds = orc.triangulate(P1, P1, x, x, st, np.array([7, 1, 0], np.uint8))
    assert useds.tolist() == [1, 0, 0] and not X4s[:, 1:].any() and not xyzs[1:].any() and np.array_equal(X4s[:, 0], X4[:, 0])


def test_convert_points_from_homogeneous_threshold():
    """cv2 leaves a column unscaled where |w| <= FLT_EPSILON and multiplies by the float 1 / w elsewhere; the oracle does the same"""
    from oracle.triangulate_oracle import OracleTriangulate  # noqa: F401 -- the rule is restated below as the oracle states it
    fe = np.finfo(np.float32).eps
    for w in (1e-8, fe, -fe, np.nextafter(fe, np.float32(1)), 3.0, -7.0, 0.0):
        Q = np.array([[1.0, 2.0, 3.0, w]], np.float32)
        got = cv2.convertPointsFromHomogeneous(Q).reshape(3)
        w32 = np.float32(w)
        scale = np.float32(1.0) / w32 if abs(w32) > fe else np.float32(1.0)
        assert np.array_equal(got, Q[0, :3] * scale), (w, got)


def _numpy_last_row(P1, P2, a, b):
    out = np.zeros((4, a.shape[0]), np.float32)
    for i in range(a.shape[0]):
        A = np.array([[float(x) * P[2, k] - P[r, k] for k in range(4)] for P, pt in ((P1, a[i]), (P2, b[i]))
                      for r, x in ((0, pt[0]), (1, pt[1]))])
        out[:, i] = np.linalg.svd(A)[2][3]
    return out


def test_the_checks_have_teeth(orc):
    """numpy's SVD (LAPACK's sign convention) fails the bits or the sign check on the general scenes. The restatement without OpenCV's
    final sort returns the same bits there: each rotation leaves the larger norm in the lower row, so the sort only moves rows that
    were never rotated against each other (exactly orthogonal columns of A). It fails on the scene built for that, a zero column in
    both P (null vector e1, left in row 0 by the sweeps). Only scenes on which the oracle itself passes the checks count."""
    def bad(X4, want):
        return _ulps(X4, want).max() > 1 or _sign_check(X4, want)[:2] != (0, 0)

    fails = {"numpy svd": [], "no sort": []}
    for name, fam, P1, P2, a, b in tc.scenes():
        want, _ = _cv2(P1, P2, a, b)
        if bad(orc.triangulate(P1, P2, a, b)[0], want):
            continue                        # zero disparity, baseline 1e-6: w or the whole column is rounding noise
        faults = [("no sort", orc.triangulate(P1, P2, a, b, sort=False)[0])]
        if fam == "general":
            faults.append(("numpy svd", _numpy_last_row(P1, P2, a, b)))
        for what, X4 in faults:
            if bad(X4, want):
                fails[what].append(name)
    assert fails["numpy svd"] and fails["no sort"] == ["zero first column in P1 and P2"], fails
    print(f"numpy svd fails on {fails['numpy svd']}")
