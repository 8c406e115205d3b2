"""CPU test: the oracle (oracle/hv_oracle_triangulate.c) and cv2.triangulatePoints against the 50-digit reference of
tests/triangulate_ref.py on every scene of tests/triangulate_common.py. The angle between a returned column and the exact null vector
must satisfy

    sin ∠ <= 64 u σ1 / (σ3 − σ4) + 4 u_f32

(u = 2^-53; σ the singular values of the DLT matrix, descending): a backward-stable SVD of A perturbed by a few u σ1, plus the
rounding of the column to float. Where σ3 ≈ σ4 the bound exceeds 1 and says nothing (the null space is not a line: P1 == P2 with equal
points, for one); the test counts and names those points rather than passing them silently."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
import triangulate_common as tc  # noqa: E402
import triangulate_ref as ref  # noqa: E402

cv2 = pytest.importorskip("cv2")
mp = pytest.importorskip("mpmath")
U, UF = 2.0 ** -53, 2.0 ** -24
PER_SCENE = 40


@pytest.fixture(scope="module")
def orc():
    from oracle import triangulate_oracle
    if not os.path.exists(triangulate_oracle.ORACLE_SO):
        subprocess.check_call(["make", "-C", ROOT, "oracle"])
    return triangulate_oracle.OracleTriangulate()


def test_oracle_and_cv2_are_within_the_bound_of_the_exact_null_vector(orc):
    vacuous, checked, worst = {}, 0, 0.0
    for name, fam, P1, P2, a, b in tc.scenes():
        a, b = a[:PER_SCENE], b[:PER_SCENE]
        X4 = orc.triangulate(P1, P2, a, b)[0]
        C4 = cv2.triangulatePoints(P1, P2, np.ascontiguousarray(a.T), np.ascontiguousarray(b.T))
        for i in range(a.shape[0]):
            v, s = ref.null_vector(P1, P2, a[i], b[i])
            gap = s[2] - s[3]
            bound = 64 * U * s[0] / gap + 4 * UF if gap > 0 else mp.inf
            if bound >= 1:
                vacuous[name] = vacuous.get(name, 0) + 1
                continue
            for who, q in (("oracle", X4[:, i]), ("cv2", C4[:, i])):
                e = ref.sin_angle(q, v)
                assert e <= bound, f"{name} point {i} ({who}): sin angle {mp.nstr(e, 5)} above {mp.nstr(bound, 5)}"
                worst = max(worst, float(e / bound))
            checked += 1
    assert checked >= 500
    print(f"{checked} points within the bound (largest error / bound {worst:.3g}); bound vacuous (σ3 ≈ σ4) at: {vacuous or 'none'}")
    assert set(vacuous) <= {"P1 == P2"}, vacuous


def test_reference_sees_the_rank_of_p1_equal_p2():
    """P1 == P2 with equal points: rank 2, so σ3 = σ4 = 0 in the reference -- the case the bound cannot cover"""
    P1, _ = tc.stereo_pair()
    _, s = ref.null_vector(P1, P1, (100.0, 50.0), (100.0, 50.0))
    assert s[3] == 0 and s[2] < mp.mpf(10) ** -40 * s[0] and s[1] > 1e-3 * s[0]
