"""GPU: the EPnP pose that the device's hv_solve_pnp_ransac returns, against the extended-precision reference of tests/epnp_ref.py
and bit for bit against the oracle (oracle/hv_oracle_pnp.c): t and rvec, which is what the device returns (the oracle's R is
checked in tests/test_epnp_ref.py). The scenes are those of tests/test_epnp_ref.py with no outliers, and the
threshold is 8 px, so that the final EPnP runs on nearly every point (a 4-point RANSAC model on noisy points can leave out a few);
the reference is computed on the inliers the device reports."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import epnp_ref  # noqa: E402
import pnp_common as pc  # noqa: E402
from test_epnp_ref import MIN_GATED, reference_of  # noqa: E402
from test_gpu_pnp import _host, _same  # noqa: E402

pytestmark = pytest.mark.gpu
KK = (pc.FX, pc.FY, pc.CX, pc.CY)
FAMILIES = pc.epnp_families()


@pytest.fixture(scope="module")
def orc():
    import subprocess
    from oracle import pnp_oracle
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if not os.path.exists(pnp_oracle.ORACLE_SO):
        subprocess.check_call(["make", "-C", root, "oracle"])
    return pnp_oracle.OraclePnp()


@pytest.mark.parametrize("family", list(FAMILIES))
def test_device_epnp_matches_the_reference(hv, orc, family):
    gated = 0
    for name, X, x in FAMILIES[family]:
        got = _host(hv, X, x, 100, 8.0, 0.99)
        _same(got, orc.solve_pnp_ransac(X, x, *KK, 100, 8.0, 0.99), name)
        ok, r, t, mask, inl = got
        assert ok == 1 and inl >= 0.9 * X.shape[0], f"{name}: {inl} of {X.shape[0]} inliers"
        sel = mask.astype(bool)                         # the final EPnP runs on the RANSAC model's inliers, in index order
        ref = reference_of(orc, X[sel], x[sel])
        if ref["determined"]:
            epnp_ref.check(ref, None, t, r, name)
            gated += 1
    assert gated >= MIN_GATED[family]
