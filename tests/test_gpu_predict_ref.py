"""GPU sweep of the fused IMU predict kernel against the extended-precision reference (tests/predict_ref.py), through the C ABI only:
from both starting states, bursts of 1..17 samples under every normalisation mode, both rotation branches and their boundary,
irregular timestamps, the bias random walks, and the strip geometries the kernel deals tiles for. m, P and dydx must lie within the
reference's componentwise bound (entries with a zero bound exact); the worst error / bound and the oracle's max|dP_ij| / sqrt(P_ii P_jj)
are printed per case."""
import ctypes
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import ekf_common as C
import predict_ref as PR

pytestmark = pytest.mark.gpu


def _params(trail, ms, walk=None):
    from hybvio_b200 import capi
    p = capi.EkfParams()
    capi.load().hv_ekf_default_params(ctypes.byref(p))
    return PR.with_walk(C.params_with(lambda: p, trail, ms), walk or {})


CASES = PR.sweep_cases()


@pytest.mark.parametrize("start,trail,ms,name", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_predict_matches_extended_precision_reference(hv, oracle_lk, start, trail, ms, name):
    import torch
    from hybvio_b200 import capi
    from oracle import ekf_oracle
    N = PR.state_dim(trail, ms)
    bg = np.zeros(3) if start == "default" else PR.dense_state(N)[0][PR.BGA:PR.BGA + 3]
    pat = PR.make_pattern(name, bg)
    p = _params(trail, ms, pat.walk)
    e = capi.Ekf(hv, p)
    e.set_imu_batching(pat.batch)
    m0, P0 = PR.start_state(start, e)
    assert np.array_equal(m0[PR.BGA:PR.BGA + 3], bg)
    ref = PR.Reference(p, m0, P0)
    PR.drive(e, pat.calls, ref)
    if pat.mean_launch:
        d = torch.zeros(20, dtype=torch.float64, device="cuda")
        e.predicted_mean_device(d.data_ptr())
        torch.cuda.synchronize()
        pred = d.cpu().numpy().copy()
    e.flush()
    m, P = e.download()
    dydx = e.get_dydx()
    e.close()

    o = ekf_oracle.OracleEKF(p)
    o.upload(m0, P0)
    PR.drive(o, pat.calls)
    _, Po = o.download()
    o.close()

    r = PR.ratios(ref, m, P, dydx)
    zeros = int(((ref.BP == 0) & (ref.P == 0)).sum())
    print(f"\nPREDICT {start} N={N} {name}: samples {ref.k}, worst error / bound m {r['m']:.3g} P {r['P']:.3g} dydx {r['dydx']:.3g}; "
          f"exact zeros {zeros}; oracle scaled error {PR.scaled_error(Po, ref.P):.3g}, kernel {PR.scaled_error(P, ref.P):.3g}")
    for what, v in r.items():
        assert v <= 1.0, f"{what}: error / bound = {v:.3g}"
    if start == "default":
        assert zeros > 0 and not P[(ref.BP == 0) & (ref.P == 0)].any(), "a structural zero moved"
    if pat.mean_launch:
        assert np.array_equal(pred, m[:20]), np.abs(pred - m[:20]).max()
