"""CPU tests of the extended-precision predict reference (tests/predict_ref.py) that the GPU sweep of the IMU predict kernel compares
against: the reference must agree with the C oracle within its bound on every case of the sweep, the comparator must reject subtly
wrong results that the max|dP| / max|P| gate of the other EKF tests accepts, and the sweep's inputs and shapes must reach both rotation
branches and every strip-tile configuration of the kernel."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import ekf_common as C
import ekf_script
import predict_ref as PR


def _params(trail, ms, walk=None):
    from oracle import ekf_oracle
    o = ekf_oracle.OracleEKF()
    p = o.default_params()
    o.close()
    return PR.with_walk(C.params_with(lambda: p, trail, ms), walk or {})


CASES = PR.sweep_cases()


@pytest.mark.parametrize("start,trail,ms,name", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_reference_agrees_with_c_oracle(oracle_lk, start, trail, ms, name):
    """The C oracle (fp64, sample by sample, Taylor-series matrix exponential) is within the bound in m, P and dydx."""
    from oracle import ekf_oracle
    probe = ekf_oracle.OracleEKF(_params(trail, ms))
    bg = PR.start_state(start, probe)[0][PR.BGA:PR.BGA + 3]
    probe.close()
    pat = PR.make_pattern(name, bg)
    p = _params(trail, ms, pat.walk)
    o = ekf_oracle.OracleEKF(p)
    m, P = PR.start_state(start, o)
    ref = PR.Reference(p, m, P)
    PR.drive(o, pat.calls, ref)
    gm, gP = o.download()
    r = PR.ratios(ref, gm, gP, o.get_dydx())
    o.close()
    print(f"\nN={len(m)} {start} {name}: oracle error / bound m {r['m']:.3g} P {r['P']:.3g} dydx {r['dydx']:.3g}")
    assert max(r.values()) <= 1.0, r


def _fault_state():
    """A filter after ten frames of tests/ekf_script.run_frames at trail 20 (C oracle): the recent trail slots are correlated with the
    inertial state, the others still hold the 1e8 prior, so max|P| = 1e8. The quaternion is scaled by 1.05 (the norm of the dense
    state's) so that where a normalisation happens shows in the result (until the first normalisation, after sample 0 of the burst)."""
    from oracle import ekf_oracle
    o = ekf_oracle.OracleEKF(_params(20, 0))
    ekf_script.run_frames(o, frames=10, n_list=(8, 20, 40))
    m, P = o.download()
    o.close()
    m[PR.ORI:PR.ORI + 4] *= 1.05
    return m, P


@pytest.mark.parametrize("norm", ["some", "every"])
@pytest.mark.parametrize("state", ["frames", "dense"])
def test_comparator_rejects_injected_faults(oracle_lk, state, norm):
    """Each fault, injected into the reference at one sample of a 16-sample jittered burst with the gyro-bias random walk on, moves m or
    P by more than 10x the bound, with some normalisations and with a normalisation after every sample (the reference's own loop,
    backend.cpp:734-735). From the filter after ten frames, the max|dP| / max|P| < 1e-9 gate accepts at least the P(vel, bat) scaling, the
    strips without the last sample's D and the P00 product without D's columns 16..19: that is the gap this comparator closes."""
    if state == "frames":
        m, P = _fault_state()
        assert np.abs(P).max() == 1e8 and np.abs(P[20:, :20]).max() > 0
    else:
        m, P = PR.dense_state(PR.state_dim(20, 0))
    p = _params(20, 0, PR.WALKS["bga-rev0.1"])
    calls = PR.jitter_calls(n=16, seed=3, norm=norm)
    # the host drops the first call; no normalisation after it, so that the quaternion keeps its norm of 1.05 through sample 0
    calls[0] = calls[0][:3] + (False,)
    good = PR.reference_run(p, m, P, calls)
    assert good.k == 16
    at = {"p_vel_bat": 8, "stale_drift_q": 8, "strips_miss_last_d": 15, "late_normalisation": 0, "d_cols_16_19_dropped": 8,
          "previous_sinc": 8}
    assert set(at) == set(PR.FAULTS) and calls[at["late_normalisation"] + 1][3]
    for name, k in at.items():
        bad = PR.reference_run(p, m, P, calls, faults={name: k})
        r = max(PR.ratios(good, bad.m, bad.P).values())
        rel = ekf_script.rel_err(np.asarray(bad.P, np.float64), np.asarray(good.P, np.float64))
        print(f"\n{state} {norm} {name} at sample {k}: error / bound {r:.3g}, max|dP| / max|P| {rel:.3g}")
        assert r >= 10.0, name
        if state == "frames" and name in ("p_vel_bat", "strips_miss_last_d", "d_cols_16_19_dropped"):
            assert rel < C.TOL_P_REL, name


def test_sweep_reaches_both_rotation_branches_and_every_strip_tiling():
    """The boundary samples lie just below, exactly at and just above x = 0.01 in the kernel's fp64 expression; the large-rotation
    patterns take the closed form and ordinary samples the series; the 0.1 s gap the closed form and the 0.5 s gap the series. The shapes
    have trail 1 (N = 27), every rest % 8, ntile on both sides of 16, 32 and 48, ntile > 96 and N >= 700."""
    for bg in (np.zeros(3), PR.dense_state(PR.state_dim(PR.BASE_TRAIL, 0))[0][PR.BGA:PR.BGA + 3]):
        calls = PR.boundary_calls(bg)
        xs, prev = [], None
        for t, g, a, _ in calls:
            if prev is not None:
                xs.append(PR.rotation_x(np.asarray(g) - bg, t - prev))
            prev = t
        below, at, above = xs[0], xs[2], xs[4]
        assert below < PR.BRANCH_X and at == PR.BRANCH_X and above > PR.BRANCH_X
        assert np.nextafter(below, np.inf) >= PR.BRANCH_X * (1 - 4 * PR.U) and above <= PR.BRANCH_X * (1 + 4 * PR.U)
        assert PR.branches(calls, bg) == [False, False, True, False, True, False]
    zero = np.zeros(3)
    assert all(PR.branches(PR.rotation_calls("large"), zero))
    mixed = PR.branches(PR.rotation_calls("mixed"), zero)
    assert any(mixed) and not all(mixed)
    assert not any(PR.branches(PR.burst(17, "never"), zero))
    irr = PR.irregular_calls()
    ts = [c[0] for c in irr]
    assert PR.branches(irr, zero).count(True) == 1 and len(PR.branches(irr, zero)) == len(irr) - 3      # first, duplicate, backwards
    assert any(abs(b - a - 0.1) < 1e-12 for a, b in zip(ts, ts[1:])) and any(abs(b - a - 0.5) < 1e-12 for a, b in zip(ts, ts[1:]))

    shapes = PR.sweep_shapes()
    geo = [(t, PR.state_dim(t, ms), *PR.strip_geometry(PR.state_dim(t, ms))) for t, ms in shapes]
    assert any(t == 1 and N == 27 for t, N, _, _ in geo)
    assert {rest % 8 for _, _, rest, _ in geo} == set(range(8))
    nts = {nt for _, _, _, nt in geo}
    assert {16, 17, 32, 33, 48, 49} <= nts and max(nts) > 96 and max(N for _, N, _, _ in geo) >= 700
    assert max(PR.strip_passes(nt) for nt in nts) >= 3


def test_dense_start_state_spans_the_stated_range():
    """(b): diagonal from 1e-12 to 1e8, correlations up to 0.999, quaternion of norm 1.05."""
    m, P = PR.dense_state(PR.state_dim(PR.BASE_TRAIL, 0))
    d = np.diag(P)
    assert np.isclose(d.min(), 1e-12) and np.isclose(d.max(), 1e8)
    corr = P / np.sqrt(d[:, None] * d[None, :])
    np.fill_diagonal(corr, 0)
    assert 0.99 < np.abs(corr).max() < 1.0
    assert np.isclose(np.linalg.norm(m[PR.ORI:PR.ORI + 4]), 1.05)
    assert np.array_equal(P, P.T)
