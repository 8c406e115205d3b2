"""CPU tests of the componentwise reference of the visual Kalman update (tests/visual_update_ref.py): the C oracle is within the
per-entry bound on every realistic case, faults that the normwise 1e-9 gates of ekf_common let through fail the bound by orders of
magnitude, and the cases reach every kernel path the launchers can pick on their state layouts."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ekf_common as C  # noqa: E402
import ekf_ops_ref as E  # noqa: E402
import kalman_ref as K  # noqa: E402
import visual_update_ref as V  # noqa: E402

CASES = V.cases()


def _f64(res):
    return np.asarray(res.m, np.float64), np.asarray(res.P, np.float64)


def _old_gates_pass(m, P, m_ref, P_ref):
    return np.abs(m - m_ref).max() < C.TOL_M and np.abs(P - P_ref).max() / np.abs(P_ref).max() < C.TOL_P_REL


def _ratio(res, m, P):
    return max(E.bound_ratio(m, res.m, res.Bm), E.bound_ratio(P, res.P, res.BP))


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_c_oracle_is_within_the_per_entry_bound(oracle_lk, case):
    """OracleEKF.visual_update (fp64 Cholesky) against the longdouble reference, every entry of m and P within its bound; the check
    (inlier and gross outlier) against chi2 within tau."""
    from oracle import ekf_oracle
    c = case
    ref = c.reference()
    o = ekf_oracle.OracleEKF(V.oracle_params(c.trail, c.ms))
    o.upload(c.m, c.P)
    st, c2 = o.visual_check(c.H, c.f, c.y, V.R_VIS)
    st_out, _ = o.visual_check(c.H, c.f, c.y_out, V.R_VIS)
    o.visual_update(c.H, c.f, c.y, V.R_VIS)
    m1, P1 = o.download()
    o.close()
    r, where = V.worst(ref, m1, P1, c.trail, c.ms)
    print(f"\n{c.name} {'/'.join(c.path)} kappa={ref.kappa:.3g} C_VIS={ref.C:g}: oracle worst ratio {r:.3g} at {where}")
    assert r <= 1.0, where
    if c.n <= K.CHI2_MAX_N:
        ref_st, ref_c2 = K.check(c.P, c.H, c.f, c.y, V.R_VIS, 100.0)
        assert st == ref_st == 0 and st_out == 3
        assert K.chi2_error(ref_c2, c2) <= K.tau(c.n, ref.kappa)


def test_row_chunked_reference_is_the_same_update():
    """The chunked form of the reference (a downdate per chunk of rows, residuals corrected by H_k (m_cur - m_0)) is within the bound
    of the whole update: the equivalence the row-chunked kernel rests on."""
    c = V.Case("map47", (V._S(21),), 5)
    ref = c.reference()
    for chunks in (2, 3, V.chain_chunks(c.n, c.l, c.N)):
        r = _ratio(ref, *_f64(c.reference(chunks=chunks)))
        print(f"{c.name}: {chunks} chunks, ratio {r:.3g}")
        assert r <= 1.0


@pytest.mark.parametrize("spec", [(V._S(9),), (V._S(14),)], ids=["n36", "n56"])
def test_per_entry_bound_rejects_faults_the_normwise_gates_accept(spec):
    """Each fault passes ekf_common's gates (|dm| < 1e-9 absolute, max|dP| / max|P| < 1e-9) and fails the per-entry bound by at least
    100x: the last inertial row and column (the time shift) not downdated, the bias rows and columns scaled by 1 + 1e-9, entries below
    1e-13 max|P| flushed to zero, m's accelerometer-transform and time-shift entries left at their prior, and a chunked update whose
    later chunks use m_0 instead of m_cur in their residual (on a track that agrees with its prediction to 1e-4 of the noise, where the
    mean barely moves)."""
    c = V.Case("filled", spec, 77)
    good = c.reference()
    m1, P1 = _f64(good)
    A = np.abs(P1)
    faults = {}
    X = P1.copy(); X[E.SFT, :] = c.P[E.SFT, :]; X[:, E.SFT] = c.P[:, E.SFT]
    faults["time-shift row / column not downdated"] = (good, m1, X)
    X = P1.copy(); X[E.BGA:E.SFT, :] *= 1 + 1e-9; X[:, E.BGA:E.SFT] *= 1 + 1e-9
    faults["bias rows / columns x (1 + 1e-9)"] = (good, m1, X)
    X = P1.copy(); X[A < 1e-13 * A.max()] = 0.0
    faults["entries < 1e-13 max|P| flushed"] = (good, m1, X)
    mm = m1.copy(); mm[E.BAT:E.SFT + 1] = c.m[E.BAT:E.SFT + 1]
    faults["m accelerometer transform + time shift at prior"] = (good, mm, P1)
    y = c.f + 1e-4 * (c.y - c.f)
    quiet = c.reference(y=y)
    faults["chunked: residual from m_0"] = (quiet, *_f64(c.reference(y=y, chunks=3, stale_residual=True)))
    for name, (ref, m, P) in faults.items():
        mr, Pr = _f64(ref)
        old = _old_gates_pass(m, P, mr, Pr)
        r = _ratio(ref, m, P)
        print(f"{c.name}: {name}: normwise |dm| {np.abs(m - mr).max():.2e}, dP {np.abs(P - Pr).max() / np.abs(Pr).max():.2e} "
              f"(1e-9 gates {'pass' if old else 'fail'}), per-entry ratio {r:.3g}")
        assert old, name
        assert r >= 100.0, name


def test_cases_reach_every_kernel_path():
    """Per state layout, the kernel paths the cases take (each case also runs with H 8 bytes past a 16-byte boundary, which stages H
    without bulk copies) include every path kalman_ref.reachable names there; each of the check batch's row counts 8 / 20 / 40 / 84 is
    a case on the benchmark's layout; and the device chain runs the 84-row tracks of the map layouts in row chunks."""
    got = {}
    for c in CASES:
        got.setdefault((c.trail, c.ms), set()).update({c.path, c.path_misaligned})
    for (trail, ms), paths in sorted(got.items()):
        print(f"N={K.state_dim(trail, ms)}: " + ", ".join(sorted("/".join(p) for p in paths)))
    for trail, ms in V.LAYOUTS:
        missing = set(K.reachable(trail, ms)) - got[(trail, ms)]
        assert not missing, (K.state_dim(trail, ms), missing)
    ns = {c.n for c in CASES if c.N == 160}
    assert set(V.CHECK_BATCH_N) <= ns
    assert {c.N for c in CASES if c.n == 84 and V.chain_chunks(c.n, c.l, c.N) > 1} >= {202, 301, 400}
