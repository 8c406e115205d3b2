"""CPU tests of the extended-precision Kalman reference (tests/kalman_ref.py) that the GPU sweep of the update paths compares
against: the comparator must reject subtly wrong results, the reference must agree with the C oracle, and the sweep's shape
list must reach every kernel path the launchers can pick."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import ekf_common as C
import kalman_ref as K

R, NS = 0.05, 100.0             # visualR and the default noise_scale (noiseScale = 1e4)


def _oracle_params(trail, ms):
    from oracle import ekf_oracle
    o = ekf_oracle.OracleEKF()
    p = o.default_params()
    o.close()
    return C.params_with(lambda: p, trail, ms)


def _case(trail, ms, n, kappa=1e3, seed=None):
    N = K.state_dim(trail, ms)
    l = K.visual_l(n, N)
    seed = n if seed is None else seed
    m, P = K.make_state(trail, ms, n, l, kappa, seed)
    H, f = K.make_measurement(n, l, seed)
    y = f + K.residual(P, H, R, NS, 0.5, seed)
    return m, P, H, f, y


def _ratio(ref, got, n, kappa):
    em, eP = K.errors(ref[0], ref[1], got[0], got[1])
    t = K.tau(n, kappa)
    return max(em, eP) / t


@pytest.mark.parametrize("trail,ms,n", [(6, 0, 16), (20, 0, 40), (5, 2, 24)])
def test_comparator_rejects_injected_faults(trail, ms, n):
    """Results built from the reference with one fault each must fail the comparison at tau = 8 n u kappa(S):
    one 8-CTA column block of P not downdated, R scaled by 1 + 1e-8, one residual entry off by 1e-7 |v|, one off-diagonal 8 x 8 tile
    of S transposed."""
    m, P, H, f, y = _case(trail, ms, n)
    N = len(m)
    kappa = K.kappa_S(P, H, R, NS)
    assert 1e2 <= kappa <= 1e4
    good = K.update(m, P, H, f, y, R, NS, trail)
    _, c2 = K.check(P, H, f, y, R, NS)
    t = K.tau(n, kappa)

    B = (N + 7) // 8
    Pb = good[1].copy()
    Pb[:, 3 * B:4 * B] = P[:, 3 * B:4 * B]
    v = y - f
    dv = np.zeros(n); dv[n // 2] = 1e-7 * np.linalg.norm(v)

    def tile_T(S):
        S = S.copy()
        S[0:8, 8:16] = S[0:8, 8:16].T.copy()
        S[8:16, 0:8] = S[0:8, 8:16].T
        return S

    faults = {"P block not downdated": (good[0], Pb),
              "R * (1 + 1e-8)": K.update(m, P, H, f, y, R, NS, trail, rdiag_scale=1 + 1e-8),
              "v entry + 1e-7 |v|": K.update(m, P, H, f, y, R, NS, trail, v_delta=dv),
              "S tile transposed": K.update(m, P, H, f, y, R, NS, trail, transform_S=tile_T)}
    for name, bad in faults.items():
        if bad is None:           # a transposed tile can leave S indefinite: the kernels return an error, so the fault cannot pass either
            print(f"N={N} n={n} kappa={kappa:.3g}: {name}: S no longer positive definite")
            continue
        r = _ratio(good, bad, n, kappa)
        print(f"N={N} n={n} kappa={kappa:.3g}: {name}: error / tau = {r:.3g}")
        assert r > 1.0, name
    for name, kw in (("R * (1 + 1e-8)", dict(rdiag_scale=1 + 1e-8)), ("v entry + 1e-7 |v|", dict(v_delta=dv)),
                     ("S tile transposed", dict(transform_S=tile_T))):
        bad = K.check(P, H, f, y, R, NS, **kw)[1]
        assert bad is None or K.chi2_error(c2, bad) > t, name
    # at kappa ~ 1e3 the transposed tile leaves S indefinite; on a well-conditioned S it stays positive definite and must be caught
    m3, P3, H3, f3, y3 = _case(trail, ms, n, kappa=3.0)
    k3 = K.kappa_S(P3, H3, R, NS)
    bad = K.update(m3, P3, H3, f3, y3, R, NS, trail, transform_S=tile_T)
    assert bad is not None
    r = _ratio(K.update(m3, P3, H3, f3, y3, R, NS, trail), bad, n, k3)
    print(f"N={N} n={n} kappa={k3:.3g}: S tile transposed: error / tau = {r:.3g}")
    assert r > 1.0


@pytest.mark.parametrize("trail,ms,n", [(5, 2, 1), (6, 0, 16), (5, 2, 40), (20, 0, 2), (20, 0, 26), (20, 0, 87), (20, 0, 99),
                                        (40, 0, 42)])
def test_reference_agrees_with_c_oracle(oracle_lk, trail, ms, n):
    """The C oracle (fp64 Cholesky, a different association order) is within tau of the reference in m, P and chi2, same status."""
    from oracle import ekf_oracle
    m, P, H, f, y = _case(trail, ms, n)
    kappa = K.kappa_S(P, H, R, NS)
    st, c2 = K.check(P, H, f, y, R, NS)
    ref = K.update(m, P, H, f, y, R, NS, trail)
    o = ekf_oracle.OracleEKF(_oracle_params(trail, ms))
    o.upload(m, P)
    so, co = o.visual_check(H, f, y, R)
    o.visual_update(H, f, y, R)
    got = o.download()
    o.close()
    t = K.tau(n, kappa)
    r, rc = _ratio(ref, got, n, kappa), K.chi2_error(c2, co) / t
    print(f"N={len(m)} n={n} kappa={kappa:.3g}: oracle error / tau = {r:.3g} (m, P), {rc:.3g} (chi2)")
    assert so == st == 0 and abs(float(c2) - K.chi2inv95(n)) > 1e-3 * K.chi2inv95(n)
    assert r <= 1.0 and rc <= 1.0


def test_path_predicates_match_the_documented_boundaries():
    """The restated predicates put the boundaries where the launchers' comments and the shared-memory formulas do: n = 32 / 33, N = 160:
    n N = 4095 / 4096 at n = 25 / 26, cluster / single-CTA at 86 / 87, shared / global tableau at 98 / 99; N = 300: 41 / 42 and 69 / 70."""
    p = lambda n, N: K.kernel_path(n, K.visual_l(n, N), N)
    assert p(32, 62)[1] == "one-stage" and p(33, 62)[1].startswith("two-stage")
    assert p(25, 160)[2] == "dsmem" and p(26, 160)[2] == "l2"
    assert p(86, 160)[0] == "cluster" and p(87, 160) == ("single-smem",)
    assert p(98, 160) == ("single-smem",) and p(99, 160) == ("single-global",)
    assert p(41, 300)[0] == "cluster" and p(42, 300) == ("single-smem",)
    assert p(69, 300) == ("single-smem",) and p(70, 300) == ("single-global",)
    assert p(40, 61) == ("cluster", "two-stage-l2", "dsmem", "loop")


def test_sweep_covers_every_reachable_kernel_path():
    """Every (kernel) x (S reduction) x (Z exchange) x (H / P staging) combination some dense visual shape reaches on the sweep's state
    layouts is in the sweep, and so are both sides of each boundary. The last loop guards a precondition of the two-stage S reduction
    through L2: the cluster's partial slices of S fit into the 8 N^2 doubles of the exchange buffer for every supported N."""
    shapes = K.sweep_shapes()
    got = {(K.state_dim(t, ms), K.kernel_path(n, l, K.state_dim(t, ms))) for t, ms, n, l in shapes}
    for t, ms in K.CONFIGS:
        N = K.state_dim(t, ms)
        for path in K.reachable(t, ms):
            assert (N, path) in got, (N, path)
    paths = {p for _, p in got}
    for p in [("single-smem",), ("single-global",), ("cluster", "two-stage-l2", "dsmem", "loop"), ("cluster", "two-stage-l2", "l2", "loop"),
              ("cluster", "two-stage-l2", "dsmem", "bulk"), ("cluster", "two-stage-l2-bulk", "l2", "bulk-P-loop-H")]:
        assert p in paths, p
    ns = {(K.state_dim(t, ms), n) for t, ms, n, _ in shapes}
    for need in [(160, 25), (160, 26), (160, 32), (160, 33), (160, 86), (160, 87), (160, 98), (160, 99), (300, 41), (300, 42),
                 (300, 69), (300, 70), (300, 200), (300, 300), (62, 62), (61, 61), (61, 1), (62, 2), (62, 3)]:
        assert need in ns, need
    assert any(l == K.state_dim(t, ms) and n < 10 for t, ms, n, l in shapes)
    for N in range(20, K.EK2_MAXN + 1):
        for n in range(33, N + 1, 8):
            MT = (n + 7) >> 3
            assert K.EK2_C * 64 * (MT * (MT + 1) // 2) <= 8 * N * N
