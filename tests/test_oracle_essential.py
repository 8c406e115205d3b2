"""CPU: the essential-matrix RANSAC oracle (oracle/hv_oracle_essential.c, which the device matches bit for bit) against cv2 4.13's
cv2.findEssentialMat(..., cv2.RANSAC, prob, threshold, maxIters):
  - the five-point solver alone (m == 5, where cv2 returns every solution) on 2000 seeded configurations;
  - the whole call on the seeded grid of tests/essential_common.py, with cv2's baseline code path and with its defaults;
  - the degenerate scenes (recorded, not gated);
  - a numpy restatement of the acceptance loop over the oracle's per-subset solutions, with one injected fault at a time;
  - the rounding margin of the iteration bound (CUDA's log and pow against glibc's) for every point count up to the limit.
Where the oracle and cv2 differ, each difference must have one of three named reasons, and the test shows it:
  threshold  a point whose error lies within rounding of the threshold;
  order      two solutions of one subset with the same inlier count: cv2 keeps the first in its Durand-Kerner root order, the oracle the
             one of smaller hidden variable; cv2's E is then one of the oracle's solutions with the winning count;
  accuracy   same mask, and on the winning subset's five points cv2's E satisfies the essential-matrix constraints at least 10 times
             worse than the oracle's (the two within 1e-4)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import essential_common as ec  # noqa: E402
import essential_ref as er  # noqa: E402

cv2 = pytest.importorskip("cv2")


@pytest.fixture(scope="module")
def orc():
    import subprocess
    from oracle import essential_oracle
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if not os.path.exists(essential_oracle.ORACLE_SO):
        subprocess.check_call(["make", "-s", "-C", root, "oracle"])
    return essential_oracle.OracleEssential()


def _cv(p1, p2, prob=0.999, thr=1.0, mi=1000):
    E, mask = cv2.findEssentialMat(p1, p2, ec.K, cv2.RANSAC, prob, thr, mi)
    if E is None:
        return np.zeros((0, 3, 3)), None
    return E.reshape(-1, 3, 3), mask.ravel()


def _dist(A, B):
    return min(np.linalg.norm(A - B), np.linalg.norm(A + B))


def _constraint_residual(E, q):
    """max over the essential-matrix constraints (epipolar on q, 2 E E^T E - tr(E E^T) E, det E) for a unit-norm E"""
    x1 = np.c_[q[:, 0], q[:, 1], np.ones(len(q))]
    x2 = np.c_[q[:, 2], q[:, 3], np.ones(len(q))]
    ep = np.abs(np.einsum("ij,jk,ik->i", x2, E, x1)).max()
    return max(ep, np.abs(2 * E @ E.T @ E - np.trace(E @ E.T) * E).max(), abs(np.linalg.det(E)))


def test_five_point_solver_matches_cv2(orc):
    """2000 general configurations: the same number of solutions and each E within 1e-9 of one of cv2's (Frobenius, up to sign), or
    the difference is cv2's accuracy (its E violates the constraints >= 10x more than the oracle's, which satisfies them to 1e-12).
    Where the counts differ, the extended-precision reference (tests/essential_ref.py) decides: the oracle's count must be its count."""
    rng = np.random.default_rng(2024)
    stats = {"exact": 0, "accuracy": 0, "count": 0}
    for k in range(2000):
        p1, p2 = ec.scene(rng, 5, 0.0, 0.5, "side" if k % 2 else "forward", rot=0.1)
        Ec, _ = _cv(p1, p2)
        Eo, _ = orc.find_essential_cv(p1, p2, ec.FX, ec.FY, ec.CX, ec.CY)
        q, _ = orc.compact(p1, p2, ec.FX, ec.FY, ec.CX, ec.CY)
        for S in Eo:
            assert _constraint_residual(S, q) < 1e-12, f"configuration {k}: an oracle solution is not an essential matrix"
        if len(Ec) != len(Eo):
            # cv2 drops a pair of real roots whose Durand-Kerner iterates keep an imaginary part above its 1e-10 cut; every cv2 solution
            # is still one of the oracle's
            stats["count"] += 1
            assert len(Eo) == er.solve5(q, determined=False)["count"], f"configuration {k}: the reference disagrees with the oracle"
            assert all(min(_dist(C, S) for S in Eo) < 1e-6 for C in Ec), f"configuration {k}"
            continue
        worst = "exact"
        for S in Eo:
            j = int(np.argmin([_dist(S, C) for C in Ec]))
            if _dist(S, Ec[j]) < 1e-9:
                continue
            rc, ro = _constraint_residual(Ec[j], q), _constraint_residual(S, q)
            assert rc >= 10 * ro and _dist(S, Ec[j]) < 1e-1, f"configuration {k}: |dE| {_dist(S, Ec[j]):.3g}, residuals cv2 {rc:.3g} oracle {ro:.3g}"
            worst = "accuracy"
        stats[worst] += 1
    print("five-point solver vs cv2:", stats)
    assert stats["exact"] >= 1500 and stats["count"] <= 4


def _replay(q, err, ns, m, t2, prob, max_iters, strict=True, le=True, as_float=True, shrink=True):
    """numpy restatement of RANSACPointSetRegistrator::run's acceptance loop over per-subset errors err (iters, 10, m) and solution
    counts ns; returns (iteration, solution, count) of the result, or None. Keyword arguments inject one fault each."""
    niters, good, best, it = max(max_iters, 1), 0, None, 0
    from oracle.essential_oracle import OracleEssential
    upd = OracleEssential().update_niters
    while it < niters:
        for r in range(ns[it]):
            e = err[it, r].astype(np.float32) if as_float else err[it, r]
            c = int(((e <= t2) if le else (e < t2)).sum())
            if (c > max(good, 4)) if strict else (c >= max(good, 4)):
                good, best = c, (it, r, c)
                if shrink:
                    niters = upd(prob, (m - c) / m, niters)
        it += 1
    return best


def _t2(thr):
    t = thr / ((ec.FX + ec.FY) / 2.0)
    return np.float32(t * t)


def _trace(orc, p1, p2, max_iters, status=None, sub=None):
    q, idx = orc.compact(p1, p2, ec.FX, ec.FY, ec.CX, ec.CY, status)
    sub = orc.subsets(len(q), max(max_iters, 1)) if sub is None else sub
    ns, S, err = orc.hypotheses(q, sub)
    return q, idx, ns, S, err


def _explain(orc, case, p1, p2, Ec, mc, Eo, mo):
    """The reason the oracle's result differs from cv2's (see the module's docstring), or None."""
    _, _, m, _, _, _, prob, thr, mi = case
    q, idx, ns, S, err = _trace(orc, p1, p2, mi)
    t2 = _t2(thr)
    best = _replay(q, err, ns, m, t2, prob, mi)
    if mc is not None and Eo.shape[0] == 1:
        E = Eo[0]
        ec_err = np.array([orc_err for orc_err in _errs(Ec[0], q)], np.float32)
        eo_err = np.array(_errs(E, q), np.float32)
        diff = np.flatnonzero(mc[idx] != mo[idx])
        if len(diff) and np.all(np.abs(eo_err[diff] / t2 - 1) < 1e-5) or len(diff) and np.all(np.abs(ec_err[diff] / t2 - 1) < 1e-5):
            return "threshold"
        if best is not None:
            it, r, c = best
            same = [S[it, k] for k in range(ns[it]) if k != r and (err[it, k].astype(np.float32) <= t2).sum() == c]
            if any(_dist(Ec[0], X) < 1e-6 for X in same):
                return "order"
        if best is not None and not len(diff) and _dist(Ec[0], E) < 1e-4:
            qs = q[orc.subsets(m, best[0] + 1)[best[0]]]        # the winning subset's five points
            if _constraint_residual(Ec[0], qs) >= 10 * _constraint_residual(E, qs):
                return "accuracy"
    return None


def _errs(E, q):
    x1, y1, x2, y2 = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    ex0 = (E[0, 0] * x1 + E[0, 1] * y1) + E[0, 2]
    ex1 = (E[1, 0] * x1 + E[1, 1] * y1) + E[1, 2]
    ex2 = (E[2, 0] * x1 + E[2, 1] * y1) + E[2, 2]
    et0 = (E[0, 0] * x2 + E[1, 0] * y2) + E[2, 0]
    et1 = (E[0, 1] * x2 + E[1, 1] * y2) + E[2, 1]
    r = (x2 * ex0 + y2 * ex1) + ex2
    return r * r / (((ex0 * ex0 + ex1 * ex1) + et0 * et0) + et1 * et1)


@pytest.mark.parametrize("optimized", [False, True])
def test_whole_call_matches_cv2(orc, optimized):
    """Every case of the grid: the mask identical to cv2's and E within 1e-8 up to sign, or one of the three named reasons."""
    prev = cv2.useOptimized()
    cv2.setUseOptimized(optimized)
    try:
        stats = {}
        for case in ec.cases():
            name, _, m, _, _, _, prob, thr, mi = case
            p1, p2 = ec.case_points(case)
            Ec, mc = _cv(p1, p2, prob, thr, mi)
            Eo, mo = orc.find_essential_cv(p1, p2, ec.FX, ec.FY, ec.CX, ec.CY, prob, thr, mi)
            assert len(Eo) == len(Ec), f"{name}: {len(Eo)} solutions, cv2 {len(Ec)}"
            if not len(Ec):
                stats["none"] = stats.get("none", 0) + 1
                continue
            if np.array_equal(mc, mo) and _dist(Ec[0], Eo[0]) < 1e-8:
                stats["exact"] = stats.get("exact", 0) + 1
                continue
            why = _explain(orc, case, p1, p2, Ec, mc, Eo, mo)
            assert why is not None, f"{name}: mask differs at {np.flatnonzero(mc != mo)[:8]}, |dE| = {_dist(Ec[0], Eo[0]):.3g}"
            stats[why] = stats.get(why, 0) + 1
        print(f"whole call vs cv2 (optimized={optimized}):", stats)
        assert stats.get("exact", 0) >= 0.6 * sum(stats.values())
    finally:
        cv2.setUseOptimized(prev)


def test_degenerate_scenes_are_recorded(orc):
    """Zero motion, pure rotation, a plane and repeated points: the oracle against cv2, printed, not gated."""
    for name, p1, p2 in ec.degenerate_scenes():
        Ec, mc = _cv(p1, p2)
        Eo, mo = orc.find_essential_cv(p1, p2, ec.FX, ec.FY, ec.CX, ec.CY)
        same_mask = mc is not None and np.array_equal(mc, mo)
        dE = _dist(Ec[0], Eo[0]) if len(Ec) and len(Eo) else float("nan")
        print(f"{name}: cv2 {0 if mc is None else int(mc.sum())} inliers, oracle {int(mo.sum())}; same mask {same_mask}; |dE| {dE:.3g}")


def test_status_selects_and_compacts_in_index_order(orc):
    rng = np.random.default_rng(77)
    p1, p2 = ec.scene(rng, 300, 0.3, 0.5)
    st = (rng.random(300) > 0.3).astype(np.uint8) * 3
    Eo, mo = orc.find_essential_cv(p1, p2, ec.FX, ec.FY, ec.CX, ec.CY, status=st)
    Ec, mc = _cv(p1[st > 0], p2[st > 0])
    Eu, mu = orc.find_essential_cv(p1[st > 0], p2[st > 0], ec.FX, ec.FY, ec.CX, ec.CY)
    assert not mo[st == 0].any()
    assert np.array_equal(mo[st > 0], mu) and np.array_equal(Eo, Eu)
    assert np.array_equal(mu, mc) and _dist(Eo[0], Ec[0]) < 1e-6


def test_sampling_replay_matches_cv2_first_subset(orc):
    """With a threshold that makes every point an inlier the loop stops after its first subset: cv2's E is one of the solutions of
    the replay's first subset."""
    rng = np.random.default_rng(8)
    for k in range(40):
        m = int(rng.integers(6, 500))
        p1 = np.c_[rng.uniform(0, ec.W, m), rng.uniform(0, ec.H, m)].astype(np.float32)
        p2 = (p1 + rng.normal(0, 15, (m, 2))).astype(np.float32)
        Ec, _ = _cv(p1, p2, 0.999, 1e6, 1000)
        q, _, ns, S, _ = _trace(orc, p1, p2, 1)
        assert min(_dist(Ec[0], S[0, r]) for r in range(ns[0])) < 1e-6, k


def _faults(orc, p1, p2, prob, thr, mi, status=None):
    """The oracle's result and the replay under each injected fault: {fault: (iteration, solution, count) or None}."""
    q, idx, ns, S, err = _trace(orc, p1, p2, mi, status)
    m, t2 = len(q), _t2(thr)
    out = {"correct": _replay(q, err, ns, m, t2, prob, mi)}
    out[">= acceptance"] = _replay(q, err, ns, m, t2, prob, mi, strict=False)
    out["< inlier test"] = _replay(q, err, ns, m, t2, prob, mi, le=False)
    out["double inlier test"] = _replay(q, err, ns, m, t2, prob, mi, as_float=False)
    t = np.float32(thr * thr)
    out["threshold not scaled"] = _replay(q, err, ns, m, t, prob, mi)
    out["niters never shrinks"] = _replay(q, err, ns, m, t2, prob, mi, shrink=False)

    def result(best, SS):
        return None if best is None else (SS[best[0], best[1]], best[2])
    res = {k: result(v, S) for k, v in out.items()}
    # wrong seed, no distinct indices, compaction out of order: other subsets or another order of the same points
    from test_oracle_essential_rng import subsets_numpy
    for name, sub, qq in (("wrong RNG seed", subsets_numpy(m, mi, seed=0x12345678), q),
                          ("indices not distinct", subsets_numpy(m, mi, distinct=False), q),
                          ("compaction out of order", orc.subsets(m, mi), q[::-1].copy())):
        ns2, S2, err2 = orc.hypotheses(qq, sub)
        res[name] = result(_replay(qq, err2, ns2, m, t2, prob, mi), S2)
    return res, q, ns, S, err


def _differs(a, b):
    if (a is None) != (b is None):
        return True
    return a is not None and (a[1] != b[1] or _dist(a[0], b[0]) > 1e-12)


def test_injected_faults_are_caught(orc):
    """The correct replay reproduces the oracle's call, and every injected fault changes the result on at least one input."""
    caught = set()
    rng = np.random.default_rng(31)
    inputs = [ec.scene(rng, m, outl, noise, motion) + (prob, thr, mi)
              for m, outl, noise, motion, prob, thr, mi in ((6, 0.0, 0.3, "side", 0.999, 2.0, 1000), (8, 0.3, 0.5, "forward", 0.99, 1.0, 3),
                                                            (150, 0.3, 0.5, "side", 0.999, 1.0, 1000), (150, 0.5, 1.0, "forward", 0.99, 0.5, 300),
                                                            (40, 0.2, 0.3, "side", 0.999, 1.0, 50))]
    for p1, p2, prob, thr, mi in inputs:
        res, q, ns, S, err = _faults(orc, p1, p2, prob, thr, mi)
        Eo, nsol, mo, inl = orc.find_essential(p1, p2, ec.FX, ec.FY, ec.CX, ec.CY, prob, thr, mi)
        assert res["correct"] is not None and nsol == 1 and res["correct"][1] == inl and _dist(res["correct"][0], Eo[0].T) == 0
        caught |= {k for k, v in res.items() if k != "correct" and _differs(v, res["correct"])}
        # a threshold that lands exactly on a point's float error (catches "<"), and one just below a point's double error whose float
        # rounds down to it (catches the double test)
        it, r, c = _replay(q, err, ns, len(q), _t2(thr), prob, mi)
        e = err[it, r]
        for want_float_below in (False, True):
            for j in np.argsort(np.abs(np.log(np.maximum(e, 1e-300) / _t2(thr))))[:50]:
                f = np.float32(e[j])
                if want_float_below and not float(f) < e[j]:
                    continue
                T = float(np.sqrt(float(f))) * ((ec.FX + ec.FY) / 2.0)
                for _ in range(64):
                    got = _t2(T)
                    if got == f:
                        break
                    T = np.nextafter(T, np.inf if got < f else -np.inf)
                if _t2(T) != f:
                    continue
                r2, _, _, _, _ = _faults(orc, p1, p2, prob, T, mi)
                caught |= {k for k, v in r2.items() if k in ("< inlier test", "double inlier test") and _differs(v, r2["correct"])}
                break
    want = {">= acceptance", "< inlier test", "double inlier test", "threshold not scaled", "niters never shrinks", "wrong RNG seed",
            "indices not distinct", "compaction out of order"}
    assert caught == want, f"not caught: {sorted(want - caught)}"


def test_iteration_bound_rounding_margin():
    """cvRound(log(1 - p) / log(1 - (1 - ep)^5)) for every m in 6..HV_ESSENTIAL_MAX_POINTS and goodCount in 5..m at the tested p: with
    pow off by 4 ulp and each log by 2 ulp (twice CUDA's documented bounds for double pow and log), the quotient never crosses a
    half-integer, so CUDA's and glibc's results cannot round to different iteration counts."""
    ms, gs = [], []
    for m in range(6, 4097):
        g = np.arange(5, m, dtype=np.int64)        # goodCount == m gives denom = 0 exactly on both
        ms.append(np.full(g.shape, m, np.int64)); gs.append(g)
    m = np.concatenate(ms).astype(np.float64)
    g = np.concatenate(gs).astype(np.float64)
    ep = (m - g) / m
    base = 1.0 - ep
    u = np.finfo(np.float64).eps
    for p in (0.99, 0.999, 0.5, 0.95, 0.9999):
        num = np.log(max(1.0 - p, np.finfo(np.float64).tiny))
        lo = hi = None
        for sp in (-4, 4):
            pw = np.power(base, 5.0) * (1 + sp * u)
            den = np.log(1.0 - pw)
            for sl in (-2, 2):
                r = (num * (1 + sl * u)) / (den * (1 - sl * u))
                lo = r if lo is None else np.minimum(lo, r)
                hi = r if hi is None else np.maximum(hi, r)
        # a quotient of HV_ESSENTIAL_MAX_ITERS + 1 or more keeps niters (-num >= niters * (-denom)) whatever its rounding
        ok = (np.floor(lo + 0.5) == np.floor(hi + 0.5)) | (lo >= 4097)
        assert ok.all(), f"p = {p}: {int((~ok).sum())} (m, goodCount) pairs within the error of a rounding boundary"
