"""CPU: the solvePnPRansac oracle (oracle/hv_oracle_pnp.c, which the device matches bit for bit) against cv2 4.13's
cv2.solvePnPRansac(..., flags=SOLVEPNP_P3P) on the seeded scenes of tests/pnp_common.py.

Gated on every scene, m = 4 to 4096:
- cv2's return value and its inlier set, exactly;
- rvec and tvec within 1e-6, except where the test names the reason:
  - m == 4 is P3P only. The solvers differ (OpenCV's is not restated), so the tolerance is the pose's conditioning: 1e-5 at far depths;
  - EPnP on 4 or 5 inliers: M (2n x 12) then has a null space of 12 - 2n > 1 dimensions, and OpenCV's SVD and this one return
    different bases of it, so the result depends on that basis.
With iterationsCount=1 the mask is the first subset's model's, which replays cv::RNG(~0)'s draws and the float32 scoring. A numpy
restatement of the acceptance loop equals cv2 on every scene, and each of seven injected faults makes it differ on at least one."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import pnp_common as pc  # noqa: E402

cv2 = pytest.importorskip("cv2")
KK = (pc.FX, pc.FY, pc.CX, pc.CY)


@pytest.fixture(scope="module")
def orc():
    import subprocess
    from oracle import pnp_oracle
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if not os.path.exists(pnp_oracle.ORACLE_SO):
        subprocess.check_call(["make", "-C", root, "oracle"])
    return pnp_oracle.OraclePnp()


def _cv2(X, x, it, thr, conf):
    ok, r, t, inl = cv2.solvePnPRansac(X, x, pc.K, None, iterationsCount=it, reprojectionError=thr, confidence=conf, flags=cv2.SOLVEPNP_P3P)
    mask = np.zeros(X.shape[0], np.uint8)
    if inl is not None:
        mask[inl.ravel()] = 1
    return ok, r.ravel(), t.ravel(), mask


def test_whole_call_matches_cv2(orc):
    n = explained = 0
    for name, seed, m, outl, noise, motion, depth, thr, it, conf in pc.cases():
        X, x, _, _ = pc.scene(np.random.default_rng(seed), m, outl, noise, motion, depth)
        ok, r, t, mask, inl = orc.solve_pnp_ransac(X, x, *KK, it, thr, conf)
        cok, cr, ct, cmask = _cv2(X, x, it, thr, conf)
        assert ok == int(cok), name
        n += 1
        if not ok:
            continue
        assert np.array_equal(mask, cmask), f"{name}: inliers differ at {np.flatnonzero(mask != cmask)}"
        assert inl == int(mask.sum())
        d = max(np.abs(r - cr).max(), np.abs(t - ct).max() / max(1.0, np.abs(ct).max()))
        if m == 4:
            assert d < 1e-5, (name, d)
        elif inl <= 5:
            explained += d >= 1e-6
        else:
            assert d < 1e-6, (name, d)
    assert n == 135
    print(f"{explained} poses from 4 or 5 inliers depart from cv2's")


@pytest.mark.parametrize("m,noise", [(6, 1.0), (20, 0.5), (150, 2.0), (300, 1.0), (4096, 0.5)])
def test_epnp_matches_cv2_on_noisy_points(orc, m, noise):
    """OpenCV refines with one EPnP in double on the inliers (cv2.solvePnP(..., SOLVEPNP_EPNP) on float64 points). Its control points
    follow the sign convention of OpenCV's Jacobi SVD, which the oracle restates; with any other signs the noisy pose moves by 1e-3."""
    for seed in range(12):
        X, x, _, _ = pc.scene(np.random.default_rng(seed), m, 0.0, noise, pc.MOTIONS[seed % 3], pc.DEPTHS[seed % 2])
        r, tv = orc.epnp(X, x, *KK)
        _, cr, ct = cv2.solvePnP(X.astype(np.float64), x.astype(np.float64), pc.K, None, flags=cv2.SOLVEPNP_EPNP)
        assert np.abs(r - cr.ravel()).max() < 1e-9 and np.abs(tv - ct.ravel()).max() < 1e-9 * max(1.0, np.abs(ct).max()), seed


def _residual(R, t, X, x):
    p = (R @ X.astype(np.float64).T).T + t
    u = (pc.K @ p.T).T
    return np.abs(u[:, :2] / u[:, 2:] - x).max()


def test_p3p_matches_cv2_solvep3p(orc):
    """counts and solutions against cv2.solveP3P (OpenCV's own solver): every cv2 solution with positive depths is one of the oracle's,
    within 1e-6, or, where cv2's own solver is less accurate (up to 1e-4 at far depths), the oracle's solution reprojects the three
    points at least as well as cv2's; the oracle's are checked against the 60-digit reference in test_pnp_ref.py. The counts may differ only where cv2 returns a solution with a point behind the
    camera (dropped here) or near a double root."""
    rng = np.random.default_rng(90)
    same = 0
    for k in range(400):
        X, x, _, _ = pc.scene(rng, 3, 0.0, 0.0, pc.MOTIONS[k % 3], pc.DEPTHS[k % 2])
        n, rv, tv = cv2.solveP3P(X, x, pc.K, None, flags=cv2.SOLVEPNP_P3P)
        ours = orc.p3p(X.astype(np.float64), x, *KK)
        theirs = []
        for r, t in zip(rv, tv):
            R = cv2.Rodrigues(r)[0]
            if ((R @ X.astype(np.float64).T).T + t.ravel())[:, 2].min() > 0:
                theirs.append((R, t.ravel()))
        for R, t in theirs:
            j = min(range(len(ours)), key=lambda i: np.abs(R - ours[i][0]).max())
            Ro, to = ours[j]
            d = max(np.abs(R - Ro).max(), np.abs(t - to).max() / max(1.0, np.abs(t).max()))
            if d > 1e-6:     # cv2's own rounding: the oracle's solution reprojects the three points at least as well
                assert _residual(Ro, to, X, x) <= _residual(R, t, X, x) + 1e-9, k
        same += len(theirs) == len(ours)
    assert same >= 390, same


@pytest.mark.parametrize("seed", range(6))
def test_first_subset_mask_replays_cv2(orc, seed):
    """iterationsCount=1: the mask is the first subset's model's (RNG replay, P3P model, Rodrigues round trip, float32 scoring)"""
    rng = np.random.default_rng(300 + seed)
    for m, outl in ((20, 0.3), (150, 0.5), (600, 0.7)):
        X, x, _, _ = pc.scene(rng, m, outl, 0.5, pc.MOTIONS[seed % 3], pc.DEPTHS[seed % 2])
        ok, _, _, mask, _ = orc.solve_pnp_ransac(X, x, *KK, 1, 2.0, 0.99)
        cok, _, _, cmask = _cv2(X, x, 1, 2.0, 0.99)
        assert ok == int(cok) and (not ok or np.array_equal(mask, cmask)), (seed, m)


def _rng_subsets(m, iters, seed=0xFFFFFFFFFFFFFFFF, distinct=True):
    """cv::RNG(seed).uniform(0, m) draws of 4-point subsets, a repeated index drawn again (distinct)"""
    st, out = seed, []
    for _ in range(iters):
        d = []
        while len(d) < 4:
            st = ((st & 0xFFFFFFFF) * 4164903690 + (st >> 32)) & 0xFFFFFFFFFFFFFFFF
            v = (st & 0xFFFFFFFF) % m
            if distinct and v in d:
                continue
            d.append(v)
        out.append(d)
    return np.array(out, np.int32)


def test_subsets_are_cv_rng_draws(orc):
    for m in (5, 10, 150, 4096):
        assert np.array_equal(orc.subsets(m, 200), _rng_subsets(m, 200))


def _loop(orc, X, x, it, thr, conf, fault=None):
    """numpy restatement of the acceptance loop on the oracle's models: (ok, mask)"""
    m = X.shape[0]
    t2 = np.float32(np.float64(np.float32(thr)) ** 2)
    if fault == "double inliers":
        t2 = np.float64(np.float32(thr)) ** 2
    subs = _rng_subsets(m, 4096, 12345 if fault == "another seed" else 0xFFFFFFFFFFFFFFFF, fault != "repeated indices")
    floor = 4 if fault == "floor" else 3
    niters, good, best = max(it, 1), 0, None

    def inliers(model):
        R = orc.rodrigues(model[0])
        p = (R @ X.astype(np.float64).T).T + model[1]
        z = np.where(p[:, 2] != 0, 1.0 / p[:, 2], 1.0)
        u = (p[:, :2] * z[:, None] * [pc.FX, pc.FY] + [pc.CX, pc.CY]).astype(np.float32)
        if fault == "double inliers":
            e = ((x.astype(np.float64) - u.astype(np.float64)) ** 2).sum(1)
        else:
            dd = x - u
            e = dd[:, 0] * dd[:, 0] + dd[:, 1] * dd[:, 1]
        return e <= t2
    k = 0
    while k < niters:
        d = subs[k]
        k += 1
        mdl = orc.model4(X[d].astype(np.float64), x[d], *KK)
        if mdl is None:
            continue
        c = int(inliers(mdl).sum())
        if (c >= max(good, floor)) if fault == ">=" else (c > max(good, floor)):
            good, best = c, mdl
            niters = orc.update_niters(conf, (m - c) / m, niters)
    if best is None:
        return 0, np.zeros(m, np.uint8)
    mask = inliers(best)
    if fault == "mask from the refined pose":
        r, t = orc.epnp(X[mask], x[mask], *KK)
        mask = inliers((r, t))
    return 1, mask.astype(np.uint8)


FAULTS = (">=", "floor", "double inliers", "mask from the refined pose", "another seed", "repeated indices")


def test_acceptance_loop_restatement_and_injected_faults(orc):
    scenes = []
    for name, seed, m, outl, noise, motion, depth, thr, it, conf in pc.cases():
        if 5 <= m <= 300:
            X, x, _, _ = pc.scene(np.random.default_rng(seed), m, outl, noise, motion, depth)
            scenes.append((X, x, it, thr, conf, _cv2(X, x, it, thr, conf)))
    # thresholds on the float32 error of a point under the first model, where the float and double comparisons can part. There the
    # model's last bits decide, and the oracle's P3P is not OpenCV's, so these scenes are compared with the oracle, not cv2
    rng = np.random.default_rng(77)
    for k in range(12):
        X, x, _, _ = pc.scene(rng, 150, 0.3, 0.7)
        mdl = orc.model4(X[_rng_subsets(150, 1)[0]].astype(np.float64), x[_rng_subsets(150, 1)[0]], *KK)
        if mdl is None:
            continue
        R = orc.rodrigues(mdl[0])
        p = (R @ X.astype(np.float64).T).T + mdl[1]
        u = (p[:, :2] * (1.0 / p[:, 2:]) * [pc.FX, pc.FY] + [pc.CX, pc.CY]).astype(np.float32)
        dd = x - u
        e = dd[:, 0] * dd[:, 0] + dd[:, 1] * dd[:, 1]
        for j in np.argsort(e)[40:46]:
            thr = float(np.float32(np.sqrt(np.float64(e[j]))))
            o = orc.solve_pnp_ransac(X, x, *KK, 1, thr, 0.99)
            scenes.append((X, x, 1, thr, 0.99, (bool(o[0]), None, None, o[3])))
    for X, x, it, thr, conf, (cok, _, _, cmask) in scenes:
        ok, mask = _loop(orc, X, x, it, thr, conf)
        assert ok == int(cok) and (not ok or np.array_equal(mask, cmask))
    for fault in FAULTS:
        caught = any(_loop(orc, X, x, it, thr, conf, fault)[0] != int(c[0]) or not np.array_equal(_loop(orc, X, x, it, thr, conf, fault)[1], c[3])
                     for X, x, it, thr, conf, c in scenes)
        assert caught, fault


def test_epnp_on_float32_would_be_caught(orc):
    """OpenCV converts the inliers to double before EPnP (fact 1): the oracle's EPnP is cv2's on float64 points to 1e-12, while cv2's
    EPnP on the same points as float32 lies 1e-9 to 1e-7 away, far outside that"""
    for seed in range(3):
        X, x, _, _ = pc.scene(np.random.default_rng(seed), 150, 0.0, 1.0, "side", "far")
        _, cr, ct = cv2.solvePnP(X.astype(np.float64), x.astype(np.float64), pc.K, None, flags=cv2.SOLVEPNP_EPNP)
        _, fr, ft = cv2.solvePnP(X, x, pc.K, None, flags=cv2.SOLVEPNP_EPNP)
        r, t = orc.epnp(X, x, *KK)
        ours = max(np.abs(r - cr.ravel()).max(), np.abs(t - ct.ravel()).max())
        f32 = max(np.abs(r - fr.ravel()).max(), np.abs(t - ft.ravel()).max())
        assert ours < 1e-12 and f32 > 1e-9, (ours, f32)


def test_cv2_facts(orc):
    """facts of cv2 4.13's solvePnPRansac that the oracle restates: with four points the result is solvePnP(P3P) on them with every
    index an inlier (2, 6); n < 4 is refused, confidence 0 or 1 is refused, iterations <= 0 runs one (5); float64 inputs are converted
    to float32 first (7)"""
    rng = np.random.default_rng(4)
    X, x, _, _ = pc.scene(rng, 4, 0.0, 0.5)
    ok, r, t, inl = cv2.solvePnPRansac(X, x, pc.K, None, flags=cv2.SOLVEPNP_P3P)
    _, r1, t1 = cv2.solvePnP(X, x, pc.K, None, flags=cv2.SOLVEPNP_P3P)
    assert ok and np.array_equal(r, r1) and np.array_equal(t, t1) and np.array_equal(inl.ravel(), np.arange(4))
    o = orc.solve_pnp_ransac(X, x, *KK)
    assert o[0] == 1 and np.abs(o[1] - r.ravel()).max() < 1e-6 and o[4] == 4
    with pytest.raises(cv2.error):
        cv2.solvePnPRansac(X[:3], x[:3], pc.K, None, flags=cv2.SOLVEPNP_P3P)
    X, x, _, _ = pc.scene(rng, 150, 0.3, 0.5)
    for conf in (0.0, 1.0):
        with pytest.raises(cv2.error):
            cv2.solvePnPRansac(X, x, pc.K, None, confidence=conf, flags=cv2.SOLVEPNP_P3P)
    a = _cv2(X, x, 0, 8.0, 0.99)
    b = _cv2(X, x, 1, 8.0, 0.99)
    assert np.array_equal(a[3], b[3]) and np.array_equal(orc.solve_pnp_ransac(X, x, *KK, 0)[3], a[3])
    c = cv2.solvePnPRansac(X.astype(np.float64), x.astype(np.float64), pc.K, None, flags=cv2.SOLVEPNP_P3P)
    d = cv2.solvePnPRansac(X, x, pc.K, None, flags=cv2.SOLVEPNP_P3P)
    assert np.array_equal(c[1], d[1]) and np.array_equal(c[3], d[3])


@pytest.mark.parametrize("m", [20, 150, 600])
def test_epnp_matches_cv2_on_noise_free_points(orc, m):
    """OpenCV refines with one EPnP in double on the inliers (cv2.solvePnP(..., SOLVEPNP_EPNP) on float64 points)"""
    X, x, R, t = pc.scene(np.random.default_rng(m), m, 0.0, 0.0, "forward", "near")
    r, tv = orc.epnp(X, x, *KK)
    _, cr, ct = cv2.solvePnP(X.astype(np.float64), x.astype(np.float64), pc.K, None, flags=cv2.SOLVEPNP_EPNP)
    assert np.abs(r - cr.ravel()).max() < 1e-6 and np.abs(tv - ct.ravel()).max() < 1e-5


def test_p3p_recovers_the_true_pose(orc):
    """noise-free triples: one P3P solution is the pose the points were made with"""
    rng = np.random.default_rng(8)
    for k in range(200):
        X, x, R, t = pc.scene(rng, 3, 0.0, 0.0, pc.MOTIONS[k % 3], pc.DEPTHS[k % 2])
        sols = orc.p3p(X.astype(np.float64), x, *KK)
        assert 1 <= len(sols) <= 4
        Xc = (R @ X.astype(np.float64).T).T + t
        err = min(np.abs((Rs @ X.astype(np.float64).T).T + ts - Xc).max() for Rs, ts in sols)
        assert err < 1e-3 * Xc[:, 2].max(), (k, err)


def test_small_inputs_and_thresholds(orc):
    rng = np.random.default_rng(2)
    for m in (0, 3):
        X, x, _, _ = pc.scene(rng, m, 0.0, 0.5)
        ok, r, t, mask, inl = orc.solve_pnp_ransac(X, x, *KK)
        assert ok == 0 and inl == 0 and not r.any() and not t.any() and not mask.any()
    X, x, _, _ = pc.scene(rng, 300, 0.3, 0.5)
    assert orc.solve_pnp_ransac(X, x, *KK, 100, float("nan"), 0.99)[0] == 0
    a = orc.solve_pnp_ransac(X, x, *KK, 100, -1.0, 0.99)
    b = orc.solve_pnp_ransac(X, x, *KK, 100, 1.0, 0.99)
    assert a[0] == b[0] and np.array_equal(a[3], b[3])


def test_trigonometry_of_plus_minus_times_divide(orc):
    for th in np.linspace(0.0, np.pi, 97):
        s, c = orc.sincos(th)
        assert abs(s - np.sin(th)) < 2e-15 and abs(c - np.cos(th)) < 2e-15     # a few ulps: three angle doublings
    for y, x in ((0.0, 1.0), (1.0, 0.0), (0.3, -0.7), (2.0, 1e-3), (1e-9, -1.0)):
        assert abs(orc.atan2(y, x) - np.arctan2(y, x)) < 4e-16
    for v in (np.array([0.1, -0.2, 0.3]), np.array([0.0, 0.0, 3.1]), np.array([1e-4, 0.0, 0.0])):
        assert np.abs(orc.rodrigues(orc.rodrigues(v)) - v).max() < 1e-12
        assert np.abs(orc.rodrigues(v) - cv2.Rodrigues(v)[0]).max() < 1e-15
