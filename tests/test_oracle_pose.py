"""CPU: the relative-pose oracle (oracle/hv_oracle_pose.c, which the device matches bit for bit) against cv2 4.13's cv2.recoverPose(E,
p1, p2, K, distanceThresh=..., mask=...), on E and the inlier mask of the essential oracle over every scene of
tests/essential_common.cases() and 40 five-point scenes (the first solution), with the inlier mask and without one, at distanceThresh
50, 5 and 1e9: the same count, identical masks (in cv2's values: the input mask's value, or 255 without one, where a point is good), and
R and t within 1e-9. Where they differ, each difference must have one of two named reasons, and the test shows it:
  tie           two candidates share the winning count; which of them is first in OpenCV's order depends on its SVD's sign conventions.
                cv2's (R, t) is then another of the oracle's candidates, with the same count and, under it, cv2's mask;
  undetermined  a point whose depth lies within rounding of 0 or of the threshold (tests/pose_ref.py decides).
The degenerate scenes, E = 0 and a rank-1 E are recorded, not gated."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import essential_common as ec  # noqa: E402

cv2 = pytest.importorskip("cv2")
DISTS = (50.0, 5.0, 1e9)


@pytest.fixture(scope="module")
def orc():
    import subprocess
    from oracle import essential_oracle, pose_oracle
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if not os.path.exists(pose_oracle.ORACLE_SO):
        subprocess.check_call(["make", "-s", "-C", root, "oracle"])
    return essential_oracle.OracleEssential(), pose_oracle.OraclePose()


def _cv(E, p1, p2, dist, mask):
    g, R, t, m = cv2.recoverPose(E, p1, p2, ec.K, distanceThresh=dist, mask=None if mask is None else mask.reshape(-1, 1).copy())[:4]
    return g, R, t.ravel(), m.ravel()


def _cv_values(good, mask):
    return np.where(good, 255 if mask is None else mask, 0).astype(np.uint8)


def _undetermined(E, p1, p2, idx):
    """the points idx that the extended-precision reference cannot decide at double precision under some candidate"""
    import mpmath as mp
    import pose_ref as pr
    q = ec.normalise(p1, p2)
    cands, kappa, _ = pr.decompose(E)
    out = []
    with mp.workdps(pr.DPS):
        for i in idx:
            vals = [pr.point_values(cands[k], q[i], mp.mpf(64 * pr.U64 * max(kappa[k], 1.0))) for k in range(4)]
            out.append(not all(pr.decide(v, d)[1] for v in vals for d in DISTS))
    return np.array(out, bool)


def _compare(op, name, E, p1, p2, mask, dist, record):
    good, R, t, mo, fl, _ = op.recover_pose(E, p1, p2, ec.FX, ec.FY, ec.CX, ec.CY, dist, mask, details=True)
    gc, Rc, tc, mc = _cv(E, p1, p2, dist, mask)
    if good == gc and np.array_equal(_cv_values(mo > 0, mask), mc) and np.abs(R - Rc).max() < 1e-9 and np.abs(t - tc).max() < 1e-9:
        return
    what = f"{name} dist {dist:g} mask {mask is not None}"
    use = np.ones(len(p1), bool) if mask is None else mask > 0
    cnt = (fl.astype(bool) & use[:, None]).sum(0)
    R1, R2, tt = op.decompose(E)
    cands = [(R1, tt), (R2, tt), (R1, -tt), (R2, -tt)]
    k = [j for j, (Rj, tj) in enumerate(cands) if np.abs(Rj - Rc).max() < 1e-9 and np.abs(tj - tc).max() < 1e-9]
    assert len(k) == 1, f"{what}: cv2's (R, t) is none of the oracle's candidates"
    k = k[0]
    if cnt[k] == good == gc and np.array_equal(_cv_values(fl[:, k] > 0, mask), mc):
        record["tie"].append(what)
        return
    # otherwise the same candidate, and every point where the masks differ is undetermined
    ow = [j for j, (Rj, tj) in enumerate(cands) if np.array_equal(Rj, R) and np.array_equal(tj, t)]
    assert ow == [k], f"{what}: cv2 picks candidate {k} with {gc}, the oracle {ow} with {good}"
    diff = np.flatnonzero(_cv_values(fl[:, k] > 0, mask) != mc)
    und = _undetermined(E, p1, p2, diff)
    assert und.all(), f"{what}: points {diff[~und]} differ and are determined"
    record["undetermined"].append(f"{what}: points {diff.tolist()}")


def test_oracle_matches_cv2(orc):
    oe, op = orc
    record = {"tie": [], "undetermined": []}
    runs = 0
    for case in ec.cases():
        p1, p2 = ec.case_points(case)
        E, mask = oe.find_essential_cv(p1, p2, ec.FX, ec.FY, ec.CX, ec.CY, *case[6:9])
        if not len(E):
            continue
        for dist in DISTS:
            for mk in (mask, None):
                _compare(op, case[0], E[0], p1, p2, mk, dist, record)
                runs += 1
    rng = np.random.default_rng(43)
    for k in range(40):
        p1, p2 = ec.scene(rng, 5, 0.0, 0.5, "side" if k % 2 else "forward")
        E, mask = oe.find_essential_cv(p1, p2, ec.FX, ec.FY, ec.CX, ec.CY)
        assert len(E) >= 1
        for dist in DISTS:
            _compare(op, f"five-{k} ({len(E)} solutions)", E[0], p1, p2, mask, dist, record)
            runs += 1
    for why, items in record.items():
        print(f"{why}: {len(items)} of {runs}")
        for it in items:
            print("   ", it)
    assert runs > 1200


def test_stacked_E_is_refused_as_cv2_refuses_it(orc):
    oe, _ = orc
    p1, p2 = ec.scene(np.random.default_rng(3), 5, 0.0, 0.3)
    E, _ = oe.find_essential_cv(p1, p2, ec.FX, ec.FY, ec.CX, ec.CY)
    if len(E) > 1:
        with pytest.raises(cv2.error):
            cv2.recoverPose(E.reshape(-1, 3), p1, p2, ec.K)


def test_zero_mask_and_default_threshold(orc):
    """an all-zero mask gives good 0 and (R1, t), each of its own decomposition (all four candidates tie); without a mask the good
    points hold 255; distanceThresh defaults to 50"""
    oe, op = orc
    p1, p2 = ec.scene(np.random.default_rng(8), 150, 0.1, 0.5)
    E, mask = oe.find_essential_cv(p1, p2, ec.FX, ec.FY, ec.CX, ec.CY)
    R1, _, t = op.decompose(E[0])
    g, R, tt, m = op.recover_pose(E[0], p1, p2, ec.FX, ec.FY, ec.CX, ec.CY, 50.0, np.zeros(150, np.uint8))
    gc, Rc, tc, mc = _cv(E[0], p1, p2, 50.0, np.zeros(150, np.uint8))
    assert g == gc == 0 and not m.any() and not mc.any() and np.array_equal(R, R1) and np.array_equal(tt, t)
    R1c, _, t_c = cv2.decomposeEssentialMat(E[0])
    assert np.array_equal(Rc, R1c) and np.array_equal(tc, t_c.ravel()) and np.abs(Rc - R1).max() < 1e-9
    g, R, tt, m = op.recover_pose(E[0], p1, p2, ec.FX, ec.FY, ec.CX, ec.CY)
    gc, Rc, tc, mc = cv2.recoverPose(E[0], p1, p2, ec.K)[:4]
    assert g == gc and np.array_equal(_cv_values(m > 0, None), mc.ravel()) and set(np.unique(mc)) <= {0, 255}


def test_degenerate_inputs_are_recorded(orc):
    """Zero motion, pure rotation, a plane and repeated points, and E = 0 and a rank-1 E: the oracle against cv2, printed, not gated."""
    oe, op = orc
    items = []
    for name, p1, p2 in ec.degenerate_scenes():
        E, mask = oe.find_essential_cv(p1, p2, ec.FX, ec.FY, ec.CX, ec.CY)
        if len(E):
            items.append((name, E[0], p1, p2, mask))
    p1, p2 = ec.scene(np.random.default_rng(12), 150, 0.1, 0.5)
    items.append(("E = 0", np.zeros((3, 3)), p1, p2, None))
    items.append(("rank 1", np.outer([0.3, -0.5, 0.8], [0.6, 0.64, 0.48]), p1, p2, None))
    for name, E, p1, p2, mask in items:
        for dist in DISTS:
            g, R, t, m = op.recover_pose(E, p1, p2, ec.FX, ec.FY, ec.CX, ec.CY, dist, mask)
            gc, Rc, tc, mc = _cv(E, p1, p2, dist, mask)
            same = np.array_equal(_cv_values(m > 0, mask), mc)
            print(f"{name} dist {dist:g}: good {g} / cv2 {gc}; same mask {same}; |dR| {np.abs(R - Rc).max():.3g} |dt| {np.abs(t - tc).max():.3g}")
