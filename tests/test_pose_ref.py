"""CPU: the relative-pose oracle (oracle/hv_oracle_pose.c, which the device matches bit for bit) against the 50-digit reference
(tests/pose_ref.py), on E and the inlier mask of the essential oracle over the seeded scenes of tests/essential_common.py (every case
with m <= 20, every fifth with m = 150), five-point scenes (first solution), pure rotation and a plane, at distance_thresh 50, 5 and
1e9. Per scene:
  - each of the oracle's four candidates (R, t) lies within 64 u max(kappa, 1) of a distinct candidate of the reference, entrywise,
    kappa being the reference's componentwise condition number of that candidate with respect to E;
  - on every point whose decisions are determined at double precision (pose_ref's bound), the oracle's four decisions equal the
    reference's;
  - where every used point is determined, the counts are the reference's and the winner is the reference's winner, or, where
    candidates tie at the winning count, one of them."""
import os
import sys
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import essential_common as ec  # noqa: E402

pytest.importorskip("mpmath")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DISTS = (50.0, 5.0, 1e9)
U64 = 2.0 ** -52


def _scenes():
    """(name, E (3, 3) row-major, p1, p2, inlier mask)"""
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle.essential_oracle import OracleEssential
    oe = OracleEssential()
    out = []
    for case in ec.cases():
        m = case[2]
        if m > 150 or (m == 150 and case[1] % 5):
            continue
        p1, p2 = ec.case_points(case)
        E, mask = oe.find_essential_cv(p1, p2, ec.FX, ec.FY, ec.CX, ec.CY, *case[6:9])
        if len(E):
            out.append((case[0], E[0], p1, p2, mask))
    rng = np.random.default_rng(41)
    for k in range(10):
        p1, p2 = ec.scene(rng, 5, 0.0, 0.5, "side" if k % 2 else "forward")
        E, mask = oe.find_essential_cv(p1, p2, ec.FX, ec.FY, ec.CX, ec.CY)
        out.append((f"five-{k}", E[0], p1, p2, mask))
    for name, p1, p2 in ec.degenerate_scenes():
        if name.startswith(("rotation", "plane")):
            E, mask = oe.find_essential_cv(p1, p2, ec.FX, ec.FY, ec.CX, ec.CY)
            if len(E):
                out.append((name, E[0], p1, p2, mask))
    return out


def _check(scene):
    """the gates on one scene: (name, failures, undetermined used points, ties) -- run in a worker process"""
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import pose_ref as pr
    from oracle.pose_oracle import OraclePose
    name, E, p1, p2, mask = scene
    op = OraclePose()
    q = ec.normalise(p1, p2)
    ref, cands, kappa, _ = pr.recover_pose(E, q, DISTS)
    fails, undet, ties = [], 0, 0
    R1, R2, t = op.decompose(E)
    mine = [np.r_[R1.ravel(), t], np.r_[R2.ravel(), t], np.r_[R1.ravel(), -t], np.r_[R2.ravel(), -t]]
    theirs = [np.array([float(x) for x in c]) for c in cands]
    perm = []
    for k in range(4):
        d = [np.abs(mine[k] - theirs[j]).max() for j in range(4)]
        j = int(np.argmin(d))
        bound = 64 * U64 * max(kappa[j], 1.0)
        if d[j] > bound:
            fails.append(f"{name}: candidate {k} is {d[j]:.3g} from the reference's nearest (bound {bound:.3g})")
        perm.append(j)
    if sorted(perm) != [0, 1, 2, 3]:
        fails.append(f"{name}: candidates map to {perm}")
        return name, fails, undet, ties
    for dist in DISTS:
        for mk in (mask, None):
            use = np.ones(len(q), bool) if mk is None else mk > 0
            good, R, tt, mo, fl, _ = op.recover_pose(E, p1, p2, ec.FX, ec.FY, ec.CX, ec.CY, dist, mk, details=True)
            rflags, det = ref[dist]
            mine_flags = fl.astype(bool)
            # oracle candidate k is reference candidate perm[k]
            diff = np.flatnonzero(det & (mine_flags != rflags[:, perm]).any(1))
            if len(diff):
                fails.append(f"{name} dist {dist} mask {mk is not None}: determined decisions differ at points {diff[:10]}")
            undet += int((~det & use).sum())
            if (det | ~use).all():
                w, cnt, tied = pr.winner(rflags, use)
                ow = int(np.flatnonzero([(np.abs(np.r_[R.ravel(), tt] - mine[k]).max() == 0) for k in range(4)])[0])
                if not np.array_equal((mine_flags & use[:, None]).sum(0), cnt[perm]):
                    fails.append(f"{name} dist {dist}: counts {(mine_flags & use[:, None]).sum(0)} != reference {cnt[perm]}")
                if perm[ow] not in tied:
                    fails.append(f"{name} dist {dist}: winner {perm[ow]} not among the reference's {tied}")
                ties += len(tied) > 1
    return name, fails, undet, ties


def test_oracle_matches_the_extended_precision_reference():
    scenes = _scenes()
    assert len(scenes) > 80
    with ProcessPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        results = list(ex.map(_check, scenes))
    fails = [f for _, fs, _, _ in results for f in fs]
    undet = sum(u for _, _, u, _ in results)
    ties = sum(t for _, _, _, t in results)
    print(f"{len(scenes)} scenes x {len(DISTS)} thresholds x 2 masks: {undet} undetermined used points, {ties} tied winners")
    assert not fails, "\n".join(fails[:20])
