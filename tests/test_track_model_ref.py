"""CPU tests of the extended-precision reference of the per-track measurement model (tests/track_model_ref.py): the C oracle and the
reference's own golden vectors lie within its per-entry tolerance, six injected faults lie far outside it, and the sweep the GPU
tests run covers the pose counts, layouts, parameters and statuses the kernel has paths for."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_tri  # noqa: E402
import track_model_ref as TR  # noqa: E402
import tri_common  # noqa: E402

GROUPS = TR.sweep_cases()


@pytest.fixture(scope="module")
def orc(oracle_lk):
    from oracle import tri_oracle
    return tri_oracle.OracleTri()


@pytest.fixture(scope="module")
def refs():
    """Reference ensemble of every sweep track, [group][track]."""
    return [[TR.Reference(t, seed=100 * gi + k) for k, t in enumerate(g.tracks)] for gi, g in enumerate(GROUPS)]


def _oracle(orc, t):
    return TR.oracle_result(orc.track_model(t.m, t.trail, t.stereo, t.idx, t.T1, t.T2, t.ip, t.vel, t.time_shift))


def test_sweep_cases_are_decided(refs):
    undecided = [(g.name, t.label) for g, rs in zip(GROUPS, refs) for t, r in zip(g.tracks, rs) if not r.decided]
    assert not undecided, undecided


def test_oracle_within_tolerance_on_default_parameter_sweep(orc, refs):
    worst, count = {k: 0.0 for k in TR.OUTPUTS}, 0
    for g, rs in zip(GROUPS, refs):
        if not g.default_params:
            continue
        for t, r in zip(g.tracks, rs):
            ok, rat, note = TR.compare(r, _oracle(orc, t))
            assert ok, (g.name, t.label, r.status, rat, note)
            for k, v in rat.items():
                worst[k] = max(worst[k], v)
            count += 1
    print(f"\nC oracle vs reference, {count} default-parameter sweep tracks: worst error / tolerance",
          {k: f"{v:.3g}" for k, v in worst.items()})
    assert count >= 100


def test_golden_vectors_within_tolerance():
    """tests/golden/tri_golden.npz holds the outputs of the reference's own triangulation.cpp: statuses equal on every case, values
    within the tolerance wherever the status is OK."""
    g = np.load(os.path.join(HERE, "golden", "tri_golden.npz"))
    worst, seen = {k: 0.0 for k in TR.OUTPUTS}, set()
    for i, (seed, kw, cor) in enumerate(make_golden_tri.cases()):
        tc = make_golden_tri.build(seed, kw, cor)
        for ets in (1, 0):
            p = f"c{i}_t{ets}_"
            t = TR.Track(tc["m"], tc["trail"], tc["stereo"], tc["idx"], tc["T1"], tc["T2"], tc["ip"], tc["vel"], bool(ets))
            r = TR.Reference(t, seed=i)
            gold = dict(tri_status=int(g[p + "status"][0]), vu_status=int(g[p + "status"][1]), pf=g[p + "pf"], dpf=g[p + "dpf"],
                        depth=float(g[p + "depth"][0]), H=g[p + "H"], f=g[p + "f"])
            gold.update(rows=gold["H"].shape[0], cols=gold["H"].shape[1])
            assert r.decided, (i, ets)
            assert r.status == (gold["tri_status"], gold["vu_status"]), (i, seed, cor, ets)
            seen.add(gold["tri_status"])
            if gold["tri_status"] != TR.OK:
                continue
            ok, rat, _ = TR.compare(r, gold)
            assert ok, (i, seed, cor, ets, rat)
            for k, v in rat.items():
                worst[k] = max(worst[k], v)
    print("\ngolden vectors of the compiled reference vs reference: worst error / tolerance", {k: f"{v:.3g}" for k, v in worst.items()})
    assert seen == {TR.OK, TR.BEHIND, TR.BAD_COND, TR.NO_CONVERGENCE}


def test_known_answer_visual():
    """TEST_CASE "visual" of the reference's test/triangulation.cpp: OK and sum |pf - pf_e| < 1e-5."""
    k = tri_common.reference_visual_kat()
    t = TR.Track(k["m"], k["trail"], False, k["idx"], k["T1"], None, k["ip"], k["vel"], True)
    o = TR.evaluate(t)
    assert (o["status"], o["vu_status"]) == (TR.OK, TR.VU_OK) and o["H"].shape == (20, 83)
    assert np.abs(o["pf"].astype(np.float64) - k["pf_expected"]).sum() < 1e-5


def _applies(fault, t, r):
    if r.status != (TR.OK, TR.VU_OK):
        return False
    if fault == "H_time_column":
        return t.time_shift
    if fault == "drop_obs_32_up":
        return t.nobs > 32
    if fault == "camera1_own_quaternion_with_camera0_baseline":
        return t.stereo
    return True


def test_injected_faults_exceed_the_tolerance(refs):
    """Every fault exceeds the tolerance by at least 100x on every sweep track it applies to; the first three pass the relative
    1e-9 gate of test_gpu_track_model.py on some of them."""
    lines = []
    for fi, fault in enumerate(TR.FAULTS):
        factors, accepted = [], 0
        for g, rs in zip(GROUPS, refs):
            for t, r in zip(g.tracks, rs):
                if not _applies(fault, t, r):
                    continue
                f = TR.evaluate(t, fault=fault)
                dev = dict(tri_status=f["status"], vu_status=f["vu_status"], rows=f["rows"], cols=f["cols"],
                           **{k: np.asarray(f[k], np.float64) for k in TR.OUTPUTS})
                rat = TR.ratios(r, dev)
                factors.append(max(rat.values()))
                accepted += TR.old_gate_accepts({k: np.asarray(r.out[k], np.float64) for k in TR.OUTPUTS}, dev)
        assert factors, fault
        lines.append(f"  {fi + 1}. {fault}: {len(factors)} tracks, smallest factor {min(factors):.3g}, median {np.median(factors):.3g};"
                     f" the old gate accepts it on {accepted}")
        assert min(factors) >= 100, (fault, min(factors))
        if fi < 3:
            assert accepted > 0, fault
    print("\ninjected faults, error / tolerance:\n" + "\n".join(lines))


def test_sweep_coverage(refs):
    combos, statuses, trails, hybrid = set(), set(), set(), False
    big = False
    for g, rs in zip(GROUPS, refs):
        trails.add(g.trail)
        hybrid = hybrid or (g.map_size > 0 and len(g.base["m"]) > TR.MAXN)
        for t, r in zip(g.tracks, rs):
            combos.add((t.npose, t.stereo, t.time_shift))
            statuses.add(r.status[0])
            big = big or (t.nobs > 32 and t.rows > 64 and r.status == (TR.OK, TR.VU_OK))
    for npose in range(2, TR.MAXPOSE + 1):
        for stereo in (True, False):
            for ts in (True, False):
                assert (npose, stereo, ts) in combos, (npose, stereo, ts)
    assert big
    assert {TR.OK, TR.BEHIND, TR.BAD_COND, TR.NO_CONVERGENCE, TR.BAD_DEPTH} <= statuses, statuses
    assert {4, 8, 20, 30} <= trails and hybrid
    changed = {k for g in GROUPS for k in TR.DEFAULTS if g.params[k] != TR.DEFAULTS[k]}
    assert changed == set(TR.DEFAULTS), changed
