"""GPU sweep of the per-track measurement model (hv_ekf_track_models, hv_ekf_visual_tracks) against the extended-precision
reference (tests/track_model_ref.py), through the C ABI only. Statuses, rows and cols must be equal; pf, depth, dpf, H and f must lie
within the reference's per-entry tolerance, entries with sigma = 0 exact. The worst error / tolerance is printed per track."""
import ctypes
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import track_model_ref as TR  # noqa: E402

pytestmark = pytest.mark.gpu
GROUPS = TR.sweep_cases()


def _ekf(hv, trail, map_size, m):
    from hybvio_b200 import capi
    p = capi.EkfParams()
    capi.load().hv_ekf_default_params(ctypes.byref(p))
    p.camera_trail_length = trail
    p.hybrid_map_size = map_size
    e = capi.Ekf(hv, p)
    assert e.N == len(m)
    e.upload(m=m)
    return e


def _fmt(r):
    return " ".join(f"{k} {v:.2g}" for k, v in r.items())


def _run_group(hv, g, tracks):
    e = _ekf(hv, g.trail, g.map_size, g.base["m"])
    e.set_camera_model(g.base["T1"], g.base["T2"], use_stereo=g.stereo, estimate_time_shift=g.time_shift, **g.params)
    got = e.track_models([(t.idx, t.ip, t.vel) for t in tracks])
    e.close()
    return got


@pytest.mark.parametrize("gi", range(len(GROUPS)), ids=[g.name for g in GROUPS])
def test_track_models_match_extended_precision_reference(hv, gi):
    """One launch per group: every track of the group, mixed pose counts, the same state."""
    g = GROUPS[gi]
    got = _run_group(hv, g, g.tracks)
    worst = {k: 0.0 for k in TR.OUTPUTS}
    lines, bad = [], []
    for k, (t, d) in enumerate(zip(g.tracks, got)):
        ref = TR.Reference(t, seed=100 * gi + k)
        assert ref.decided, (g.name, t.label)
        ok, rat, note = TR.compare(ref, d)
        lines.append(f"  {t.label:>12} nobs {t.nobs:2d} status {ref.status}: {_fmt(rat)}")
        if not ok:
            bad.append((t.label, ref.status, (d["tri_status"], d["vu_status"]), (d["rows"], d["cols"]), rat))
        for key, v in rat.items():
            worst[key] = max(worst[key], v)
    print(f"\n{g.name}: worst error / tolerance {_fmt(worst)}\n" + "\n".join(lines))
    assert not bad, bad


def _boundary_cases():
    """Thresholds placed just above, just below and exactly at the reference's own |dJ / J|, rcond and depth of one track."""
    t = GROUPS[0].tracks[6]
    o = TR.evaluate(t)
    assert o["status"] == TR.OK
    jd, rc, dep = float(o["Jds"][-1]), float(o["rcond"]), float(o["depth"])
    out = []
    for name, key, v in (("conv", "convergence_threshold", jd), ("rcond", "rcond_threshold", rc)):
        for side, x in (("above", v * (1 + 1e-6)), ("below", v * (1 - 1e-6)), ("at", v)):
            out.append((f"{name}-{side}", {key: x}))
    for side, x in (("below", dep * (1 - 1e-9)), ("above", dep * (1 + 1e-9)), ("at", dep)):
        out.append((f"min_dist-{side}", {"min_dist": x}))
        out.append((f"max_dist-{side}", {"max_dist": x}))
    return t, out


def test_boundary_cases_built_from_the_reference(hv):
    t0, cases = _boundary_cases()
    g = GROUPS[0]
    seen, lines, bad = set(), [], []
    for name, prm in cases:
        t = TR.Track(t0.m, t0.trail, t0.stereo, t0.idx, t0.T1, t0.T2, t0.ip, t0.vel, t0.time_shift, prm, name)
        gp = TR.Group(name, g.base, g.trail, g.map_size, g.stereo, g.time_shift, prm, [t])
        d = _run_group(hv, gp, [t])[0]
        ref = TR.Reference(t, seed=7)
        ok, rat, note = TR.compare(ref, d)
        seen.add((name.split("-")[0], ref.status[0]))
        lines.append(f"  {name:>15}: device {(d['tri_status'], d['vu_status'])}, ensemble {sorted(ref.statuses)}, {note}: {_fmt(rat)}")
        if not ok:
            bad.append((name, d["tri_status"], sorted(ref.statuses), rat, note))
    print("\nboundary cases:\n" + "\n".join(lines))
    assert not bad, bad
    # both sides of every threshold were reached
    assert {("rcond", TR.OK), ("rcond", TR.BAD_COND), ("min_dist", TR.OK), ("min_dist", TR.BAD_DEPTH), ("max_dist", TR.OK),
            ("max_dist", TR.BAD_DEPTH), ("conv", TR.OK)} <= seen, seen


def test_device_gated_chain_rejecting_every_track(hv):
    """hv_ekf_visual_tracks over 2..21-pose tracks with a prior and a chi_outlier_r under which every outlier check rejects: no update
    runs, the state is bit-identical afterwards, so every model saw the same state; statuses, pf and depth against the reference.
    Covers the per-track launches with trackOffset and programmatic dependent launch."""
    g = GROUPS[0]
    tracks = [t for t in g.tracks if t.label.endswith("none")]
    assert sorted(t.npose for t in tracks) == list(range(2, TR.MAXPOSE + 1))
    e = _ekf(hv, g.trail, g.map_size, g.base["m"])
    A = np.random.RandomState(3).normal(0, 1, (e.N, e.N))
    P0 = 1e-10 * (A @ A.T) / e.N + np.diag(np.full(e.N, 1e-10))
    e.upload(m=g.base["m"], P=P0)
    e.set_camera_model(g.base["T1"], g.base["T2"], use_stereo=g.stereo, estimate_time_shift=g.time_shift)
    m0, Pa = e.download()
    got, succ = e.visual_tracks([(t.idx, t.ip, t.vel) for t in tracks], 1e-7, 0.01, max_successful_updates=5, lookahead=4)
    m1, Pb = e.download()
    e.close()
    assert succ == 0
    assert np.array_equal(m0.view(np.uint64), m1.view(np.uint64)) and np.array_equal(Pa.view(np.uint64), Pb.view(np.uint64))
    worst, lines = {"pf": 0.0, "depth": 0.0}, []
    for k, (t, d) in enumerate(zip(tracks, got)):
        ref = TR.Reference(t, seed=500 + k)
        assert ref.decided
        ok, rat, note = TR.compare(ref, d, keys=("pf", "depth"))
        assert ok, (t.label, ref.status, (d["tri_status"], d["vu_status"]), rat)
        assert not d["updated"] and (ref.status != (TR.OK, TR.VU_OK) or d["outlier_status"] != 0), (t.label, d)
        lines.append(f"  {t.label:>12}: outlier status {d['outlier_status']}, {_fmt(rat)}")
        for key, v in rat.items():
            worst[key] = max(worst[key], v)
    print(f"\ngated chain: worst error / tolerance {_fmt(worst)}\n" + "\n".join(lines))
