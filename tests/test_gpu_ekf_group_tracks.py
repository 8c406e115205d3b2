"""GPU tests of hv_ekf_group_visual_tracks: the visual-update chains of a group of filters, stepped with the launches of one chain, must
leave every filter exactly where hv_ekf_visual_tracks would have left it. Every group filter has a twin (hv_ekf_clone) stepped by the
per-filter call; comparisons are exact (the float64 bits of m, P, chi2, pf, depth; statuses, counts, pose counts). pf and depth are
compared where the model ran to completion (triangulator status OK): for a track the success counter gated off on the device they are
whatever the model's output buffer held before, in the per-filter call as well."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import tri_common  # noqa: E402
import test_gpu_ekf_group as G  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(HERE)
TRAILS = (6, 20)                # N = 62 (BASELINE config 4) and N = 160 (config 2)
CHI_R, VIS_R = 0.01, 0.004
HV_ERR_INVALID, HV_ERR_UNSUPPORTED, HV_ERR_STATE = -1, -5, -6


def make_tracks(base, count, seed, stereo=True):
    """`count` tracks of mixed length (2 .. min(trail + 1, 21) poses) on the pose trail of `base`: noisy inliers, gross outliers
    (every 4th, from the second), tracks behind the cameras (every 7th, from the fourth)."""
    trail = base["trail"]
    rng = np.random.RandomState(seed)
    tracks = []
    for k in range(count):
        npose = 2 + (7 * k + seed) % min(trail, 20)
        idx = np.concatenate([[0], np.sort(rng.choice(np.arange(1, trail + 1), npose - 1, replace=False))]).astype(np.int32)
        pf = base["pf_true"] + rng.normal(0, 0.4, 3)
        ip = tri_common.project(base["m"], idx, base["T1"], base["T2"], stereo, pf)
        ip = ip + rng.normal(0, 2e-3, ip.shape)
        if k % 4 == 1:
            ip[rng.randint(len(ip))] += [0.08, -0.06]
        if k % 7 == 3:
            ip = -ip
        tracks.append((idx, ip, rng.normal(0, 0.05, ip.shape)))
    return tracks


def make_group(hv, trail, S, seed=0, mono=()):
    """S filters with their own state (mean on a pose trail, a well-conditioned P) and rig; filter i is mono if i in mono. Returns the
    group filters, their twins and the bases the tracks are made from."""
    from hybvio_b200 import capi
    A, bases = [], []
    for i in range(S):
        base = tri_common.make_track(seed + i, trail=trail, npose=min(4, trail + 1), stereo=i not in mono)
        rng = np.random.RandomState(100 + seed + i)
        N = 20 + 7 * trail
        X = rng.normal(0, 1, (N, N))
        e = capi.Ekf(hv, G._params(trail))
        e.upload(m=base["m"], P=1e-4 * (X @ X.T) / N + np.diag(np.full(N, 1e-4)))
        e.set_camera_model(base["T1"], base["T2"], use_stereo=i not in mono)
        e.set_first_sample_time(0.999)
        A.append(e)
        bases.append(base)
    return A, [e.clone() for e in A], bases


def params(max_succ=5, lookahead=0, chi_r=CHI_R, vis_r=VIS_R):
    return dict(chi_outlier_r=chi_r, visual_r=vis_r, max_successful_updates=max_succ, lookahead=lookahead)


def _bits(x):
    return np.ascontiguousarray(x, dtype=np.float64).view(np.uint64)


def assert_same_results(a, b, what):
    (ra, sa), (rb, sb) = a, b
    assert sa == sb, (what, sa, sb)
    assert len(ra) == len(rb), what
    for k, (x, y) in enumerate(zip(ra, rb)):
        assert (x["tri_status"], x["vu_status"], x["outlier_status"], x["updated"]) == \
               (y["tri_status"], y["vu_status"], y["outlier_status"], y["updated"]), (what, k, x, y)
        assert _bits([x["chi2"]]) == _bits([y["chi2"]]), (what, k)
        if x["tri_status"] == 0:
            assert np.array_equal(_bits(x["pf"]), _bits(y["pf"])) and _bits([x["depth"]]) == _bits([y["depth"]]), (what, k)


def step_both(A, B, tracks, prms):
    """Group call on A, per-filter calls on the twins B; every record, count and state compared."""
    from hybvio_b200 import capi
    got = capi.ekf_group_visual_tracks(A, tracks, prms)
    for i, (b, t, p) in enumerate(zip(B, tracks, prms)):
        exp = b.visual_tracks(t, **p) if len(t) else ([], 0)
        assert_same_results(got[i], exp, f"filter {i}")
    for i, (a, b) in enumerate(zip(A, B)):
        G.assert_same(a, b, f"filter {i}")
    return got


@pytest.mark.parametrize("lookahead", (0, 1, 3))
@pytest.mark.parametrize("S", (1, 2, 3, 8, 16))
@pytest.mark.parametrize("trail", TRAILS)
def test_group_equals_per_filter_chains(hv, trail, S, lookahead):
    """S filters, 20 candidate stereo tracks each (mixed length, outliers, tracks behind the cameras), max 5 successful updates."""
    A, B, bases = make_group(hv, trail, S, seed=10 * trail + S)
    tracks = [make_tracks(bases[i], 20, 7 * i + trail) for i in range(S)]
    got = step_both(A, B, tracks, [params(lookahead=lookahead)] * S)
    seen = set(x["outlier_status"] for r, _ in got for x in r)
    assert {0, 3}.issubset(seen), seen
    assert any(s == 5 for _, s in got)
    for e in A + B:
        e.close()


@pytest.mark.parametrize("lookahead", (0, 2))
@pytest.mark.parametrize("trail", TRAILS)
def test_heterogeneous_group(hv, trail, lookahead):
    """Different track counts (one filter without tracks), different max_successful_updates (chains that stop at different steps, one
    unlimited), a mono filter among stereo ones, a filter in the separate form (chi_outlier_r < 0: check and update as two gated
    launches), a chain with a track behind the cameras and a chi2 outlier; then a second round on the updated states."""
    S = 6
    A, B, bases = make_group(hv, trail, S, seed=3 + trail, mono=(2,))
    counts = [20, 0, 12, 7, 20, 3]
    prms = [params(5, lookahead), params(5, lookahead), params(2, lookahead), params(0, lookahead),
            params(4, lookahead, chi_r=-1.0), params(1, lookahead)]
    for rnd in range(2):
        tracks = [make_tracks(bases[i], counts[i], 31 * i + rnd, stereo=i != 2) for i in range(S)]
        got = step_both(A, B, tracks, prms)
        assert got[1] == ([], 0)
        r0 = got[0][0]
        assert any(x["tri_status"] == 2 for x in r0) and any(x["outlier_status"] == 3 for x in r0)
        assert any(x["updated"] for x in got[4][0])
    for e in A + B:
        e.close()


def test_group_member_against_the_oracle_flow(hv):
    """One filter of a group of 3 against the per-track loop driven with the oracles (oracle model + oracle EKF)."""
    import test_gpu_track_model as TM
    from hybvio_b200 import capi
    from oracle import ekf_oracle, tri_oracle
    A, _, bases = make_group(hv, 20, 3, seed=40)
    base = tri_common.make_track(7, npose=4, stereo=True)
    tracks = TM.chain_tracks(base, 14, 21)
    e = A[1]
    rng = np.random.RandomState(3)
    X = rng.normal(0, 1, (e.N, e.N))
    P0 = 1e-4 * (X @ X.T) / e.N + np.diag(np.full(e.N, 1e-4))
    e.upload(m=base["m"], P=P0)
    e.set_camera_model(base["T1"], base["T2"], use_stereo=True)
    okf = ekf_oracle.OracleEKF(e.params)
    okf.upload(m=base["m"], P=P0)
    exp, exp_succ = TM.sequential_reference_flow(tri_oracle.OracleTri(), okf, tracks, base, CHI_R, VIS_R, 5)
    got = capi.ekf_group_visual_tracks(A, [make_tracks(bases[0], 10, 1), tracks, make_tracks(bases[2], 16, 2)], [params(5)] * 3)
    res, succ = got[1]
    assert succ == exp_succ == 5
    for k, (g, x) in enumerate(zip(res, exp)):
        assert (g["tri_status"], g["vu_status"], g["outlier_status"], g["updated"]) == (x["tri_status"], x["vu_status"], x["outlier_status"], x["updated"]), (k, g, x)
    ma, Pa = e.download(); mb, Pb = okf.download()
    assert np.abs(ma - mb).max() < 1e-9 and np.abs(Pa - Pb).max() / np.abs(Pb).max() < 1e-9
    okf.close()
    for f in A:
        f.close()


def test_launch_count(hv):
    """lookahead 0: 2 launches per step of the longest chain for 1 filter and for 16 alike; one more per step with a filter in the
    separate form."""
    from hybvio_b200 import capi
    for S, sep in ((1, False), (16, False), (16, True)):
        A, _, bases = make_group(hv, 20, S, seed=50 + S)
        counts = [20 - (i % 5) for i in range(S)]
        tracks = [make_tracks(bases[i], counts[i], i) for i in range(S)]
        prms = [params(5, 0, chi_r=-1.0 if (sep and i == 3) else CHI_R) for i in range(S)]
        c0 = hv.launches
        capi.ekf_group_visual_tracks(A, tracks, prms)
        longest = max(counts)
        sep_steps = counts[3] if sep else 0
        assert hv.launches - c0 == 2 * longest + sep_steps, (S, sep, hv.launches - c0)
        for e in A:
            e.close()


_FRAMES = r"""
import os, sys
import numpy as np
sys.path.insert(0, {root!r}); sys.path.insert(0, os.path.join({root!r}, "tests"))
import test_gpu_ekf_group_tracks as T
import test_gpu_ekf_group as G
from hybvio_b200 import capi
hv = capi.Context(0)
S, trail = 8, 20
A, B, bases = T.make_group(hv, trail, S, seed=60)
for k in range(3):
    t = 1.0 + 0.05 * k
    imu = [G.frame(t + 0.001 * i, 100 * i + k, imu=10, tail=()) for i in range(S)]
    tail = [G.frame(t, 0, imu=0, tail=("sym", "aug")) for i in range(S)]
    tracks = [T.make_tracks(bases[i], 20, 13 * i + k) for i in range(S)]
    prms = [T.params(5, 0)] * S
    capi.ekf_group_run_device(A, imu)
    got = capi.ekf_group_visual_tracks(A, tracks, prms)
    capi.ekf_group_run_device(A, tail)
    for i, b in enumerate(B):
        b.run_device(imu[i], len(imu[i]))
        T.assert_same_results(got[i], b.visual_tracks(tracks[i], **prms[i]), "frame %d filter %d" % (k, i))
        b.run_device(tail[i], len(tail[i]))
    for i in range(S):
        G.assert_same(A[i], B[i], "frame %d filter %d" % (k, i))
hv.sync()
print("frames ok")
"""


@pytest.mark.parametrize("no_pdl", (False, True))
def test_multi_session_frame(no_pdl):
    """Three frames of 8 sessions at N = 160: group IMU bursts -> group visual-update chains -> group [SYMMETRIZE,] AUGMENT, against
    per-filter twins (hv_ekf_run_device / hv_ekf_visual_tracks), in latency mode and in throughput mode (HV_EKF_NO_PDL=1; read once
    per process)."""
    env = dict(os.environ)
    env.pop("HV_EKF_NO_PDL", None)
    if no_pdl:
        env["HV_EKF_NO_PDL"] = "1"
    r = subprocess.run([sys.executable, "-c", _FRAMES.format(root=ROOT)], capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0 and "frames ok" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]


def _raw(ekfs, tracks, prms, count=None, out=True):
    """The C call with raw arrays (None entries become NULL). Returns (rc, records per filter, counts)."""
    from hybvio_b200 import capi
    n = len(ekfs)
    keep, obs = [], []
    for e, t in zip(ekfs, tracks):
        if t is None or e is None:
            obs.append(None)
            continue
        o, k = capi.Ekf._pack_tracks(e, t) if len(t) else (None, None)
        keep.append(k)
        obs.append(o)
    outs = [(capi.TrackResult * max(len(t), 1))() if (out and t is not None) else None for t in tracks]
    E = (ctypes.c_void_p * n)(*[e.h if e else None for e in ekfs])
    Tr = (ctypes.POINTER(capi.TrackObs) * n)(*[ctypes.cast(o, ctypes.POINTER(capi.TrackObs)) if o is not None else None for o in obs])
    K = (ctypes.c_int * n)(*[len(t) if t is not None else 1 for t in tracks])
    P = (capi.VisualUpdateParams * n)(*[capi._visual_params(**p) for p in prms])
    O = (ctypes.POINTER(capi.TrackResult) * n)(*[ctypes.cast(o, ctypes.POINTER(capi.TrackResult)) if o is not None else None for o in outs])
    succ = (ctypes.c_int * n)()
    rc = capi.load().hv_ekf_group_visual_tracks(E, n if count is None else count, Tr, K, P, O, succ)
    return rc, [capi._track_results(o)[:len(t)] if o is not None else None for o, t in zip(outs, tracks)], list(succ)


def _snapshot(e):
    m, P = e.download()
    return _bits(m).copy(), _bits(P).copy(), e.pose_count()


def test_refusals(hv):
    """Every refusal returns its code before anything is issued: m, P and pose count of every filter and the context's launch count
    unchanged."""
    from hybvio_b200 import capi
    lib = capi.load()
    A, _, bases = make_group(hv, 20, 3, seed=70)
    tr = [make_tracks(bases[i], 6, i) for i in range(3)]
    pr = [params()] * 3
    other = capi.Ekf(hv, G._params(6))
    other.set_camera_model(bases[0]["T1"], bases[0]["T2"], use_stereo=True)
    hv2 = capi.Context(0)
    foreign = capi.Ekf(hv2, G._params(20))
    foreign.set_camera_model(bases[0]["T1"], bases[0]["T2"], use_stereo=True)
    nocam = capi.Ekf(hv, G._params(20))
    big = capi.Ekf(hv, G._params(30))                 # N = 230: an 84-row track does not fit the cluster kernel whole
    big.set_camera_model(bases[0]["T1"], bases[0]["T2"], use_stereo=True)
    long_track = [(np.arange(21, dtype=np.int32), np.zeros((42, 2)), np.zeros((42, 2)))]
    one_pose = [(np.zeros(1, np.int32), np.zeros((2, 2)), np.zeros((2, 2)))]
    beyond = [(np.array([0, 21], np.int32), np.zeros((4, 2)), np.zeros((4, 2)))]
    cases = [
        ("NULL filter", [A[0], None], [tr[0], tr[1]], HV_ERR_INVALID),
        ("NULL tracks", [A[0], A[1]], [tr[0], None], HV_ERR_INVALID),
        ("filter twice", [A[0], A[1], A[0]], tr, HV_ERR_INVALID),
        ("other context", [A[0], foreign], tr[:2], HV_ERR_INVALID),
        ("unequal state dimension", [A[0], other], tr[:2], HV_ERR_INVALID),
        ("a single pose", [A[0], A[1]], [tr[0], one_pose], HV_ERR_INVALID),
        ("pose index beyond the trail", [A[0], A[1]], [tr[0], beyond], HV_ERR_INVALID),
        ("no camera model", [A[0], nocam], tr[:2], HV_ERR_STATE),
        ("no camera model, no tracks", [A[0], nocam], [tr[0], []], HV_ERR_STATE),
        ("84 rows at N = 230", [big], [long_track], HV_ERR_UNSUPPORTED),
    ]
    everyone = A + [other, foreign, nocam, big]
    snaps = {id(e): _snapshot(e) for e in everyone}
    c0 = hv.launches
    for name, ekfs, tracks, code in cases:
        rc, _, _ = _raw(ekfs, tracks, [params()] * len(ekfs))
        assert rc == code, (name, rc, lib.hv_last_error())
        if code == HV_ERR_UNSUPPORTED:
            assert b"filter 0" in lib.hv_last_error() and b"track 0" in lib.hv_last_error()
    rc, _, _ = _raw(A[:2], tr[:2], pr[:2], out=False)
    assert rc == HV_ERR_INVALID                                             # NULL out[i]
    rc, _, _ = _raw(A[:2], tr[:2], pr[:2], count=0)
    assert rc == HV_ERR_INVALID
    assert _raw([A[0]] * 65, [tr[0]] * 65, [params()] * 65)[0] == HV_ERR_INVALID      # count > HV_EKF_GROUP_MAX
    E = (ctypes.c_void_p * 1)(A[0].h)
    K = (ctypes.c_int * 1)(-1)
    P = (capi.VisualUpdateParams * 1)(capi._visual_params(**params()))
    assert lib.hv_ekf_group_visual_tracks(E, 1, None, K, P, None, None) == HV_ERR_INVALID      # negative count / NULL arrays
    assert lib.hv_ekf_group_visual_tracks(None, 1, None, None, None, None, None) == HV_ERR_INVALID
    assert hv.launches == c0
    for e in everyone:
        s, ref = _snapshot(e), snaps[id(e)]
        assert np.array_equal(s[0], ref[0]) and np.array_equal(s[1], ref[1]) and s[2] == ref[2]
    hv2.sync()
    for e in everyone:
        e.close()


def test_numerical_failure_matches_the_per_filter_call(hv):
    """A P that is not positive definite in one filter of three: HV_ERR_STATE after every result has been written, the message names
    that filter; records, counts and states equal those of per-filter calls on twins."""
    from hybvio_b200 import capi
    lib = capi.load()
    A, B, bases = make_group(hv, 20, 3, seed=80)
    bad = -1e3 * np.eye(A[1].N)
    A[1].upload(P=bad); B[1].upload(P=bad)
    tracks = [make_tracks(bases[i], 8, 5 * i) for i in range(3)]
    rc, res, succ = _raw(A, tracks, [params()] * 3)
    assert rc == HV_ERR_STATE and b"filter 1" in lib.hv_last_error(), (rc, lib.hv_last_error())
    for i in range(3):
        t = tracks[i]
        obs, keep = B[i]._pack_tracks(t)
        out = (capi.TrackResult * len(t))()
        s = ctypes.c_int(0)
        prm = capi._visual_params(**params())
        rci = lib.hv_ekf_visual_tracks(B[i].h, obs, len(t), ctypes.byref(prm), out, ctypes.byref(s))
        assert rci == (HV_ERR_STATE if i == 1 else 0), (i, rci)
        assert_same_results((res[i], succ[i]), (capi._track_results(out), s.value), f"filter {i}")
        G.assert_same(A[i], B[i], f"filter {i}")
    for e in A + B:
        e.close()
