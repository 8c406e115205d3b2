"""GPU: the device-gated visual-update chain (hv_ekf_visual_tracks) on state sizes where long tracks no longer fit the cluster kernel
whole and run in its row-chunked form -- trail 20 + 14 / 47 / 80 hybrid-map points (N = 202 / 301 / 400) and trail 30 (N = 230) --
against the per-track loop through the C oracles (the gates of test_gpu_track_model.test_device_gated_chain_equals_the_per_track_loop)
and against the extended-precision Kalman reference (tests/kalman_ref.py); and the up-front refusal above the size bound."""
import ctypes
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import kalman_ref as K  # noqa: E402
import tri_common  # noqa: E402
import visual_update_ref as V  # noqa: E402
from test_gpu_track_model import sequential_reference_flow  # noqa: E402

pytestmark = pytest.mark.gpu
CONFIGS = [(20, 14), (30, 0), (20, 47), (20, 80)]           # N = 202, 230, 301, 400
NPOSE = [21, 2, 14, 21, 9, 17, 5, 21, 12, 19, 3, 21, 16, 7]


def _ekf(hv, trail, ms):
    from hybvio_b200 import capi
    p = capi.EkfParams()
    capi.load().hv_ekf_default_params(ctypes.byref(p))
    p.camera_trail_length = trail
    p.hybrid_map_size = ms
    return capi.Ekf(hv, p)


def _start(trail, ms, seed):
    """A stereo rig and pose trail (tri_common), random map points, a well-conditioned prior."""
    base = tri_common.make_track(seed, trail=trail, npose=4, stereo=True)
    rng = np.random.RandomState(seed)
    m = np.concatenate([base["m"], rng.normal(0, 1.0, 3 * ms)])
    N = len(m)
    A = rng.normal(0, 1, (N, N))
    P = 1e-4 * (A @ A.T) / N + np.diag(np.full(N, 1e-4))
    return base, m, P


def _tracks(base, seed, spoil=True):
    """Stereo tracks of 2..21 poses (21: 84 rows), every 4th with a gross outlier, every 7th behind the cameras."""
    rng = np.random.RandomState(seed)
    top = min(base["trail"], 20)
    out = []
    for k, npose in enumerate(NPOSE):
        idx = np.concatenate([[0], np.sort(rng.choice(np.arange(1, top + 1), npose - 1, replace=False))]).astype(np.int32)
        pf = base["pf_true"] + rng.normal(0, 0.4, 3)
        ip = tri_common.project(base["m"], idx, base["T1"], base["T2"], True, pf) + rng.normal(0, 2e-3, (2 * npose, 2))
        if spoil and k % 4 == 1:
            ip[rng.randint(len(ip))] += [0.08, -0.06]
        if spoil and k % 7 == 3:
            ip = -ip
        out.append((idx, ip, rng.normal(0, 0.05, ip.shape)))
    return out


def _chunked(track, N):
    idx = track[0]
    n, l = 4 * len(idx), max(10 if x == 0 else 20 + 7 * x for x in idx)
    return not K.cluster_fits(n, l, N)


def _run_chain(hv, trail, ms, lookahead, chi_r, spoil):
    from oracle import ekf_oracle
    base, m0, P0 = _start(trail, ms, 7)
    base = dict(base, m=m0)
    tracks = _tracks(base, 21, spoil)
    e = _ekf(hv, trail, ms)
    okf = ekf_oracle.OracleEKF(e.params)
    e.upload(m=m0, P=P0); okf.upload(m=m0, P=P0)
    e.set_camera_model(base["T1"], base["T2"], use_stereo=True)
    vis_r, max_succ = 0.004, 6
    exp, exp_succ = sequential_reference_flow(tri_oracle(), okf, tracks, base, chi_r, vis_r, max_succ)
    launches = hv.launches
    got, succ = e.visual_tracks(tracks, chi_r, vis_r, max_successful_updates=max_succ, lookahead=lookahead)
    issued = sum(1 for g in got if g["tri_status"] != -1)
    if lookahead == 0:
        assert hv.launches - launches == (2 if chi_r >= 0 else 3) * len(tracks)      # model + fused kernel (+ the update kernel)
    assert succ == exp_succ == max_succ and issued < len(tracks)
    assert any(x["updated"] and _chunked(t, e.N) for x, t in zip(exp, tracks))     # row-chunked updates were applied
    if spoil:
        assert any(x["outlier_status"] == 3 for x in exp) and any(x["tri_status"] == 2 for x in exp)
    for k, (g, x) in enumerate(zip(got, exp)):
        assert (g["tri_status"], g["vu_status"], g["outlier_status"], g["updated"]) == (x["tri_status"], x["vu_status"], x["outlier_status"], x["updated"]), (k, g, x)
        if x["tri_status"] == 0:
            assert np.abs(g["pf"] - x["pf"]).max() < 1e-9 * max(1.0, np.abs(x["pf"]).max())
        if "chi2" in x:
            assert abs(g["chi2"] - x["chi2"]) < 1e-8 * max(1.0, abs(x["chi2"])), (k, g["chi2"], x["chi2"])
    ma, Pa = e.download(); mb, Pb = okf.download()
    em, eP = np.abs(ma - mb).max(), np.abs(Pa - Pb).max() / np.abs(Pb).max()
    print(f"N={e.N} lookahead={lookahead} chi_r={chi_r}: {succ} updates, max|dm| {em:.2e}, max|dP|/max|P| {eP:.2e}")
    assert em < 1e-9 and eP < 1e-9
    e.close(); okf.close()


_TRI = []


def tri_oracle():
    if not _TRI:
        from oracle import tri_oracle as T
        _TRI.append(T.OracleTri())
    return _TRI[0]


@pytest.mark.parametrize("lookahead", [0, 3])
@pytest.mark.parametrize("trail,ms", CONFIGS, ids=[f"N{K.state_dim(t, s)}" for t, s in CONFIGS])
def test_chain_with_row_chunked_tracks_equals_the_per_track_loop(hv, trail, ms, lookahead):
    """Fused check (chi_outlier_r) + update (visual_r) per track, 84-row tracks chunked, capped by max_successful_updates."""
    _run_chain(hv, trail, ms, lookahead, 0.01, True)


def test_chain_with_separate_update_kernels(hv):
    """chi_outlier_r < 0 (no chi2 test): the check and the update of a track are separate gated kernels, both chunked."""
    _run_chain(hv, 20, 47, 0, -1.0, False)


@pytest.mark.parametrize("trail,ms", CONFIGS, ids=[f"N{K.state_dim(t, s)}" for t, s in CONFIGS])
def test_chunked_update_matches_extended_precision_reference(hv, trail, ms):
    """One 84-row track through the chain (row-chunked at these sizes): chi2, m and P against the long-double reference, within
    tau = 8 n u kappa(S)."""
    base, m0, P0 = _start(trail, ms, 11)
    base = dict(base, m=m0)
    track = _tracks(base, 5, spoil=False)[0]
    e = _ekf(hv, trail, ms)
    assert _chunked(track, e.N)
    e.upload(m=m0, P=P0)
    e.set_camera_model(base["T1"], base["T2"], use_stereo=True)
    model = e.track_models([track])[0]
    assert model["tri_status"] == 0 and model["vu_status"] == 0 and model["rows"] == 84
    H, f, y = model["H"], model["f"], np.asarray(track[1]).ravel()
    chi_r, vis_r = 0.01, 0.004
    ns = e.params.noise_scale
    st, c2 = K.check(P0, H, f, y, chi_r, ns)
    assert st == 0
    ref = K.update(m0, P0, H, f, y, vis_r, ns, trail)
    chunks = V.chain_chunks(84, H.shape[1], e.N)
    ref_c = V.update(m0, P0, H, f, y, vis_r, ns, trail, chunks)
    got, succ = e.visual_tracks([track], chi_r, vis_r, max_successful_updates=1)
    assert succ == 1 and got[0]["updated"] and got[0]["outlier_status"] == 0
    t_chk, t_upd = K.tau(84, K.kappa_S(P0, H, chi_r, ns)), K.tau(84, K.kappa_S(P0, H, vis_r, ns))
    m1, P1 = e.download()
    em, eP = K.errors(ref[0], ref[1], m1, P1)
    rc = K.chi2_error(c2, got[0]["chi2"]) / t_chk
    rv, where = V.worst(ref_c, m1, P1, trail, ms)
    print(f"N={e.N}: error / tau = {max(em, eP) / t_upd:.3g} (m, P), {rc:.3g} (chi2); {chunks} chunks, per-entry ratio {rv:.3g} at {where}")
    assert max(em, eP) <= t_upd and rc <= 1.0
    assert rv <= 1.0, where
    e.close()


def test_chain_above_the_size_bound_is_refused_before_anything_runs(hv):
    """N = 427 (trail 20 + 89 map points): an 84-row track cannot run even in 8-row chunks (bound N <= 424): HV_ERR_UNSUPPORTED, no
    launch, the filter state bit-identical."""
    from hybvio_b200 import capi
    base, m0, P0 = _start(20, 89, 3)
    base = dict(base, m=m0)
    tracks = _tracks(base, 9, spoil=False)[:2]                  # 21 poses (refused), then 2 poses
    e = _ekf(hv, 20, 89)
    assert e.N == 427
    e.upload(m=m0, P=P0)
    e.set_camera_model(base["T1"], base["T2"], use_stereo=True)
    before = e.download()
    obs, keep = e._pack_tracks(tracks[::-1])                   # the refused track second: nothing of the first may run either
    prm = capi.VisualUpdateParams(0.01, -1.0, 0.004, 5, 0)
    out = (capi.TrackResult * len(tracks))()
    succ = ctypes.c_int(-1)
    launches = hv.launches
    rc = e.lib.hv_ekf_visual_tracks(e.h, obs, len(tracks), ctypes.byref(prm), out, ctypes.byref(succ))
    assert rc == -5                                             # HV_ERR_UNSUPPORTED
    assert hv.launches == launches
    after = e.download()
    assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])
    e.close()
