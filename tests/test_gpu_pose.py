"""GPU: cv::recoverPose on the device -- hv_recover_pose, hv_recover_pose_device and hv_recover_pose_batch_device -- against the plain-C
oracle (oracle/hv_oracle_pose.c), bit for bit in R, t, mask and good, on the seeded scenes of tests/essential_common.py with E and the
inlier mask from the essential oracle; batches of mixed jobs against the per-call results; refusals; and the chain ingest -> pyramid ->
LK -> hv_find_essential_device -> hv_recover_pose_device over a padded capacity with no host synchronisation between the calls."""
import ctypes
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import essential_common as ec  # noqa: E402

pytestmark = pytest.mark.gpu
NONE = np.float32(-1.0e6)          # HV_CORNER_NONE
DISTS = (50.0, 5.0, 1e9)


@pytest.fixture(scope="module")
def orc():
    import subprocess
    from oracle import essential_oracle, pose_oracle
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if not os.path.exists(pose_oracle.ORACLE_SO):
        subprocess.check_call(["make", "-C", root, "oracle"])
    return essential_oracle.OracleEssential(), pose_oracle.OraclePose()


@pytest.fixture(scope="module")
def scenes(orc):
    return _scenes(orc[0])


def _scenes(oe):
    """(name, p1, p2, E slots (10, 3, 3) column-major, nsol, inlier mask) of every case with a solution, and m = 5 (several solutions)"""
    out = []
    for case in ec.cases():
        p1, p2 = ec.case_points(case)
        E, nsol, mask, _ = oe.find_essential(p1, p2, ec.FX, ec.FY, ec.CX, ec.CY, *case[6:9])
        if nsol:
            out.append((case[0], p1, p2, E, nsol, mask))
    rng = np.random.default_rng(31)
    for k in range(20):
        p1, p2 = ec.scene(rng, 5, 0.0, 0.5, "side" if k % 2 else "forward")
        E, nsol, mask, _ = oe.find_essential(p1, p2, ec.FX, ec.FY, ec.CX, ec.CY)
        out.append((f"five-{k}", p1, p2, E, nsol, mask))
    return out


def _want(op, Ecm, nsol, p1, p2, mask, dist, k=(ec.FX, ec.FY, ec.CX, ec.CY)):
    g, R, t, m = op.recover_pose_cm(Ecm, p1, p2, *k, dist, mask, nsol)
    return g, np.ascontiguousarray(R.T).ravel(), t, m


def _host(hv, Ecm, p1, p2, mask, dist, k=(ec.FX, ec.FY, ec.CX, ec.CY)):
    from hybvio_b200.capi import _ptr, check
    n = p1.shape[0]
    E = np.ascontiguousarray(np.asarray(Ecm, np.float64).ravel()[:9])
    R, t = np.full(9, np.nan), np.full(3, np.nan)
    out = np.full(max(n, 1), 7, np.uint8)
    good = ctypes.c_int(-1)
    mi = None if mask is None else np.ascontiguousarray(mask, np.uint8)
    check(hv.lib.hv_recover_pose(hv.h, _ptr(E), _ptr(p1), _ptr(p2), _ptr(mi), n, *k, dist, _ptr(R), _ptr(t), _ptr(out), ctypes.byref(good)),
          "hv_recover_pose")
    return good.value, R, t, out[:n]


def _dev(p1, p2, Ecm, nsol, mask, cap=None):
    import torch
    n = p1.shape[0]
    cap = n if cap is None else cap
    b = {"xy1": torch.full((max(cap, 1), 2), float(NONE), dtype=torch.float32, device="cuda"),
         "xy2": torch.full((max(cap, 1), 2), float(NONE), dtype=torch.float32, device="cuda"),
         "E": torch.from_numpy(np.ascontiguousarray(np.asarray(Ecm, np.float64).ravel())).cuda(),
         "nsol": None if nsol is None else torch.tensor([nsol], dtype=torch.int32, device="cuda"),
         "R": torch.full((9,), float("nan"), dtype=torch.float64, device="cuda"),
         "t": torch.full((3,), float("nan"), dtype=torch.float64, device="cuda"),
         "out": torch.full((max(cap, 1),), 7, dtype=torch.uint8, device="cuda"),
         "good": torch.full((1,), -1, dtype=torch.int32, device="cuda"), "mask": None}
    if n:
        b["xy1"][:n] = torch.from_numpy(p1)
        b["xy2"][:n] = torch.from_numpy(p2)
    if mask is not None:
        b["mask"] = torch.zeros(max(cap, 1), dtype=torch.uint8, device="cuda")
        if n:
            b["mask"][:n] = torch.from_numpy(np.ascontiguousarray(mask, np.uint8))
    return b


def _job(b, n, k=(ec.FX, ec.FY, ec.CX, ec.CY), in_place=False):
    from hybvio_b200 import capi
    return capi.pose_job(b["E"], b["xy1"], b["xy2"], b["R"], b["t"], b["mask"] if in_place else b["out"], b["good"], *k, b["nsol"], b["mask"], n)


def _read(b, n, in_place=False):
    return (int(b["good"].item()), b["R"].cpu().numpy(), b["t"].cpu().numpy(), (b["mask"] if in_place else b["out"])[:n].cpu().numpy())


def _same(got, want, what):
    g, R, t, m = got
    gw, Rw, tw, mw = want
    assert g == gw, f"{what}: good {g} != {gw}"
    assert np.array_equal(m, mw), f"{what}: mask differs at {np.flatnonzero(m != mw)[:10]}"
    assert np.array_equal(R.view(np.uint64), Rw.view(np.uint64)), f"{what}: R differs (max {np.nanmax(np.abs(R - Rw))})"
    assert np.array_equal(t.view(np.uint64), tw.view(np.uint64)), f"{what}: t differs (max {np.nanmax(np.abs(t - tw))})"


@pytest.mark.parametrize("dist", DISTS)
def test_host_and_device_calls_match_the_oracle_bitwise(hv, orc, scenes, dist):
    import torch
    _, op = orc
    for name, p1, p2, E, nsol, mask in scenes:
        m = p1.shape[0]
        Ecm = E.reshape(-1)
        for mk in (mask, None):
            want = _want(op, Ecm, nsol, p1, p2, mk, dist)
            _same(_host(hv, Ecm, p1, p2, mk, dist), want, f"{name} host mask {mk is not None}")
            b = _dev(p1, p2, Ecm, nsol, mk)
            before = hv.launches
            hv.recover_pose_device(b["E"], b["xy1"], b["xy2"], b["R"], b["t"], b["out"], b["good"], ec.FX, ec.FY, ec.CX, ec.CY, dist,
                                   d_nsol=b["nsol"], d_mask_in=b["mask"], n=m)
            assert hv.launches == before + 1
            torch.cuda.synchronize()
            _same(_read(b, m), want, f"{name} device mask {mk is not None}")
        # in place on the inlier mask, with the count read on the device
        b = _dev(p1, p2, Ecm, nsol, mask)
        hv.recover_pose_batch_device([_job(b, m, in_place=True)], dist)
        torch.cuda.synchronize()
        _same(_read(b, m, in_place=True), _want(op, Ecm, nsol, p1, p2, mask, dist), f"{name} in place")


def test_python_wrapper_returns_cv2_values_and_shapes(hv, orc, scenes):
    _, op = orc
    name, p1, p2, E, nsol, mask = scenes[40]
    Erm = E[0].T
    for mk in (mask * 3, None):
        g, R, t, m = hv.recover_pose(Erm, p1, p2, ec.FX, ec.FY, ec.CX, ec.CY, 50.0, mk)
        gw, Rw, tw, mw = op.recover_pose(Erm, p1, p2, ec.FX, ec.FY, ec.CX, ec.CY, 50.0, mk)
        assert g == gw and np.array_equal(R, Rw) and np.array_equal(t.ravel(), tw) and t.shape == (3, 1) and m.shape == (p1.shape[0], 1)
        assert np.array_equal(m.ravel(), np.where(mw > 0, 255 if mk is None else mk, 0))
    with pytest.raises(ValueError):
        hv.recover_pose(np.zeros((6, 3)), p1, p2, ec.FX, ec.FY, ec.CX, ec.CY)


def test_small_degenerate_and_zero_count_inputs_match_the_oracle(hv, orc, scenes):
    import torch
    _, op = orc
    rng = np.random.default_rng(9)
    E0 = scenes[50][3].reshape(-1)
    for m in (0, 1, 4, 5, 6):
        p1, p2 = ec.scene(rng, m, 0.0, 0.3)
        _same(_host(hv, E0, p1, p2, None, 50.0), _want(op, E0, 1, p1, p2, None, 50.0), f"m = {m}")
    p1, p2 = ec.scene(rng, 150, 0.2, 0.5)
    u, v = np.array([0.3, -0.5, 0.8]), np.array([0.6, 0.64, 0.48])
    for what, Ecm in (("E = 0", np.zeros(9)), ("rank 1", np.outer(u, v).T.ravel())):
        _same(_host(hv, Ecm, p1, p2, None, 50.0), _want(op, Ecm, 1, p1, p2, None, 50.0), what)
    for dist in (0.0, -1.0, float("nan"), float("inf")):
        _same(_host(hv, E0, p1, p2, None, dist), _want(op, E0, 1, p1, p2, None, dist), f"dist {dist}")
    assert _host(hv, E0, p1, p2, None, float("nan"))[0] == 0
    zero = np.zeros(150, np.uint8)
    assert _host(hv, E0, p1, p2, zero, 50.0)[0] == 0
    # nsol 0: good 0, zero mask, R = t = 0
    b = _dev(p1, p2, E0, 0, None)
    hv.recover_pose_device(b["E"], b["xy1"], b["xy2"], b["R"], b["t"], b["out"], b["good"], ec.FX, ec.FY, ec.CX, ec.CY, d_nsol=b["nsol"])
    torch.cuda.synchronize()
    g, R, t, m = _read(b, 150)
    assert g == 0 and not m.any() and not R.any() and not t.any()


@pytest.mark.parametrize("njobs", [1, 2, 5, 64])
def test_batches_match_the_per_call_results(hv, orc, njobs):
    import torch
    oe, _ = orc
    rng = np.random.default_rng(100 + njobs)
    ms = [0, 4, 5, 6, 150, 600, 2000, 20, 300, 8, 4096]
    bufs, jobs, singles = [], [], []
    for j in range(njobs):
        m = ms[j % len(ms)]
        p1, p2 = ec.scene(rng, m, [0.1, 0.3, 0.5][j % 3], 0.5, "side" if j % 2 else "forward")
        k = (ec.FX * (1 + 0.01 * (j % 5)), ec.FY * (1 - 0.01 * (j % 3)), ec.CX + j % 7, ec.CY)
        E, nsol, mask, _ = oe.find_essential(p1, p2, *k, 0.99, 1.0, 200) if m >= 5 else (np.eye(3)[None].repeat(10, 0), 0, np.zeros(m, np.uint8), 0)
        nsol_arg = None if j % 4 == 3 else nsol
        mk = None if j % 3 == 2 else mask
        b, s = _dev(p1, p2, E.reshape(-1), nsol_arg, mk), _dev(p1, p2, E.reshape(-1), nsol_arg, mk)
        bufs.append((b, m))
        jobs.append(_job(b, m, k))
        before = hv.launches
        hv.recover_pose_device(s["E"], s["xy1"], s["xy2"], s["R"], s["t"], s["out"], s["good"], *k, 20.0, d_nsol=s["nsol"], d_mask_in=s["mask"],
                               n=m)
        assert hv.launches == before + 1
        singles.append((s, m))
    before = hv.launches
    hv.recover_pose_batch_device(jobs, 20.0)
    assert hv.launches == before + 1
    torch.cuda.synchronize()
    for j in range(njobs):
        _same(_read(*bufs[j]), _read(*singles[j]), f"job {j} of {njobs}")


def test_refusals_launch_nothing_and_leave_buffers_untouched(hv):
    import torch
    from hybvio_b200 import capi
    p1, p2 = ec.scene(np.random.default_rng(3), 50, 0.2, 0.5)
    E = np.eye(3).ravel() * 0.5
    b = _dev(p1, p2, E, 1, np.ones(50, np.uint8))
    big = _dev(*ec.scene(np.random.default_rng(4), 4097, 0.2, 0.5), E, 1, None)
    nan, inf = float("nan"), float("inf")
    lib = hv.lib

    def dev(n=50, fx=ec.FX, fy=ec.FY, cx=ec.CX, cy=ec.CY, bb=b, drop=()):
        p = {k: (None if k in drop or bb[k] is None else bb[k].data_ptr()) for k in ("E", "nsol", "xy1", "xy2", "mask", "R", "t", "out", "good")}
        return lib.hv_recover_pose_device(hv.h, p["E"], p["nsol"], p["xy1"], p["xy2"], p["mask"], n, fx, fy, cx, cy, 50.0, p["R"], p["t"],
                                          p["out"], p["good"])

    cases = [(-1, dict(n=-1)), (-1, dict(drop=("E",))), (-1, dict(drop=("R",))), (-1, dict(drop=("t",))), (-1, dict(drop=("good",))),
             (-1, dict(drop=("xy1",))), (-1, dict(drop=("xy2",))), (-1, dict(drop=("out",))), (-5, dict(n=4097, bb=big)),
             (-5, dict(fx=0.0)), (-5, dict(fy=nan)), (-5, dict(cx=inf)), (-5, dict(cy=-inf))]
    snap = {k: v.clone() for k, v in b.items() if v is not None}
    for rc, kw in cases:
        before = hv.launches
        assert dev(**kw) == rc, kw
        assert hv.launches == before, kw
    assert lib.hv_recover_pose_device(None, None, None, None, None, None, 0, 1.0, 1.0, 0.0, 0.0, 50.0, None, None, None, None) == -1
    # n = 0 accepts NULL points and mask
    before = hv.launches
    assert dev(n=0, drop=("xy1", "xy2", "out", "mask")) == 0 and hv.launches == before + 1
    torch.cuda.synchronize()
    b["R"].copy_(snap["R"]); b["t"].copy_(snap["t"]); b["good"].copy_(snap["good"])
    # host call: a non-finite E and the checks above
    R, t, out, good = np.full(9, 3.0), np.full(3, 3.0), np.full(50, 7, np.uint8), ctypes.c_int(-9)
    before = hv.launches
    for rc, Eh, n, fx in ((-5, np.r_[E[:8], nan], 50, ec.FX), (-5, np.r_[E[:8], inf], 50, ec.FX), (-1, E, -1, ec.FX), (-5, E, 50, 0.0),
                          (-5, E, 4097, ec.FX)):
        Eh = np.ascontiguousarray(Eh, np.float64)
        assert lib.hv_recover_pose(hv.h, Eh.ctypes.data, p1.ctypes.data, p2.ctypes.data, None, n, fx, ec.FY, ec.CX, ec.CY, 50.0, R.ctypes.data,
                                   t.ctypes.data, out.ctypes.data, ctypes.byref(good)) == rc, (rc, n, fx)
    assert (R == 3.0).all() and (t == 3.0).all() and (out == 7).all() and good.value == -9
    # batch
    ok = _job(b, 50)
    bad = _job(b, 50)
    bad.n = -3
    J = (capi.PoseJob * 65)(*([ok] * 65))
    assert lib.hv_recover_pose_batch_device(hv.h, J, 0, 50.0) == -1
    assert lib.hv_recover_pose_batch_device(hv.h, J, 65, 50.0) == -1
    assert lib.hv_recover_pose_batch_device(hv.h, None, 1, 50.0) == -1
    assert lib.hv_recover_pose_batch_device(None, J, 1, 50.0) == -1
    J2 = (capi.PoseJob * 3)(ok, ok, bad)
    assert lib.hv_recover_pose_batch_device(hv.h, J2, 3, 50.0) == -1
    huge = _job(big, 4097)
    assert lib.hv_recover_pose_batch_device(hv.h, (capi.PoseJob * 2)(ok, huge), 2, 50.0) == -5
    assert hv.launches == before
    torch.cuda.synchronize()
    for k, v in snap.items():
        assert torch.equal(b[k].view(torch.uint8), v.view(torch.uint8)), k


def test_lk_essential_pose_chain_matches_the_oracle(hv, orc):
    """ingest -> pyramid -> LK (device, padded capacity) -> hv_find_essential_device -> hv_recover_pose_device on the essential call's
    d_E, d_nsol and d_mask (refined in place), with no host synchronisation between the calls; against the oracle run on the
    compacted points."""
    import torch
    from hybvio_b200 import capi, synth
    oe, op = orc
    w, h, n, cap = 752, 480, 300, 384
    L0, _ = synth.stereo_frame(0, w, h)
    L1, _ = synth.stereo_frame(3, w, h)
    p0, p1 = hv.pyramid(w, h), hv.pyramid(w, h)
    ing = capi.Ingest(hv, w, h)
    ing.frame(L0, p0, want_gray=False)
    ing.frame(L1, p1, want_gray=False)
    pts = synth.interior_points(n, w, h, seed=11, margin=20)
    d_prev = torch.full((cap, 2), float(NONE), dtype=torch.float32, device="cuda")
    d_prev[:n] = torch.from_numpy(np.ascontiguousarray(pts, np.float32))
    d_next = torch.zeros((cap, 2), dtype=torch.float32, device="cuda")
    d_st = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    d_ts = torch.zeros(cap, dtype=torch.int32, device="cuda")
    E = torch.full((90,), float("nan"), dtype=torch.float64, device="cuda")
    nsol, inl = torch.full((1,), -1, dtype=torch.int32, device="cuda"), torch.full((1,), -1, dtype=torch.int32, device="cuda")
    mask = torch.full((cap,), 7, dtype=torch.uint8, device="cuda")
    R, t = torch.full((9,), float("nan"), dtype=torch.float64, device="cuda"), torch.full((3,), float("nan"), dtype=torch.float64, device="cuda")
    good = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    before = hv.launches
    hv.lk_track_device(p0, p1, d_prev.data_ptr(), d_next.data_ptr(), d_st.data_ptr(), d_ts.data_ptr(), cap, False)
    hv.find_essential_device(d_prev, d_next, E, nsol, mask, inl, ec.FX, ec.FY, ec.CX, ec.CY, 0.999, 1.0, 1000, d_status=d_st)
    mid = hv.launches
    hv.recover_pose_device(E, d_prev, d_next, R, t, mask, good, ec.FX, ec.FY, ec.CX, ec.CY, 50.0, d_nsol=nsol, d_mask_in=mask)
    assert hv.launches == mid + 1 and mid > before
    torch.cuda.synchronize()
    st = d_st.cpu().numpy()
    used = np.flatnonzero(st)
    a, b = d_prev.cpu().numpy()[used], d_next.cpu().numpy()[used]
    Ew, nw, mw, _ = oe.find_essential(a, b, ec.FX, ec.FY, ec.CX, ec.CY, 0.999, 1.0, 1000)
    assert nw == 1 and mw.sum() > n // 3
    gw, Rw, tw, mpw = _want(op, Ew.reshape(-1), nw, a, b, mw, 50.0)
    got = _read({"good": good, "R": R, "t": t, "out": mask}, cap)
    full = np.zeros(cap, np.uint8)
    full[used] = mpw
    _same(got, (gw, Rw, tw, full), "LK chain")
    assert gw > n // 3
    ing.close()
    p0.release()
    p1.release()
