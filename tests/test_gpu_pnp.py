"""GPU: cv::solvePnPRansac (SOLVEPNP_P3P) on the device -- hv_solve_pnp_ransac, hv_solve_pnp_ransac_device and
hv_solve_pnp_ransac_batch_device -- against the plain-C oracle (oracle/hv_oracle_pnp.c), bit for bit in rvec, tvec, mask, inliers and ok,
on the seeded scenes of tests/pnp_common.py and degenerate ones (coplanar, collinear, all outliers, repeated points) at thresholds
including 0, -1, NaN and inf; batches of mixed jobs against the per-call results; refusals; and the chain ingest -> pyramid -> LK ->
hv_solve_pnp_ransac_device over a padded capacity with no host synchronisation between the calls."""
import ctypes
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import pnp_common as pc  # noqa: E402

pytestmark = pytest.mark.gpu
NONE = np.float32(-1.0e6)          # HV_CORNER_NONE
KK = (pc.FX, pc.FY, pc.CX, pc.CY)


@pytest.fixture(scope="module")
def orc():
    import subprocess
    from oracle import pnp_oracle
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if not os.path.exists(pnp_oracle.ORACLE_SO):
        subprocess.check_call(["make", "-C", root, "oracle"])
    return pnp_oracle.OraclePnp()


def _host(hv, X, x, it, thr, conf, status=None, k=KK):
    from hybvio_b200.capi import _ptr, check
    n = X.shape[0]
    r, t = np.full(3, np.nan), np.full(3, np.nan)
    mask = np.full(max(n, 1), 7, np.uint8)
    inl, ok = ctypes.c_int(-1), ctypes.c_int(-1)
    st = None if status is None else np.ascontiguousarray(status, np.uint8)
    X = np.ascontiguousarray(X, np.float32)
    x = np.ascontiguousarray(x, np.float32)
    check(hv.lib.hv_solve_pnp_ransac(hv.h, _ptr(X), _ptr(x), _ptr(st), n, *k, it, thr, conf, _ptr(r), _ptr(t), _ptr(mask),
                                     ctypes.byref(inl), ctypes.byref(ok)), "hv_solve_pnp_ransac")
    return ok.value, r, t, mask[:n], inl.value


def _dev(X, x, status=None, cap=None):
    import torch
    n = X.shape[0]
    cap = n if cap is None else cap
    b = {"xyz": torch.zeros((max(cap, 1), 3), dtype=torch.float32, device="cuda"),
         "xy": torch.full((max(cap, 1), 2), float(NONE), dtype=torch.float32, device="cuda"),
         "r": torch.full((3,), float("nan"), dtype=torch.float64, device="cuda"),
         "t": torch.full((3,), float("nan"), dtype=torch.float64, device="cuda"),
         "mask": torch.full((max(cap, 1),), 7, dtype=torch.uint8, device="cuda"),
         "inl": torch.full((1,), -1, dtype=torch.int32, device="cuda"), "ok": torch.full((1,), -1, dtype=torch.int32, device="cuda"),
         "st": None}
    if n:
        b["xyz"][:n] = torch.from_numpy(np.ascontiguousarray(X, np.float32))
        b["xy"][:n] = torch.from_numpy(np.ascontiguousarray(x, np.float32))
    if status is not None:
        b["st"] = torch.zeros(max(cap, 1), dtype=torch.uint8, device="cuda")
        if n:
            b["st"][:n] = torch.from_numpy(np.ascontiguousarray(status, np.uint8))
    return b


def _job(b, n, k=KK):
    from hybvio_b200 import capi
    return capi.pnp_job(b["xyz"], b["xy"], b["r"], b["t"], b["mask"], b["inl"], b["ok"], *k, b["st"], n)


def _read(b, n):
    return int(b["ok"].item()), b["r"].cpu().numpy(), b["t"].cpu().numpy(), b["mask"][:n].cpu().numpy(), int(b["inl"].item())


def _same(got, want, what):
    ok, r, t, m, inl = got
    okw, rw, tw, mw, inlw = want
    assert ok == okw and inl == inlw, f"{what}: ok {ok}/{okw} inliers {inl}/{inlw}"
    assert np.array_equal(m, mw), f"{what}: mask differs at {np.flatnonzero(m != mw)[:10]}"
    assert np.array_equal(r.view(np.uint64), rw.view(np.uint64)), f"{what}: rvec differs (max {np.nanmax(np.abs(r - rw))})"
    assert np.array_equal(t.view(np.uint64), tw.view(np.uint64)), f"{what}: tvec differs (max {np.nanmax(np.abs(t - tw))})"


def _case(case):
    name, seed, m, outl, noise, motion, depth, thr, it, conf = case
    X, x, _, _ = pc.scene(np.random.default_rng(seed), m, outl, noise, motion, depth)
    return X, x, it, thr, conf


def test_host_and_device_calls_match_the_oracle_bitwise(hv, orc):
    import torch
    for case in pc.cases():
        X, x, it, thr, conf = _case(case)
        m = X.shape[0]
        st = (np.arange(m) % 7 != 3).astype(np.uint8) * 9 if case[1] % 3 == 0 else None
        want = orc.solve_pnp_ransac(X, x, *KK, it, thr, conf, st)
        _same(_host(hv, X, x, it, thr, conf, st), want, f"{case[0]} host")
        b = _dev(X, x, st)
        before = hv.launches
        hv.solve_pnp_ransac_device(b["xyz"], b["xy"], b["r"], b["t"], b["mask"], b["inl"], b["ok"], *KK, it, thr, conf, d_status=b["st"], n=m)
        assert hv.launches == before + 1
        torch.cuda.synchronize()
        _same(_read(b, m), want, f"{case[0]} device")
        b = _dev(X, x, st)
        hv.solve_pnp_ransac_batch_device([_job(b, m)], it, thr, conf)
        torch.cuda.synchronize()
        _same(_read(b, m), want, f"{case[0]} batch of 1")


def test_python_wrapper_returns_cv2_values_and_shapes(hv, orc):
    X, x, _, _ = pc.scene(np.random.default_rng(5), 150, 0.2, 0.5)
    ok, r, t, inl = hv.solve_pnp_ransac(X, x, *KK)
    okw, rw, tw, mw, _ = orc.solve_pnp_ransac(X, x, *KK)
    assert ok is True and okw == 1 and r.shape == (3, 1) and t.shape == (3, 1) and inl.dtype == np.int32 and inl.shape[1] == 1
    assert np.array_equal(r.ravel(), rw) and np.array_equal(t.ravel(), tw) and np.array_equal(inl.ravel(), np.flatnonzero(mw))
    ok, r, t, inl = hv.solve_pnp_ransac(X[:3], x[:3], *KK)
    assert ok is False and inl is None and not r.any() and not t.any()


def _degenerate(rng):
    """(name, X, x): coplanar, collinear, all outliers and repeated points"""
    out = []
    X, x, R, t = pc.scene(rng, 150, 0.2, 0.5)
    Xp = X.copy()
    Xp[:, 2] = 4.0                                                     # coplanar world points, projected exactly
    xc = (pc.K @ ((R @ Xp.T).T + t).T).T
    out.append(("coplanar", Xp, (xc[:, :2] / xc[:, 2:]).astype(np.float32)))
    s = rng.uniform(-2, 2, 150)
    Xl = np.c_[s, 0.5 * s, 5.0 + 0.1 * s].astype(np.float32)          # collinear
    xl = (pc.K @ ((R @ Xl.T).T + t).T).T
    out.append(("collinear", Xl, (xl[:, :2] / xl[:, 2:]).astype(np.float32)))
    out.append(("all outliers", X, np.c_[rng.uniform(0, pc.W, 150), rng.uniform(0, pc.H, 150)].astype(np.float32)))
    Xr, xr = np.repeat(X[:10], 15, 0), np.repeat(x[:10], 15, 0)      # each point 15 times
    out.append(("repeated", Xr, xr))
    out.append(("one point 150 times", np.repeat(X[:1], 150, 0), np.repeat(x[:1], 150, 0)))
    return out


def test_degenerate_scenes_and_thresholds_match_the_oracle(hv, orc):
    rng = np.random.default_rng(41)
    for name, X, x in _degenerate(rng):
        for thr in (8.0, 1.0):
            _same(_host(hv, X, x, 100, thr, 0.99), orc.solve_pnp_ransac(X, x, *KK, 100, thr, 0.99), f"{name} thr {thr}")
    X, x, _, _ = pc.scene(rng, 300, 0.3, 0.5)
    for thr in (0.0, -1.0, float("nan"), float("inf"), 1e-3):
        for it in (1, 100, -5, 0):
            _same(_host(hv, X, x, it, thr, 0.99), orc.solve_pnp_ransac(X, x, *KK, it, thr, 0.99), f"thr {thr} iterations {it}")
    assert _host(hv, X, x, 100, float("nan"), 0.99)[0] == 0
    assert _host(hv, X, x, 100, -1.0, 0.99)[4] == _host(hv, X, x, 100, 1.0, 0.99)[4]
    for m in (0, 1, 3, 4, 5):
        Xm, xm, _, _ = pc.scene(rng, m, 0.0, 0.3)
        _same(_host(hv, Xm, xm, 100, 8.0, 0.99), orc.solve_pnp_ransac(Xm, xm, *KK, 100, 8.0, 0.99), f"m = {m}")


@pytest.mark.parametrize("njobs", [1, 2, 5, 64])
def test_batches_match_the_per_call_results(hv, njobs):
    import torch
    rng = np.random.default_rng(200 + njobs)
    ms = [0, 4, 5, 6, 150, 600, 3, 20, 300, 8, 4096]
    bufs, jobs, singles = [], [], []
    for j in range(njobs):
        m = ms[j % len(ms)]
        X, x, _, _ = pc.scene(rng, m, [0.1, 0.3, 0.5][j % 3], 0.5, pc.MOTIONS[j % 3], pc.DEPTHS[j % 2])
        k = (pc.FX * (1 + 0.01 * (j % 5)), pc.FY * (1 - 0.01 * (j % 3)), pc.CX + j % 7, pc.CY)
        st = (rng.random(m) > 0.1).astype(np.uint8) if j % 3 == 1 else None
        b, s = _dev(X, x, st), _dev(X, x, st)
        bufs.append((b, m))
        jobs.append(_job(b, m, k))
        before = hv.launches
        hv.solve_pnp_ransac_device(s["xyz"], s["xy"], s["r"], s["t"], s["mask"], s["inl"], s["ok"], *k, 200, 2.0, 0.999, d_status=s["st"], n=m)
        assert hv.launches == before + 1
        singles.append((s, m))
    before = hv.launches
    hv.solve_pnp_ransac_batch_device(jobs, 200, 2.0, 0.999)
    assert hv.launches == before + 1
    torch.cuda.synchronize()
    for j in range(njobs):
        _same(_read(*bufs[j]), _read(*singles[j]), f"job {j} of {njobs}")


def test_refusals_launch_nothing_and_leave_buffers_untouched(hv):
    import torch
    from hybvio_b200 import capi
    X, x, _, _ = pc.scene(np.random.default_rng(3), 50, 0.2, 0.5)
    b = _dev(X, x, np.ones(50, np.uint8))
    Xb, xb, _, _ = pc.scene(np.random.default_rng(4), 4097, 0.2, 0.5)
    big = _dev(Xb, xb)
    nan, inf = float("nan"), float("inf")
    lib = hv.lib

    def dev(n=50, fx=pc.FX, fy=pc.FY, cx=pc.CX, cy=pc.CY, it=100, conf=0.99, bb=b, drop=()):
        p = {k: (None if k in drop or bb[k] is None else bb[k].data_ptr()) for k in ("xyz", "xy", "st", "r", "t", "mask", "inl", "ok")}
        return lib.hv_solve_pnp_ransac_device(hv.h, p["xyz"], p["xy"], p["st"], n, fx, fy, cx, cy, it, 8.0, conf, p["r"], p["t"], p["mask"],
                                              p["inl"], p["ok"])

    cases = [(-1, dict(n=-1)), (-1, dict(drop=("r",))), (-1, dict(drop=("t",))), (-1, dict(drop=("inl",))), (-1, dict(drop=("ok",))),
             (-1, dict(drop=("xyz",))), (-1, dict(drop=("xy",))), (-1, dict(drop=("mask",))), (-1, dict(conf=0.0)), (-1, dict(conf=1.0)),
             (-1, dict(conf=nan)), (-1, dict(conf=-0.5)), (-5, dict(n=4097, bb=big)), (-5, dict(it=4097)),
             (-5, dict(fx=0.0)), (-5, dict(fy=nan)), (-5, dict(cx=inf)), (-5, dict(cy=-inf))]
    snap = {k: v.clone() for k, v in b.items() if v is not None}
    for rc, kw in cases:
        before = hv.launches
        assert dev(**kw) == rc, kw
        assert hv.launches == before, kw
    assert lib.hv_solve_pnp_ransac_device(None, None, None, None, 0, 1.0, 1.0, 0.0, 0.0, 100, 8.0, 0.99, None, None, None, None, None) == -1
    # n = 0 accepts NULL points and mask
    before = hv.launches
    assert dev(n=0, drop=("xyz", "xy", "mask", "st")) == 0 and hv.launches == before + 1
    torch.cuda.synchronize()
    for k in ("r", "t", "inl", "ok"):
        b[k].copy_(snap[k])
    # host call
    r, t, out, inl, ok = np.full(3, 3.0), np.full(3, 3.0), np.full(50, 7, np.uint8), ctypes.c_int(-9), ctypes.c_int(-9)
    before = hv.launches
    for rc, n, fx, conf, it in ((-1, -1, pc.FX, 0.99, 100), (-1, 50, pc.FX, 1.0, 100), (-5, 50, 0.0, 0.99, 100), (-5, 4097, pc.FX, 0.99, 100),
                                (-5, 50, pc.FX, 0.99, 5000)):
        Xh = Xb if n > 50 else X
        xh = xb if n > 50 else x
        assert lib.hv_solve_pnp_ransac(hv.h, Xh.ctypes.data, xh.ctypes.data, None, n, fx, pc.FY, pc.CX, pc.CY, it, 8.0, conf, r.ctypes.data,
                                       t.ctypes.data, out.ctypes.data, ctypes.byref(inl), ctypes.byref(ok)) == rc, (rc, n, fx, conf, it)
    assert (r == 3.0).all() and (t == 3.0).all() and (out == 7).all() and inl.value == -9 and ok.value == -9
    # batch
    good = _job(b, 50)
    bad = _job(b, 50)
    bad.n = -3
    J = (capi.PnpJob * 65)(*([good] * 65))
    assert lib.hv_solve_pnp_ransac_batch_device(hv.h, J, 0, 100, 8.0, 0.99) == -1
    assert lib.hv_solve_pnp_ransac_batch_device(hv.h, J, 65, 100, 8.0, 0.99) == -1
    assert lib.hv_solve_pnp_ransac_batch_device(hv.h, None, 1, 100, 8.0, 0.99) == -1
    assert lib.hv_solve_pnp_ransac_batch_device(None, J, 1, 100, 8.0, 0.99) == -1
    assert lib.hv_solve_pnp_ransac_batch_device(hv.h, J, 1, 100, 8.0, 1.5) == -1
    assert lib.hv_solve_pnp_ransac_batch_device(hv.h, J, 1, 4097, 8.0, 0.99) == -5
    assert lib.hv_solve_pnp_ransac_batch_device(hv.h, (capi.PnpJob * 3)(good, good, bad), 3, 100, 8.0, 0.99) == -1
    assert lib.hv_solve_pnp_ransac_batch_device(hv.h, (capi.PnpJob * 2)(good, _job(big, 4097)), 2, 100, 8.0, 0.99) == -5
    assert hv.launches == before
    torch.cuda.synchronize()
    for k, v in snap.items():
        assert torch.equal(b[k].view(torch.uint8), v.view(torch.uint8)), k


def test_lk_pnp_chain_matches_the_oracle(hv, orc):
    """ingest -> pyramid -> LK (device, padded capacity) -> hv_solve_pnp_ransac_device on LK's end points and status, with 3-D points
    back-projected from LK's input corners at seeded depths; no host synchronisation between the calls; against the oracle run on the
    compacted points."""
    import torch
    from hybvio_b200 import capi, synth
    w, h, n, cap = 752, 480, 300, 384
    L0, _ = synth.stereo_frame(0, w, h)
    L1, _ = synth.stereo_frame(3, w, h)
    p0, p1 = hv.pyramid(w, h), hv.pyramid(w, h)
    ing = capi.Ingest(hv, w, h)
    ing.frame(L0, p0, want_gray=False)
    ing.frame(L1, p1, want_gray=False)
    pts = synth.interior_points(n, w, h, seed=11, margin=20).astype(np.float32)
    Z = np.random.default_rng(12).uniform(2.0, 8.0, n)
    X = np.c_[(pts[:, 0] - pc.CX) / pc.FX * Z, (pts[:, 1] - pc.CY) / pc.FY * Z, Z].astype(np.float32)
    d_prev = torch.full((cap, 2), float(NONE), dtype=torch.float32, device="cuda")
    d_prev[:n] = torch.from_numpy(pts)
    d_xyz = torch.zeros((cap, 3), dtype=torch.float32, device="cuda")
    d_xyz[:n] = torch.from_numpy(X)
    d_next = torch.zeros((cap, 2), dtype=torch.float32, device="cuda")
    d_st = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    d_ts = torch.zeros(cap, dtype=torch.int32, device="cuda")
    r, t = torch.full((3,), float("nan"), dtype=torch.float64, device="cuda"), torch.full((3,), float("nan"), dtype=torch.float64, device="cuda")
    mask = torch.full((cap,), 7, dtype=torch.uint8, device="cuda")
    inl, ok = torch.full((1,), -1, dtype=torch.int32, device="cuda"), torch.full((1,), -1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    before = hv.launches
    hv.lk_track_device(p0, p1, d_prev.data_ptr(), d_next.data_ptr(), d_st.data_ptr(), d_ts.data_ptr(), cap, False)
    mid = hv.launches
    hv.solve_pnp_ransac_device(d_xyz, d_next, r, t, mask, inl, ok, *KK, 100, 8.0, 0.99, d_status=d_st)
    assert hv.launches == mid + 1 and mid > before
    torch.cuda.synchronize()
    st = d_st.cpu().numpy()
    used = np.flatnonzero(st)
    assert used.size > n // 2
    okw, rw, tw, mw, inlw = orc.solve_pnp_ransac(X[used], d_next.cpu().numpy()[used], *KK, 100, 8.0, 0.99)
    full = np.zeros(cap, np.uint8)
    full[used] = mw
    _same((int(ok.item()), r.cpu().numpy(), t.cpu().numpy(), mask.cpu().numpy(), int(inl.item())), (okw, rw, tw, full, inlw), "LK chain")
    assert okw == 1 and inlw >= 4
    ing.close()
    p0.release()
    p1.release()
