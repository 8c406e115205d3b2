"""GPU: cv::triangulatePoints + cv::convertPointsFromHomogeneous on the device -- hv_triangulate_points, hv_triangulate_points_device and
hv_triangulate_points_batch_device -- against the plain-C oracle (oracle/hv_oracle_triangulate.c), bit for bit in X4, xyz and used, at
n = 0 to 100 000 over padded capacities with both, one or no status arrays; used aliasing a status; batches of mixed jobs against the
per-call results; refusals; the Python wrapper against cv2; and the stereo chain ingest -> stereo + temporal LK -> triangulation ->
hv_solve_pnp_ransac_device with no host synchronisation between the calls. The layout test of hv_triangulate_job needs no GPU."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import triangulate_common as tc  # noqa: E402

gpu = pytest.mark.gpu
NONE = float(tc.NONE)


@pytest.fixture(scope="module")
def orc():
    from oracle import triangulate_oracle
    if not os.path.exists(triangulate_oracle.ORACLE_SO):
        subprocess.check_call(["make", "-C", ROOT, "oracle"])
    return triangulate_oracle.OracleTriangulate()


def _points(n, seed):
    """(P1, P2, xy1, xy2) of n points: rectified stereo, or general two-view for odd seeds"""
    return (tc.general if seed % 2 else tc.rectified)(seed, n)


def _statuses(rng, n, cap, which):
    """status, status2 over the capacity (0 in the padding) or None, as `which` asks: "both", "one" (status only), "second" (status2
    only), "none" """
    def st(p):
        s = np.zeros(cap, np.uint8)
        s[:n] = (rng.random(n) > p).astype(np.uint8) * rng.integers(1, 256, n).astype(np.uint8)
        return s
    return {"both": (st(0.2), st(0.1)), "one": (st(0.3), None), "second": (None, st(0.3)), "none": (None, None)}[which]


def _dev(a, b, s1, s2):
    import torch
    cap = a.shape[0]
    t = lambda x: None if x is None else torch.from_numpy(np.ascontiguousarray(x)).cuda()   # noqa: E731
    return {"xy1": t(a), "xy2": t(b), "s1": t(s1), "s2": t(s2),
            "X4": torch.full((4 * max(cap, 1),), float("nan"), dtype=torch.float32, device="cuda"),
            "xyz": torch.full((max(cap, 1), 3), float("nan"), dtype=torch.float32, device="cuda"),
            "used": torch.full((max(cap, 1),), 7, dtype=torch.uint8, device="cuda")}


def _read(d, n):
    return (d["X4"][:4 * n].cpu().numpy().reshape(4, n), d["xyz"][:n].cpu().numpy(), d["used"][:n].cpu().numpy())


def _host(hv, P1, P2, a, b, s1, s2):
    from hybvio_b200.capi import _ptr, check
    n = a.shape[0]
    X4, xyz, used = np.full(4 * max(n, 1), np.nan, np.float32), np.full((max(n, 1), 3), np.nan, np.float32), np.full(max(n, 1), 7, np.uint8)
    P1, P2 = np.ascontiguousarray(P1, np.float64), np.ascontiguousarray(P2, np.float64)
    check(hv.lib.hv_triangulate_points(hv.h, _ptr(P1), _ptr(P2), _ptr(a), _ptr(b), _ptr(s1), _ptr(s2), n, _ptr(X4), _ptr(xyz), _ptr(used)),
          "hv_triangulate_points")
    return X4[:4 * n].reshape(4, n), xyz[:n], used[:n]


def _same(got, want, what):
    for name, g, w in zip(("X4", "xyz", "used"), got, want):
        assert g.shape == w.shape, f"{what}: {name} shape {g.shape} / {w.shape}"
        assert np.array_equal(np.ascontiguousarray(g).view(np.uint8), np.ascontiguousarray(w).view(np.uint8)), \
            f"{what}: {name} differs at {np.argwhere(g != w)[:5].tolist()}"


@gpu
@pytest.mark.parametrize("n", [0, 1, 150, 300, 4096, 100000])
def test_host_device_and_batch_calls_match_the_oracle_bitwise(hv, orc, n):
    import torch
    from hybvio_b200 import capi
    rng = np.random.default_rng(n)
    P1, P2, a, b = _points(max(n, 1), n)
    a, b = a[:n], b[:n]
    cap = n + 37
    A, Bp = tc.padded(a, cap), tc.padded(b, cap)
    for which in ("both", "one", "second", "none"):
        s1, s2 = _statuses(rng, n, cap, which)
        want = orc.triangulate(P1, P2, A, Bp, s1, s2)
        _same(_host(hv, P1, P2, A, Bp, s1, s2), want, f"n {n} {which} host")
        d = _dev(A, Bp, s1, s2)
        before = hv.launches
        hv.triangulate_points_device(P1, P2, d["xy1"], d["xy2"], d["X4"], d["xyz"], d["used"], d["s1"], d["s2"])
        assert hv.launches == before + 1
        torch.cuda.synchronize()
        _same(_read(d, cap), want, f"n {n} {which} device")
        d = _dev(A, Bp, s1, s2)
        hv.triangulate_points_batch_device([capi.triangulate_job(P1, P2, d["xy1"], d["xy2"], d["X4"], d["xyz"], d["used"], d["s1"], d["s2"])])
        torch.cuda.synchronize()
        _same(_read(d, cap), want, f"n {n} {which} batch of 1")
        # the first n of the capacity alone, each output alone
        d = _dev(A, Bp, s1, s2)
        hv.triangulate_points_device(P1, P2, d["xy1"], d["xy2"], d["X4"], None, None, d["s1"], d["s2"], n=n)
        hv.triangulate_points_device(P1, P2, d["xy1"], d["xy2"], None, d["xyz"], None, d["s1"], d["s2"], n=n)
        torch.cuda.synchronize()
        wn = orc.triangulate(P1, P2, a, b, None if s1 is None else s1[:n], None if s2 is None else s2[:n])
        X4, xyz, used = _read(d, n)
        _same((X4, xyz), wn[:2], f"n {n} {which} one output per call")
        assert (d["used"].cpu().numpy() == 7).all() and torch.isnan(d["X4"][4 * n:]).all() and torch.isnan(d["xyz"][n:]).all()


@gpu
def test_used_may_alias_either_status(hv, orc):
    import torch
    rng = np.random.default_rng(5)
    P1, P2, a, b = _points(500, 3)
    s1, s2 = _statuses(rng, 500, 500, "both")
    want = orc.triangulate(P1, P2, a, b, s1, s2)
    for k in ("s1", "s2"):
        d = _dev(a, b, s1, s2)
        hv.triangulate_points_device(P1, P2, d["xy1"], d["xy2"], d["X4"], d["xyz"], d[k], d["s1"], d["s2"])
        torch.cuda.synchronize()
        _same(_read(d, 500)[:2] + (d[k].cpu().numpy(),), want, f"used aliasing {k}")
    u = s1.copy()
    X4, xyz = np.zeros(2000, np.float32), np.zeros((500, 3), np.float32)
    P1c, P2c = np.ascontiguousarray(P1), np.ascontiguousarray(P2)
    assert hv.lib.hv_triangulate_points(hv.h, P1c.ctypes.data, P2c.ctypes.data, a.ctypes.data, b.ctypes.data, u.ctypes.data, s2.ctypes.data,
                                        500, X4.ctypes.data, xyz.ctypes.data, u.ctypes.data) == 0
    _same((X4.reshape(4, 500), xyz, u), want, "host, used aliasing status")


@gpu
@pytest.mark.parametrize("njobs", [1, 2, 7, 64])
def test_batches_match_the_per_call_results(hv, njobs):
    import torch
    from hybvio_b200 import capi
    rng = np.random.default_rng(400 + njobs)
    ns = [0, 1, 150, 300, 4096, 37, 600, 2000]
    bufs, jobs, singles = [], [], []
    for j in range(njobs):
        n = ns[j % len(ns)]
        k = np.array([[tc.F * (1 + 0.01 * (j % 5)), 0, tc.CX + j % 7], [0, tc.F, tc.CY - j % 3], [0, 0, 1]])
        P1, P2 = tc.stereo_pair(tc.B * (1 + 0.1 * (j % 4)), k)
        if j % 3 == 2:
            P1, P2, _, _ = tc.general(j, 1)
        X = tc.cloud(rng, n)
        a, b = tc.project(P1, X, rng, 0.5), tc.project(P2, X, rng, 0.5)
        cap = n + j % 11
        A, Bp = tc.padded(a, cap), tc.padded(b, cap)
        s1, s2 = _statuses(rng, n, cap, ("both", "one", "second", "none")[j % 4])
        d, s = _dev(A, Bp, s1, s2), _dev(A, Bp, s1, s2)
        outs = [(d["X4"], d["xyz"], d["used"]), (d["X4"], None, d["used"]), (None, d["xyz"], None)][j % 3]
        jobs.append(capi.triangulate_job(P1, P2, d["xy1"], d["xy2"], *outs, d["s1"], d["s2"]))
        bufs.append((d, cap))
        so = [(s["X4"], s["xyz"], s["used"]), (s["X4"], None, s["used"]), (None, s["xyz"], None)][j % 3]
        before = hv.launches
        hv.triangulate_points_device(P1, P2, s["xy1"], s["xy2"], *so, s["s1"], s["s2"])
        assert hv.launches == before + 1
        singles.append((s, cap))
    before = hv.launches
    hv.triangulate_points_batch_device(jobs)
    assert hv.launches == before + 1
    torch.cuda.synchronize()
    for j in range(njobs):
        for key in ("X4", "xyz", "used"):
            g, w = bufs[j][0][key], singles[j][0][key]
            assert torch.equal(g.view(torch.uint8), w.view(torch.uint8)), f"job {j} of {njobs}: {key}"


@gpu
def test_refusals_launch_nothing_and_leave_buffers_untouched(hv):
    import torch
    from hybvio_b200 import capi
    lib = hv.lib
    P1, P2, a, b = _points(50, 2)
    s1, s2 = _statuses(np.random.default_rng(1), 50, 50, "both")
    d = _dev(a, b, s1, s2)
    snap = {k: v.clone() for k, v in d.items()}
    P1c, P2c = np.ascontiguousarray(P1), np.ascontiguousarray(P2)
    nanP, infP = P1c.copy(), P2c.copy()
    nanP[1, 2] = np.nan
    infP[2, 3] = np.inf

    def dev(n=50, p1=P1c, p2=P2c, drop=()):
        p = {k: (None if k in drop else d[k].data_ptr()) for k in ("xy1", "xy2", "s1", "s2", "X4", "xyz", "used")}
        return lib.hv_triangulate_points_device(hv.h, None if p1 is None else p1.ctypes.data, None if p2 is None else p2.ctypes.data,
                                                p["xy1"], p["xy2"], p["s1"], p["s2"], n, p["X4"], p["xyz"], p["used"])

    cases = [(-1, dict(n=-1)), (-1, dict(p1=None)), (-1, dict(p2=None)), (-1, dict(drop=("xy1",))), (-1, dict(drop=("xy2",))),
             (-1, dict(drop=("X4", "xyz"))), (-5, dict(n=capi.TRIANGULATE_MAX_POINTS + 1)), (-5, dict(p1=nanP)), (-5, dict(p2=infP))]
    for rc, kw in cases:
        before = hv.launches
        assert dev(**kw) == rc, kw
        assert hv.launches == before, kw
    assert lib.hv_triangulate_points_device(None, P1c.ctypes.data, P2c.ctypes.data, None, None, None, None, 0, None, None, None) == -1
    # host call
    X4, xyz, used = np.full(200, 3.0, np.float32), np.full((50, 3), 3.0, np.float32), np.full(50, 9, np.uint8)
    before = hv.launches
    for rc, n, p1, p2, x4p, xyzp in ((-1, -1, P1c, P2c, X4, xyz), (-1, 50, None, P2c, X4, xyz), (-1, 50, P1c, P2c, None, None),
                                     (-5, capi.TRIANGULATE_MAX_POINTS + 1, P1c, P2c, X4, xyz), (-5, 50, P1c, nanP, X4, xyz)):
        assert lib.hv_triangulate_points(hv.h, None if p1 is None else p1.ctypes.data, p2.ctypes.data, a.ctypes.data, b.ctypes.data, None, None,
                                         n, None if x4p is None else x4p.ctypes.data, None if xyzp is None else xyzp.ctypes.data,
                                         used.ctypes.data) == rc, (rc, n)
    assert (X4 == 3.0).all() and (xyz == 3.0).all() and (used == 9).all() and hv.launches == before
    # batch
    good = capi.triangulate_job(P1, P2, d["xy1"], d["xy2"], d["X4"], d["xyz"], d["used"], d["s1"], d["s2"])
    bad = capi.triangulate_job(P1, P2, d["xy1"], d["xy2"], d["X4"], d["xyz"], d["used"], d["s1"], d["s2"])
    bad.n = -3
    big = capi.triangulate_job(P1, P2, d["xy1"], d["xy2"], d["X4"], d["xyz"], d["used"], d["s1"], d["s2"])
    big.n = capi.TRIANGULATE_MAX_POINTS + 1
    nonfinite = capi.triangulate_job(P1, nanP, d["xy1"], d["xy2"], d["X4"], d["xyz"], d["used"], d["s1"], d["s2"])
    noout = capi.triangulate_job(P1, P2, d["xy1"], d["xy2"], None, None, d["used"], d["s1"], d["s2"])
    J = (capi.TriangulateJob * 65)(*([good] * 65))
    assert lib.hv_triangulate_points_batch_device(hv.h, J, 0) == -1
    assert lib.hv_triangulate_points_batch_device(hv.h, J, 65) == -1
    assert lib.hv_triangulate_points_batch_device(hv.h, None, 1) == -1
    assert lib.hv_triangulate_points_batch_device(None, J, 1) == -1
    assert lib.hv_triangulate_points_batch_device(hv.h, (capi.TriangulateJob * 3)(good, good, bad), 3) == -1
    assert lib.hv_triangulate_points_batch_device(hv.h, (capi.TriangulateJob * 2)(good, noout), 2) == -1
    assert lib.hv_triangulate_points_batch_device(hv.h, (capi.TriangulateJob * 2)(good, big), 2) == -5
    assert lib.hv_triangulate_points_batch_device(hv.h, (capi.TriangulateJob * 2)(nonfinite, good), 2) == -5
    assert hv.launches == before
    torch.cuda.synchronize()
    for k, v in snap.items():
        if v is not None:
            assert torch.equal(d[k].view(torch.uint8), v.view(torch.uint8)), k
    # n = 0 accepts NULL points and outputs, and is one launch
    assert dev(n=0, drop=("xy1", "xy2", "s1", "s2", "X4", "xyz", "used")) == 0 and hv.launches == before + 1
    assert lib.hv_triangulate_points(hv.h, P1c.ctypes.data, P2c.ctypes.data, None, None, None, None, 0, None, None, None) == 0
    assert hv.launches == before + 2


@gpu
def test_python_wrapper_returns_cv2s_value_and_shape(hv):
    cv2 = pytest.importorskip("cv2")
    for name, fam, P1, P2, a, b in tc.scenes():
        if fam != "general":
            continue
        want = cv2.triangulatePoints(P1, P2, np.ascontiguousarray(a.T), np.ascontiguousarray(b.T))
        for x1, x2 in ((a.T, b.T), (a.reshape(-1, 1, 2), b.reshape(-1, 1, 2)), (a, b)):
            got = hv.triangulate_points(P1, P2, x1, x2)
            assert got.shape == want.shape and got.dtype == np.float32
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), name
    assert hv.triangulate_points(P1, P2, a[:0], b[:0]).shape == (4, 0)


def test_ctypes_triangulate_job_matches_the_header(tmp_path):
    from hybvio_b200 import capi
    py = capi.TriangulateJob
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "hybvio_b200.h"', 'int main(void) {',
             'printf("size %zu\\n", sizeof(hv_triangulate_job));']
    lines += [f'printf("{f} %zu\\n", offsetof(hv_triangulate_job, {f}));' for f, _ in py._fields_]
    lines.append("return 0; }")
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines))
    subprocess.check_call(["gcc", "-std=c99", "-I" + os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = dict(ln.split() for ln in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["size"]) == ctypes.sizeof(py)
    for f, _ in py._fields_:
        assert int(got[f]) == getattr(py, f).offset, f


@gpu
def test_stereo_chain_triangulation_to_pnp_matches_the_oracle(hv, orc):
    """ingest -> pyramids of frame k's left and right and frame k+1's left -> stereo LK -> temporal LK -> hv_triangulate_points_device
    (status = stereo, status2 = temporal) -> hv_solve_pnp_ransac_device(xyz, frame k+1's points, used): the last four are four launches
    with no host synchronisation; against the oracle triangulation and the oracle PnP on the downloaded LK outputs. In synth a left
    point appears in the right image at x + d, d from 8 to 16 px, so the right camera sits at -B: P2 = K [I | (B, 0, 0)], Z = f B / d."""
    import torch
    from hybvio_b200 import capi, synth
    from oracle import pnp_oracle
    w, h, n, cap, k = 752, 480, 300, 384, 2
    fx, fy, cx, cy, base = 450.0, 450.0, 376.0, 240.0, 0.1              # depths 2.8 to 5.6 m
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]])
    P1, P2 = tc.projection(k=K), tc.projection(t=(base, 0.0, 0.0), k=K)
    L0, R0 = synth.stereo_frame(k, w, h)
    L1, _ = synth.stereo_frame(k + 1, w, h)
    pl, pr, pl1 = hv.pyramid(w, h), hv.pyramid(w, h), hv.pyramid(w, h)
    ing = capi.Ingest(hv, w, h)
    for img, p in ((L0, pl), (R0, pr), (L1, pl1)):
        ing.frame(img, p, want_gray=False)
    pts = synth.interior_points(n, w, h, seed=17, margin=30).astype(np.float32)
    f32 = lambda *s: torch.zeros(s, dtype=torch.float32, device="cuda")      # noqa: E731
    u8 = lambda: torch.full((cap,), 7, dtype=torch.uint8, device="cuda")     # noqa: E731
    d_left = torch.full((cap, 2), NONE, dtype=torch.float32, device="cuda")
    d_left[:n] = torch.from_numpy(pts)
    d_right, d_left1, d_xyz = f32(cap, 2), f32(cap, 2), f32(cap, 3)
    d_st_s, d_st_t, d_used = u8(), u8(), u8()
    d_ts_s, d_ts_t = torch.zeros(cap, dtype=torch.int32, device="cuda"), torch.zeros(cap, dtype=torch.int32, device="cuda")
    r, t = torch.full((3,), float("nan"), dtype=torch.float64, device="cuda"), torch.full((3,), float("nan"), dtype=torch.float64, device="cuda")
    mask = u8()
    inl, ok = torch.full((1,), -1, dtype=torch.int32, device="cuda"), torch.full((1,), -1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    before = hv.launches
    hv.lk_track_device(pl, pr, d_left.data_ptr(), d_right.data_ptr(), d_st_s.data_ptr(), d_ts_s.data_ptr(), cap, False)    # stereo
    hv.lk_track_device(pl, pl1, d_left.data_ptr(), d_left1.data_ptr(), d_st_t.data_ptr(), d_ts_t.data_ptr(), cap, False)  # temporal
    hv.triangulate_points_device(P1, P2, d_left, d_right, None, d_xyz, d_used, d_st_s, d_st_t)
    hv.solve_pnp_ransac_device(d_xyz, d_left1, r, t, mask, inl, ok, fx, fy, cx, cy, 100, 8.0, 0.99, d_status=d_used)
    assert hv.launches == before + 4
    torch.cuda.synchronize()
    left, right, left1 = d_left.cpu().numpy(), d_right.cpu().numpy(), d_left1.cpu().numpy()
    st_s, st_t = d_st_s.cpu().numpy(), d_st_t.cpu().numpy()
    _, xyz_o, used_o = orc.triangulate(P1, P2, left, right, st_s, st_t)
    assert np.array_equal(d_xyz.cpu().numpy().view(np.uint32), xyz_o.view(np.uint32)) and np.array_equal(d_used.cpu().numpy(), used_o)
    idx = np.flatnonzero(used_o)
    assert idx.size > n // 2
    Z = xyz_o[idx, 2]
    assert (np.median(Z) > 2.0) and (np.median(Z) < 7.0), np.median(Z)
    op = pnp_oracle.OraclePnp()
    okw, rw, tw, mw, inlw = op.solve_pnp_ransac(xyz_o[idx], left1[idx], fx, fy, cx, cy, 100, 8.0, 0.99)
    full = np.zeros(cap, np.uint8)
    full[idx] = mw
    assert int(ok.item()) == okw and int(inl.item()) == inlw
    assert np.array_equal(mask.cpu().numpy(), full)
    assert np.array_equal(r.cpu().numpy().view(np.uint64), rw.view(np.uint64)) and np.array_equal(t.cpu().numpy().view(np.uint64), tw.view(np.uint64))
    assert okw == 1 and inlw >= 4
    ing.close()
    for p in (pl, pr, pl1):
        p.release()
