"""GPU: cv::findEssentialMat (RANSAC) on the device -- hv_find_essential, hv_find_essential_device and hv_find_essential_batch_device --
against the plain-C oracle (oracle/hv_oracle_essential.c), bit for bit in E, nsol, mask and inliers, on the seeded scenes of
tests/essential_common.py with three status patterns; batches against the per-call results; refusals; and the chain ingest -> pyramid ->
LK (device) -> hv_find_essential_device on LK's status over a padded capacity."""
import ctypes
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import essential_common as ec  # noqa: E402

pytestmark = pytest.mark.gpu
NONE = np.float32(-1.0e6)          # HV_CORNER_NONE


@pytest.fixture(scope="module")
def orc():
    import subprocess
    from oracle import essential_oracle
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if not os.path.exists(essential_oracle.ORACLE_SO):
        subprocess.check_call(["make", "-C", root, "oracle"])
    return essential_oracle.OracleEssential()


def _status(kind, n, seed):
    if kind == "none":
        return None
    rng = np.random.default_rng(seed)
    return (rng.random(n) > 0.25).astype(np.uint8) * rng.integers(1, 256, n).astype(np.uint8)


def _host(hv, p1, p2, st, prob, thr, mi, fx=ec.FX, fy=ec.FY, cx=ec.CX, cy=ec.CY):
    n = p1.shape[0]
    E = np.full(90, np.nan)
    mask = np.full(max(n, 1), 7, np.uint8)
    nsol, inl = ctypes.c_int(-1), ctypes.c_int(-1)
    from hybvio_b200.capi import _ptr, check
    check(hv.lib.hv_find_essential(hv.h, _ptr(p1), _ptr(p2), _ptr(st), n, fx, fy, cx, cy, prob, thr, mi, _ptr(E), ctypes.byref(nsol),
                                   _ptr(mask), ctypes.byref(inl)), "hv_find_essential")
    return E.reshape(10, 3, 3), nsol.value, mask[:n], inl.value


def _dev_buffers(p1, p2, st, cap=None):
    import torch
    n = p1.shape[0]
    cap = n if cap is None else cap
    b = {"xy1": torch.full((max(cap, 1), 2), float(NONE), dtype=torch.float32, device="cuda"),
         "xy2": torch.full((max(cap, 1), 2), float(NONE), dtype=torch.float32, device="cuda"),
         "E": torch.full((90,), float("nan"), dtype=torch.float64, device="cuda"),
         "nsol": torch.full((1,), -1, dtype=torch.int32, device="cuda"), "inl": torch.full((1,), -1, dtype=torch.int32, device="cuda"),
         "mask": torch.full((max(cap, 1),), 7, dtype=torch.uint8, device="cuda"), "st": None}
    if n:
        b["xy1"][:n] = torch.from_numpy(p1)
        b["xy2"][:n] = torch.from_numpy(p2)
    if st is not None:
        b["st"] = torch.zeros(max(cap, 1), dtype=torch.uint8, device="cuda")
        if n:
            b["st"][:n] = torch.from_numpy(st)
    return b


def _job(b, n, fx=ec.FX, fy=ec.FY, cx=ec.CX, cy=ec.CY):
    from hybvio_b200 import capi
    return capi.essential_job(b["xy1"], b["xy2"], b["E"], b["nsol"], b["mask"], b["inl"], fx, fy, cx, cy, b["st"], n)


def _read(b, n):
    return (b["E"].cpu().numpy().reshape(10, 3, 3), int(b["nsol"].item()), b["mask"][:n].cpu().numpy(), int(b["inl"].item()))


def _same(got, want, what):
    E, ns, mask, inl = got
    Eo, nso, masko, inlo = want
    assert ns == nso, f"{what}: nsol {ns} != {nso}"
    assert inl == inlo, f"{what}: inliers {inl} != {inlo}"
    assert np.array_equal(mask, masko), f"{what}: mask differs at {np.flatnonzero(mask != masko)[:10]}"
    assert np.array_equal(E.view(np.uint64), Eo.view(np.uint64)), f"{what}: E differs (max {np.nanmax(np.abs(E - Eo))})"


CASES = list(ec.cases())


@pytest.mark.parametrize("status", ["none", "random"])
def test_host_and_device_calls_match_the_oracle_bitwise(hv, orc, status):
    import torch
    for case in CASES:
        name, seed, m, _, _, _, prob, thr, mi = case
        p1, p2 = ec.case_points(case)
        st = _status(status, m, seed)
        want = orc.find_essential(p1, p2, ec.FX, ec.FY, ec.CX, ec.CY, prob, thr, mi, st)
        _same(_host(hv, p1, p2, st, prob, thr, mi), want, f"{name} host")
        b = _dev_buffers(p1, p2, st)
        before = hv.launches
        hv.find_essential_device(b["xy1"], b["xy2"], b["E"], b["nsol"], b["mask"], b["inl"], ec.FX, ec.FY, ec.CX, ec.CY, prob, thr, mi,
                                 d_status=b["st"], n=m)
        assert hv.launches == before + 1
        torch.cuda.synchronize()
        _same(_read(b, m), want, f"{name} device")


def test_five_points_every_solution_matches_the_oracle(hv, orc):
    rng = np.random.default_rng(5)
    for k in range(300):
        p1, p2 = ec.scene(rng, 5, 0.0, 0.5, "side" if k % 2 else "forward")
        want = orc.find_essential(p1, p2, ec.FX, ec.FY, ec.CX, ec.CY)
        got = _host(hv, p1, p2, None, 0.999, 1.0, 1000)
        _same(got, want, f"five points #{k}")
        assert got[1] >= 1 and got[3] == 5 and got[2].tolist() == [1] * 5


def test_small_and_degenerate_inputs_match_the_oracle(hv, orc):
    rng = np.random.default_rng(9)
    for m in (0, 1, 4, 5, 6, 7):
        p1, p2 = ec.scene(rng, m, 0.0, 0.3)
        want = orc.find_essential(p1, p2, ec.FX, ec.FY, ec.CX, ec.CY)
        _same(_host(hv, p1, p2, None, 0.999, 1.0, 1000), want, f"m = {m}")
        if m < 5:
            assert want[1] == 0 and want[3] == 0 and not want[2].any()
    for name, p1, p2 in ec.degenerate_scenes():
        want = orc.find_essential(p1, p2, ec.FX, ec.FY, ec.CX, ec.CY)
        _same(_host(hv, p1, p2, None, 0.999, 1.0, 1000), want, name)
    # extreme but accepted parameters: threshold 0, negative, NaN, inf; max_iters 0 and -5; prob near 0
    p1, p2 = ec.scene(rng, 150, 0.3, 0.5)
    for prob, thr, mi in ((0.999, 0.0, 1000), (0.999, -1.0, 1000), (0.999, float("nan"), 1000), (0.999, float("inf"), 1000),
                          (0.999, 1.0, 0), (0.999, 1.0, -5), (1e-300, 1.0, 1000), (0.5, 1.0, 4096)):
        want = orc.find_essential(p1, p2, ec.FX, ec.FY, ec.CX, ec.CY, prob, thr, mi)
        _same(_host(hv, p1, p2, None, prob, thr, mi), want, f"prob {prob} threshold {thr} max_iters {mi}")


@pytest.mark.parametrize("njobs", [1, 2, 5, 64])
def test_batches_match_the_per_call_results(hv, njobs):
    import torch
    rng = np.random.default_rng(100 + njobs)
    ms = [0, 4, 5, 6, 150, 600, 2000, 20, 300, 8]
    bufs, jobs, singles = [], [], []
    for j in range(njobs):
        m = ms[j % len(ms)]
        p1, p2 = ec.scene(rng, m, [0.1, 0.3, 0.5][j % 3], 0.5, "side" if j % 2 else "forward")
        st = _status("random" if j % 3 == 1 else "none", m, j)
        fx, fy = ec.FX * (1 + 0.01 * (j % 5)), ec.FY * (1 - 0.01 * (j % 3))
        b = _dev_buffers(p1, p2, st)
        s = _dev_buffers(p1, p2, st)
        bufs.append((b, m))
        jobs.append(_job(b, m, fx, fy))
        before = hv.launches
        hv.find_essential_device(s["xy1"], s["xy2"], s["E"], s["nsol"], s["mask"], s["inl"], fx, fy, ec.CX, ec.CY, 0.99, 1.0, 1000,
                                 d_status=s["st"], n=m)
        assert hv.launches == before + 1
        singles.append((s, m))
    before = hv.launches
    hv.find_essential_batch_device(jobs, 0.99, 1.0, 1000)
    assert hv.launches == before + 1
    torch.cuda.synchronize()
    for j in range(njobs):
        _same(_read(*bufs[j]), _read(*singles[j]), f"job {j} of {njobs}")


def test_refusals_launch_nothing_and_leave_buffers_untouched(hv):
    import torch
    from hybvio_b200 import capi
    p1, p2 = ec.scene(np.random.default_rng(3), 50, 0.2, 0.5)
    b = _dev_buffers(p1, p2, None)
    big = _dev_buffers(*ec.scene(np.random.default_rng(4), 4097, 0.2, 0.5), None)
    nan = float("nan")
    lib = hv.lib

    def dev(n=50, prob=0.999, thr=1.0, mi=1000, fx=ec.FX, fy=ec.FY, cx=ec.CX, cy=ec.CY, bb=b, E=True):
        return lib.hv_find_essential_device(hv.h, bb["xy1"].data_ptr(), bb["xy2"].data_ptr(), None, n, fx, fy, cx, cy, prob, thr, mi,
                                            bb["E"].data_ptr() if E else None, bb["nsol"].data_ptr(), bb["mask"].data_ptr(),
                                            bb["inl"].data_ptr())

    cases = [(-1, dict(n=-1)), (-1, dict(prob=0.0)), (-1, dict(prob=1.0)), (-1, dict(prob=-0.5)), (-1, dict(prob=1.5)), (-1, dict(prob=nan)),
             (-1, dict(E=False)), (-5, dict(n=4097, bb=big)), (-5, dict(mi=4097)), (-5, dict(fx=0.0)), (-5, dict(fy=nan)),
             (-5, dict(cx=float("inf"))), (-5, dict(fx=100.0, fy=-100.0))]
    snap = {k: v.clone() for k, v in b.items() if v is not None}
    for rc, kw in cases:
        before = hv.launches
        assert dev(**kw) == rc, kw
        assert hv.launches == before, kw
    assert lib.hv_find_essential_device(None, None, None, None, 0, 1.0, 1.0, 0.0, 0.0, 0.5, 1.0, 10, None, None, None, None) == -1
    # host call and batch
    E = np.full(90, 3.0); mask = np.full(50, 7, np.uint8); ns, inl = ctypes.c_int(-9), ctypes.c_int(-9)
    before = hv.launches
    assert lib.hv_find_essential(hv.h, p1.ctypes.data, p2.ctypes.data, None, 50, ec.FX, ec.FY, ec.CX, ec.CY, 1.0, 1.0, 100,
                                 E.ctypes.data, ctypes.byref(ns), mask.ctypes.data, ctypes.byref(inl)) == -1
    assert lib.hv_find_essential(hv.h, p1.ctypes.data, p2.ctypes.data, None, 50, ec.FX, ec.FY, ec.CX, ec.CY, 0.9, 1.0, 5000,
                                 E.ctypes.data, ctypes.byref(ns), mask.ctypes.data, ctypes.byref(inl)) == -5
    assert (E == 3.0).all() and (mask == 7).all() and ns.value == -9 and inl.value == -9
    good = _job(b, 50)
    bad = _job(b, 50)
    bad.n = -3
    J = (capi.EssentialJob * 65)(*([good] * 65))
    assert lib.hv_find_essential_batch_device(hv.h, J, 0, 0.9, 1.0, 10) == -1
    assert lib.hv_find_essential_batch_device(hv.h, J, 65, 0.9, 1.0, 10) == -1
    assert lib.hv_find_essential_batch_device(hv.h, None, 1, 0.9, 1.0, 10) == -1
    J2 = (capi.EssentialJob * 3)(good, good, bad)
    assert lib.hv_find_essential_batch_device(hv.h, J2, 3, 0.9, 1.0, 10) == -1
    assert lib.hv_find_essential_batch_device(hv.h, J2, 2, 0.9, 1.0, 4097) == -5
    assert lib.hv_find_essential_batch_device(hv.h, J2, 2, nan, 1.0, 10) == -1
    assert hv.launches == before
    torch.cuda.synchronize()
    for k, v in snap.items():
        assert torch.equal(b[k].view(torch.uint8) if v.dtype == torch.float64 else b[k], v.view(torch.uint8) if v.dtype == torch.float64 else v), k


def test_lk_chain_on_device_status_matches_the_oracle(hv, orc):
    """ingest -> pyramid -> LK (device, padded capacity) -> hv_find_essential_device on LK's d_status, against the oracle fed the same
    end points and status from the host."""
    import torch
    from hybvio_b200 import synth
    w, h, n, cap = 752, 480, 300, 384
    from hybvio_b200 import capi
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
    b = _dev_buffers(np.zeros((0, 2), np.float32), np.zeros((0, 2), np.float32), None, cap)
    before = hv.launches
    hv.lk_track_device(p0, p1, d_prev.data_ptr(), d_next.data_ptr(), d_st.data_ptr(), d_ts.data_ptr(), cap, False)
    mid = hv.launches
    hv.find_essential_device(d_prev, d_next, b["E"], b["nsol"], b["mask"], b["inl"], ec.FX, ec.FY, ec.CX, ec.CY, 0.999, 1.0, 1000,
                             d_status=d_st)
    assert hv.launches == mid + 1 and mid > before
    torch.cuda.synchronize()
    st = d_st.cpu().numpy()
    assert st[n:].sum() == 0 and st[:n].sum() > n // 2
    want = orc.find_essential(d_prev.cpu().numpy(), d_next.cpu().numpy(), ec.FX, ec.FY, ec.CX, ec.CY, 0.999, 1.0, 1000, st)
    _same(_read(b, cap), want, "LK chain")
    assert want[1] == 1 and want[3] > n // 3
    ing.close()
    p0.release()
    p1.release()
