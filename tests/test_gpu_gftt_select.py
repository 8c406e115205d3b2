"""Corner selection on the device: hv_gftt_select_device / hv_gftt_corners (csrc/gftt_select.cu) through the C ABI against orc_gftt_corners
(oracle/hv_oracle_gftt.c, pinned to the compiled reference by tests/golden/gftt_golden.npz): every list BIT-identical with its count,
the padding slots set to HV_CORNER_NONE -- on the golden frames, over the detector's frame sizes and cells with a sweep of mask radius,
max_tracks and previous corners, on crafted key points (stability, signed zeros, empty cells, the rounded distance, 1 .. 16384 key
points), in the device chain detect -> select -> cornerSubPix -> stereo LK with one synchronisation, and the documented error codes."""
import os

import numpy as np
import pytest

import gftt_select_common as gc
from hybvio_b200 import synth
from oracle import gftt_oracle

HV_ERR_INVALID, HV_ERR_UNSUPPORTED = -1, -5
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gftt_golden.npz")
SIZES = [(752, 480, 3), (512, 512, 5), (203, 77, 1), (64, 64, 2), (97, 130, 7), (751, 479, 4), (1280, 720, 6)]
RADII = [0, 1, 8, 50]
MAX_TRACKS = [1, 7, 150, 100000]
NPREV = [0, 40, 500]


@pytest.fixture(scope="module")
def orc(oracle_lk):
    return gftt_oracle.OracleGftt()


def pyramid(hv, img, levels=1):
    p = hv.pyramid(img.shape[1], img.shape[0], 31, levels)
    p.build(np.ascontiguousarray(img))
    return p


def assert_list(got, want, what):
    assert got.shape == want.shape, f"{what}: {len(got)} corners, oracle {len(want)}"
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"{what}: first difference at {np.nonzero((got != want).any(axis=1))[0][:5]}"


def host_corners(hv, p, prev, r, m, cell, extra=4):
    """hv_gftt_corners with `extra` slots beyond the worst case: (list, padding)."""
    from hybvio_b200 import capi
    import ctypes
    nkp = int(np.prod(p.gftt_cells(cell)))
    cap = gc.capacity(nkp, r, m) + extra
    out = np.zeros((cap, 2), np.float32)
    cnt = ctypes.c_int(-1)
    prev = np.ascontiguousarray(prev, np.float32).reshape(-1, 2)
    capi.check(capi.load().hv_gftt_corners(hv.h, p.h, 3, cell, 1e-3, prev.ctypes.data, len(prev), r, m, out.ctypes.data, cap, ctypes.byref(cnt)),
               "hv_gftt_corners")
    return out[:cnt.value], out[cnt.value:]


def device_select(hv, d_kp, prev, r, m, extra=4):
    """hv_gftt_select_device on a device key-point tensor: (list, padding), read back after one synchronisation."""
    import torch
    nkp = d_kp.shape[0]
    cap = gc.capacity(nkp, r, m) + extra
    d_out = torch.full((cap, 2), 7.0, dtype=torch.float32, device="cuda")
    d_cnt = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    d_prev = torch.from_numpy(np.ascontiguousarray(prev, np.float32).reshape(-1, 2)).cuda() if len(prev) else None
    torch.cuda.synchronize()
    hv.gftt_select_device(d_kp, d_out, d_cnt, d_prev, r, m)
    hv.sync()
    n = int(d_cnt.item())
    out = d_out.cpu().numpy()
    return out[:n], out[n:]


def assert_padding(pad, what):
    assert np.all(pad.view(np.uint32) == gc.NONE.view(np.uint32)), f"{what}: padding {pad[:3]}"


@pytest.mark.gpu
def test_golden_lists_of_the_reference(hv):
    g = np.load(GOLD)
    for name in "ABC":
        img, prev = g[name + "_img"], g[name + "_prev"]
        p = pyramid(hv, img)
        assert_list(p.gftt_corners(None, 0, 150), g[name + "_corners_r0"], name + " r0")
        assert_list(p.gftt_corners(prev, 50, 150), g[name + "_corners_r50"], name + " r50")
        p.release()


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,k", SIZES)
@pytest.mark.parametrize("cell", [32, 16, 8])
def test_sweep_vs_oracle_both_entry_points(hv, orc, w, h, k, cell):
    import torch
    img, _ = synth.stereo_frame(k, w, h)
    kp = orc.collect(orc.response(img), cell, 1e-3)
    p = pyramid(hv, img)
    d_kp = torch.zeros((len(kp), 3), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    p.gftt_detect_device(d_kp.data_ptr(), 3, cell, 1e-3)
    hv.sync()
    assert np.array_equal(d_kp.cpu().numpy().view(np.uint32), kp.view(np.uint32))
    for nprev in NPREV:
        prev = gc.prev_points(nprev, k * 7 + nprev, w, h)
        for r in RADII:
            for m in MAX_TRACKS:
                want = orc.corners(kp, prev, r, m)
                what = f"{w}x{h} cell {cell} nprev {nprev} r {r} max {m}"
                got, pad = host_corners(hv, p, prev, r, m, cell)
                assert_list(got, want, "host " + what)
                assert_padding(pad, "host " + what)
                got, pad = device_select(hv, d_kp, prev, r, m)
                assert_list(got, want, "device " + what)
                assert_padding(pad, "device " + what)
    p.release()


@pytest.mark.gpu
def test_crafted_key_points(hv, orc):
    import torch
    for name, kp, prev, r, m in gc.crafted_cases(big=True):
        d_kp = torch.from_numpy(np.ascontiguousarray(kp, np.float32).reshape(-1, 3)).cuda()
        got, pad = device_select(hv, d_kp, prev, r, m)
        assert_list(got, orc.corners(kp, prev, r, m), name)
        assert_padding(pad, name)


@pytest.mark.gpu
def test_launch_counts(hv, orc):
    import torch
    img, _ = synth.stereo_frame(1, 752, 480)
    p = pyramid(hv, img)
    before = hv.launches
    p.gftt_corners(None, 8, 150)
    assert hv.launches - before == 2                       # detect + select
    small = pyramid(hv, img[:20, :20])
    before = hv.launches
    assert small.gftt_corners(None, 8, 150).shape == (0, 2)  # no cell: nothing launched
    assert hv.launches == before
    d_out = torch.zeros((5, 2), dtype=torch.float32, device="cuda")
    d_cnt = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    hv.gftt_select_device(torch.zeros((0, 3), dtype=torch.float32, device="cuda"), d_out, d_cnt, None, 8, 150)
    hv.sync()
    assert hv.launches == before + 1 and int(d_cnt.item()) == 0
    assert_padding(d_out.cpu().numpy(), "nkp = 0")
    p.release(); small.release()


def _chain(hv, pl, pr, r, m, prev, cell=32):
    """detect -> select -> cornerSubPix over capacity -> LK left -> right over capacity, one synchronisation at the end."""
    import torch
    nkp = int(np.prod(pl.gftt_cells(cell)))
    cap = gc.capacity(nkp, r, m) + 3
    d_kp = torch.empty((nkp, 3), dtype=torch.float32, device="cuda")
    d_xy = torch.empty((cap, 2), dtype=torch.float32, device="cuda")
    d_cnt = torch.empty((1,), dtype=torch.int32, device="cuda")
    d_next = torch.empty((cap, 2), dtype=torch.float32, device="cuda")
    d_st = torch.empty((cap,), dtype=torch.uint8, device="cuda")
    d_ts = torch.empty((cap,), dtype=torch.int32, device="cuda")
    d_prev = torch.from_numpy(np.ascontiguousarray(prev, np.float32)).cuda() if len(prev) else None
    torch.cuda.synchronize()
    pl.gftt_detect_device(d_kp.data_ptr(), 3, cell, 1e-3)
    hv.gftt_select_device(d_kp, d_xy, d_cnt, d_prev, r, m)
    pl.subpix_refine_device(d_xy)
    hv.lk_track_device(pl, pr, d_xy, d_next, d_st, d_ts, cap, False)
    hv.sync()
    return int(d_cnt.item()), d_xy.cpu().numpy(), d_next.cpu().numpy(), d_st.cpu().numpy(), d_ts.cpu().numpy()


def _check_chain(hv, orc, pl, pr, L, prev, r, m, what):
    n, xy, nxt, st, ts = _chain(hv, pl, pr, r, m, prev)
    want = orc.corners(orc.collect(orc.response(L), 32, 1e-3), prev, r, m)
    assert n == len(want), what
    ref_xy = pl.subpix_refine(want)
    ref_next, ref_st, ref_ts = hv.lk_track(pl, pr, ref_xy)
    assert_list(xy[:n], ref_xy, what + " refined")
    assert_list(nxt[:n], ref_next, what + " tracked")
    assert np.array_equal(st[:n], ref_st) and np.array_equal(ts[:n], ref_ts), what
    assert_padding(xy[n:], what + " refined padding")
    assert np.all(st[n:] == 0) and np.all(ts[n:] == 4), f"{what}: padding status {st[n:]}, track status {ts[n:]}"


@pytest.mark.gpu
@pytest.mark.parametrize("r,m", [(0, 150), (8, 150), (50, 7)])
def test_device_chain_matches_the_host_path(hv, orc, r, m):
    L, R = synth.stereo_frame(4, 752, 480)
    pl, pr = pyramid(hv, L, 3), pyramid(hv, R, 3)
    _check_chain(hv, orc, pl, pr, L, gc.prev_points(40, 3), r, m, f"host-built pyramids r {r} max {m}")
    pl.release(); pr.release()


@pytest.mark.gpu
def test_device_chain_on_batch_built_pyramids_with_device_sources(hv, orc):
    import torch
    L, R = synth.stereo_frame(6, 751, 479)
    pyrs = [hv.pyramid(751, 479, 31, 3) for _ in range(2)]
    dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (L, R)]
    torch.cuda.synchronize()
    hv.build_pyramids(pyrs, dev, device=True)
    _check_chain(hv, orc, pyrs[0], pyrs[1], L, gc.prev_points(500, 4, 751, 479), 8, 150, "batch build, device sources")
    for p in pyrs:
        p.release()


@pytest.mark.gpu
def test_error_codes(hv):
    import ctypes
    import torch
    from hybvio_b200 import capi
    lib = capi.load()
    img, _ = synth.stereo_frame(2, 256, 128)
    p = pyramid(hv, img)
    other = capi.Context(0)
    q = other.pyramid(256, 128, 31, 1)
    kp = torch.zeros((gc.MAX_KP + 1, 3), dtype=torch.float32, device="cuda")
    out = torch.zeros((2 * gc.MAX_KP + 2, 2), dtype=torch.float32, device="cuda")
    cnt = torch.zeros((1,), dtype=torch.int32, device="cuda")
    prev = torch.zeros((4, 2), dtype=torch.float32, device="cuda")
    K, O, C, P = kp.data_ptr(), out.data_ptr(), cnt.data_ptr(), prev.data_ptr()
    torch.cuda.synchronize()
    sel = lib.hv_gftt_select_device
    before = hv.launches                    # no call below launches anything
    assert sel(None, K, 10, P, 4, 8, 150, O, 40, C) == HV_ERR_INVALID
    assert sel(hv.h, None, 10, P, 4, 8, 150, O, 40, C) == HV_ERR_INVALID
    assert sel(hv.h, K, 10, None, 4, 8, 150, O, 40, C) == HV_ERR_INVALID
    assert sel(hv.h, K, 10, P, 4, 8, 150, None, 40, C) == HV_ERR_INVALID
    assert sel(hv.h, K, 10, P, 4, 8, 150, O, 40, None) == HV_ERR_INVALID
    assert sel(hv.h, K, -1, P, 4, 8, 150, O, 40, C) == HV_ERR_INVALID
    assert sel(hv.h, K, 10, P, -1, 8, 150, O, 40, C) == HV_ERR_INVALID
    assert sel(hv.h, K, 10, P, 4, 8, 0, O, 40, C) == HV_ERR_INVALID
    assert sel(hv.h, K, 10, P, 4, 8, 7, O, 6, C) == HV_ERR_INVALID        # capacity below min(max_tracks, 2 nkp) = 7
    assert sel(hv.h, K, 10, P, 4, 8, 150, O, 19, C) == HV_ERR_INVALID     # ... = 20
    assert sel(hv.h, K, 10, P, 4, 0, 7, O, 19, C) == HV_ERR_INVALID       # no radius: 2 nkp = 20 whatever max_tracks
    assert sel(hv.h, K, gc.MAX_KP + 1, P, 4, 8, 150, O, 2 * gc.MAX_KP + 2, C) == HV_ERR_UNSUPPORTED
    assert sel(hv.h, K, 10, P, 4, 46341, 150, O, 40, C) == HV_ERR_UNSUPPORTED
    host = np.zeros((200, 2), np.float32)
    hc = ctypes.c_int(-1)
    hp = np.zeros((4, 2), np.float32)
    H, HP = host.ctypes.data, hp.ctypes.data
    cor = lib.hv_gftt_corners
    nkp = int(np.prod(p.gftt_cells(32)))                                     # 8 x 4 = 32 cells
    assert cor(None, p.h, 3, 32, 1e-3, HP, 4, 8, 150, H, 64, ctypes.byref(hc)) == HV_ERR_INVALID
    assert cor(hv.h, None, 3, 32, 1e-3, HP, 4, 8, 150, H, 64, ctypes.byref(hc)) == HV_ERR_INVALID
    assert cor(hv.h, q.h, 3, 32, 1e-3, HP, 4, 8, 150, H, 64, ctypes.byref(hc)) == HV_ERR_INVALID       # pyramid of another context
    assert cor(hv.h, p.h, 3, 32, 1e-3, None, 4, 8, 150, H, 64, ctypes.byref(hc)) == HV_ERR_INVALID
    assert cor(hv.h, p.h, 3, 32, 1e-3, HP, 4, 8, 150, None, 64, ctypes.byref(hc)) == HV_ERR_INVALID
    assert cor(hv.h, p.h, 3, 32, 1e-3, HP, 4, 8, 150, H, 64, None) == HV_ERR_INVALID
    assert cor(hv.h, p.h, 3, 32, 1e-3, HP, -1, 8, 150, H, 64, ctypes.byref(hc)) == HV_ERR_INVALID
    assert cor(hv.h, p.h, 3, 32, 1e-3, HP, 4, 8, 0, H, 64, ctypes.byref(hc)) == HV_ERR_INVALID
    assert cor(hv.h, p.h, 3, 32, 1e-3, HP, 4, 8, 150, H, 2 * nkp - 1, ctypes.byref(hc)) == HV_ERR_INVALID
    assert cor(hv.h, p.h, 3, 32, 1e-3, HP, 4, 0, 7, H, 2 * nkp - 1, ctypes.byref(hc)) == HV_ERR_INVALID
    assert cor(hv.h, p.h, 5, 32, 1e-3, HP, 4, 8, 150, H, 64, ctypes.byref(hc)) == HV_ERR_UNSUPPORTED   # block size 3 only
    assert hv.launches == before
    big = hv.pyramid(1280, 720, 31, 1)
    assert cor(hv.h, big.h, 3, 4, 1e-3, HP, 4, 8, 150, H, 200, ctypes.byref(hc)) == HV_ERR_UNSUPPORTED  # 320 x 180 = 57600 key points
    assert hv.launches == before
    q.release(); other.close(); p.release(); big.release()

