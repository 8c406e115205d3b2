"""Sub-pixel corner refinement on the device: hv_subpix_refine / hv_subpix_refine_device (csrc/subpix.cu) through the C ABI against the
cv::cornerSubPix oracle (oracle/hv_oracle_subpix.c, itself bit-exact to cv2 with IPP off, test_oracle_subpix.py): every refined
corner BIT-identical, over the same sweep of windows, zero zones, criteria, images and start points; on pyramids from hv_pyr_build,
hv_pyr_build_batch with device sources and hv_ingest_frame with a remap; n = 0 .. 2000; the documented error codes."""
import numpy as np
import pytest

import subpix_common as sc
from oracle import subpix_oracle as so

HV_ERR_INVALID, HV_ERR_UNSUPPORTED = -1, -5


@pytest.fixture(scope="module")
def orc(oracle_lk):
    return so.OracleSubpix()


@pytest.fixture(scope="module")
def imgs():
    return sc.images()


def pyramid(hv, img):
    p = hv.pyramid(img.shape[1], img.shape[0], 31, 1)
    p.build(np.ascontiguousarray(img))
    return p


def device_refine(hv, p, pts, *args):
    import torch
    d = torch.from_numpy(np.ascontiguousarray(pts, np.float32)).cuda()
    torch.cuda.synchronize()
    p.subpix_refine_device(d, *args)
    hv.sync()
    return d.cpu().numpy()


def assert_bits(got, want, what):
    bad = np.nonzero((got.view(np.uint32) != want.view(np.uint32)).any(axis=1))[0]
    assert len(bad) == 0, f"{what}: {len(bad)} corners differ, first {bad[:5]}: {got[bad[:3]]} vs {want[bad[:3]]}"


@pytest.mark.gpu
@pytest.mark.parametrize("zero", sc.ZERO_ZONES, ids=str)
@pytest.mark.parametrize("win", sc.WINDOWS, ids=str)
def test_bit_exact_vs_oracle_windows_and_zero_zones(hv, orc, imgs, win, zero):
    z = sc.zero_zone(zero, win)
    for name, img in imgs.items():
        pts = sc.points(img, win, seed=len(name))
        want = orc.refine(img, pts, win, z, (3, 30, 0.01))
        p = pyramid(hv, img)
        assert_bits(p.subpix_refine(pts, win, z, (3, 30, 0.01)), want, f"host {name} win {win} zero {z}")
        assert_bits(device_refine(hv, p, pts, win, z, (3, 30, 0.01)), want, f"device {name} win {win} zero {z}")
        p.release()


@pytest.mark.gpu
@pytest.mark.parametrize("crit", sc.CRITERIA, ids=str)
def test_bit_exact_vs_oracle_criteria(hv, orc, imgs, crit):
    for win in [(2, 3), (5, 5)]:
        for name, img in imgs.items():
            pts = sc.points(img, win, seed=3)
            want = orc.refine(img, pts, win, (-1, -1), crit)
            p = pyramid(hv, img)
            assert_bits(p.subpix_refine(pts, win, (-1, -1), crit), want, f"host {name} win {win} crit {crit}")
            assert_bits(device_refine(hv, p, pts, win, (-1, -1), crit), want, f"device {name} win {win} crit {crit}")
            p.release()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [0, 1, 150, 200, 2000])
def test_counts_and_launches(hv, orc, n):
    img = sc.images()["frame752"]
    h, w = img.shape
    pts = np.random.RandomState(n).uniform([0, 0], [w - 1, h - 1], (n, 2)).astype(np.float32)
    p = pyramid(hv, img)
    want = orc.refine(img, pts, (5, 5), (-1, -1), (3, 30, 0.01)) if n else pts
    before = hv.launches
    got = p.subpix_refine(pts, (5, 5), (-1, -1), (3, 30, 0.01))
    assert hv.launches - before == (1 if n else 0)
    assert_bits(got, want, f"host n={n}")
    before = hv.launches
    assert_bits(device_refine(hv, p, pts, (5, 5), (-1, -1), (3, 30, 0.01)), want, f"device n={n}")
    assert hv.launches - before == (1 if n else 0)
    p.release()


@pytest.mark.gpu
def test_pyramids_from_batch_build_and_ingest(hv, orc):
    """Level 0 filled by the fused pyramid kernel from device sources (stereo batch), and by the ingest path with a remap table."""
    import torch
    from hybvio_b200 import capi
    from oracle import ingest_oracle as io
    frames = sc.images()
    L, R = frames["frame751"], np.ascontiguousarray(frames["frame752"][:479, :751])
    h, w = L.shape
    pyrs = [hv.pyramid(w, h, 31, 2) for _ in range(2)]
    dev = [torch.from_numpy(a.copy()).cuda() for a in (L, R)]
    torch.cuda.synchronize()
    hv.build_pyramids(pyrs, dev, device=True)
    for p, img in zip(pyrs, (L, R)):
        pts = sc.points(img, (5, 5), seed=9)
        want = orc.refine(img, pts, (5, 5), (-1, -1), (3, 30, 0.01))
        assert_bits(p.subpix_refine(pts), want, "batch build, host call")
        assert_bits(device_refine(hv, p, pts), want, "batch build, device call")
    rng = np.random.RandomState(9)
    table = np.zeros(w * h, io.REMAP_DTYPE)
    table["x0"] = np.clip(np.arange(w * h) % w + rng.randint(-2, 3, w * h), 0, w - 2)
    table["y0"] = np.clip(np.arange(w * h) // w + rng.randint(-2, 3, w * h), 0, h - 2)
    table["xfrac"] = rng.rand(w * h).astype(np.float32); table["yfrac"] = rng.rand(w * h).astype(np.float32)
    table["x0"][rng.rand(w * h) < 0.02] = io.INVALID
    ing = capi.Ingest(hv, w, h)
    ing.set_remap(table)
    gray = ing.frame(L, pyrs[0])
    assert np.array_equal(gray, pyrs[0].download(0)[0])
    pts = sc.points(gray, (7, 7), seed=10)
    want = orc.refine(gray, pts, (7, 7), (1, 2), (3, 30, 0.01))
    assert_bits(pyrs[0].subpix_refine(pts, (7, 7), (1, 2)), want, "ingest, host call")
    assert_bits(device_refine(hv, pyrs[0], pts, (7, 7), (1, 2)), want, "ingest, device call")
    ing.close()
    for p in pyrs:
        p.release()


@pytest.mark.gpu
def test_error_codes(hv):
    import ctypes
    from hybvio_b200 import capi
    lib = capi.load()
    img = sc.images()["texture"]
    h, w = img.shape
    p = pyramid(hv, img)
    xy = np.array([[10, 10], [20, 30]], np.float32)
    ptr = xy.ctypes.data
    other = capi.Context(0)
    q = other.pyramid(w, h, 31, 1)
    small = hv.pyramid(40, 20, 31, 0)
    small.build(np.zeros((20, 40), np.uint8))
    before = hv.launches                    # no call below launches anything
    for f in (lib.hv_subpix_refine, lib.hv_subpix_refine_device):
        assert f(None, p.h, ptr, 2, 5, 5, -1, -1, 3, 30, 0.01) == HV_ERR_INVALID
        assert f(hv.h, None, ptr, 2, 5, 5, -1, -1, 3, 30, 0.01) == HV_ERR_INVALID
        assert f(hv.h, p.h, None, 2, 5, 5, -1, -1, 3, 30, 0.01) == HV_ERR_INVALID
        assert f(hv.h, p.h, ptr, -1, 5, 5, -1, -1, 3, 30, 0.01) == HV_ERR_INVALID
        for win in ((0, 5), (5, 0), (16, 5), (5, 16), (-1, -1)):
            assert f(hv.h, p.h, ptr, 2, win[0], win[1], -1, -1, 3, 30, 0.01) == HV_ERR_UNSUPPORTED, win
        assert f(hv.h, q.h, ptr, 2, 5, 5, -1, -1, 3, 30, 0.01) == HV_ERR_INVALID            # pyramid of another context
        assert f(hv.h, small.h, ptr, 2, 5, 8, -1, -1, 3, 30, 0.01) == HV_ERR_INVALID         # 20 rows < 2 * 8 + 5
        assert f(hv.h, small.h, ptr, 2, 18, 5, -1, -1, 3, 30, 0.01) == HV_ERR_UNSUPPORTED   # the window limit is checked first
    q.release(); other.close(); small.release()
    # the host call checks every corner before launching anything; cv::cornerSubPix asserts on them
    for bad in ([w, 5], [5, h], [-0.001, 5], [5, np.nan]):
        pts = np.array([[10, 10], bad], np.float32)
        keep = pts.copy()
        assert lib.hv_subpix_refine(hv.h, p.h, pts.ctypes.data, 2, 5, 5, -1, -1, 3, 30, 0.01) == HV_ERR_INVALID, bad
        assert np.array_equal(pts, keep, equal_nan=True)
        assert b"outside" in lib.hv_last_error()
    assert hv.launches == before
    p.release()


@pytest.mark.gpu
def test_device_call_leaves_corners_outside_the_image_unchanged(hv, orc):
    img = sc.images()["frame752"]
    h, w = img.shape
    inside = sc.points(img, (5, 5), seed=12)
    outside = np.array([[-0.5, 10], [w, 10], [10, h], [10, -1e-6], [np.nan, 5], [1e9, -1e9]], np.float32)
    pts = np.concatenate([inside[:20], outside, inside[20:]])
    p = pyramid(hv, img)
    got = device_refine(hv, p, pts)
    want = orc.refine(img, inside, (5, 5), (-1, -1), (3, 30, 0.01))
    assert_bits(np.concatenate([got[:20], got[26:]]), want, "inside corners")
    assert np.array_equal(got[20:26].view(np.uint32), outside.view(np.uint32))
    p.release()

