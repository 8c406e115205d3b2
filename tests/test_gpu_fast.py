"""FAST corner detection on the device (csrc/fast.cu): hv_fast_detect, hv_fast_detect_device and hv_fast_detect_batch_device against the
cv::FAST oracle (oracle/hv_oracle_fast.c), bit for bit -- count, order, (x, y), response and the HV_CORNER_NONE / 0 padding -- on level 0
of pyramids built by hv_pyr_build and by hv_ingest_frame, over the images of fast_common (752 x 480, odd widths, images smaller than
7 x 7, ...) and 512 x 512, every threshold of fast_common, with and without suppression; capacities of 0, below and above the count;
batches of 1, 2, 5 and 64 mixed sizes against the per-frame calls, with launch counts; every refusal before anything is launched; and
the device chain fast -> cornerSubPix -> LK over the whole capacity against the same chain fed the oracle's list from the host."""
import ctypes

import numpy as np
import pytest

import fast_common as fc
from hybvio_b200 import capi, synth
from oracle import fast_oracle

HV_ERR_INVALID = -1
NONE = np.float32(-1.0e6)          # HV_CORNER_NONE
SENT = 777.0


@pytest.fixture(scope="module")
def orc(oracle_lk):
    return fast_oracle.OracleFast()


@pytest.fixture(scope="module")
def imgs():
    d = fc.images()
    d["frame512"] = synth.stereo_frame(7, 512, 512)[0]
    return d


def _pyr(hv, img, levels=0):
    p = hv.pyramid(img.shape[1], img.shape[0], 31, levels)
    p.build(np.ascontiguousarray(img))
    return p


def _bits(a, b, what):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    assert a.shape == b.shape, f"{what}: shape {a.shape} vs {b.shape}"
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), f"{what}: first difference at {np.nonzero((a != b).reshape(len(a), -1).any(axis=1))[0][:5]}"


def _device_buffers(cap):
    import torch
    return (torch.full((max(cap, 1), 2), SENT, dtype=torch.float32, device="cuda"), torch.full((1,), -1, dtype=torch.int32, device="cuda"),
            torch.full((max(cap, 1),), SENT, dtype=torch.float32, device="cuda"))


def _check_device(xy, cnt, resp, cap, want, what):
    xy, resp, n = xy.cpu().numpy(), resp.cpu().numpy(), int(cnt.cpu().numpy()[0])
    assert n == len(want), f"{what}: count {n} vs oracle {len(want)}"
    m = min(n, cap)
    _bits(xy[:m], want[:m, :2], what + " xy")
    _bits(resp[:m], want[:m, 2], what + " response")
    assert np.all(xy[m:cap].view(np.uint32) == NONE.view(np.uint32)), what + " xy padding"
    assert np.all(resp[m:cap] == 0.0), what + " response padding"
    assert np.all(xy[cap:] == SENT) and np.all(resp[cap:] == SENT), what + " written past the capacity"


@pytest.mark.gpu
@pytest.mark.parametrize("nonmax", [True, False], ids=["nms", "all"])
def test_device_equals_oracle(hv, orc, imgs, nonmax):
    for name, img in imgs.items():
        pyr = _pyr(hv, img)
        for t in fc.THRESHOLDS:
            want = orc.detect(img, t, nonmax)
            what = f"{name} t {t} nonmax {nonmax}"
            xy, resp = pyr.fast_detect(t, nonmax)
            _bits(xy, want[:, :2], what + " host xy")
            _bits(resp, want[:, 2], what + " host response")
            cap = len(want) + 5
            d_xy, d_cnt, d_resp = _device_buffers(cap + 3)
            before = hv.launches
            check = hv.lib.hv_fast_detect_device(hv.h, pyr.h, t, int(nonmax), d_xy.data_ptr(), d_resp.data_ptr(), cap, d_cnt.data_ptr())
            assert check == 0 and hv.launches == before + 2
            hv.sync()
            _check_device(d_xy, d_cnt, d_resp, cap, want, what + " device")
        pyr.release()


@pytest.mark.gpu
def test_ingested_pyramids(hv, orc):
    """Level 0 written by hv_ingest_frame from colour frames (its own level-0 pitch at widths that are no multiple of 4)."""
    rng = np.random.RandomState(3)
    for w, h in ((752, 480), (333, 241), (61, 37)):
        bgr = np.stack([synth.stereo_frame(j, w, h)[0] for j in range(3)], axis=2)
        bgr[..., 1] = rng.randint(0, 256, (h, w))
        ing = capi.Ingest(hv, w, h)
        pyr = hv.pyramid(w, h, 31, 2)
        gray = ing.frame(bgr, pyr)
        for t in (0, 10, 20):
            for nonmax in (True, False):
                want = orc.detect(gray, t, nonmax)
                xy, resp = pyr.fast_detect(t, nonmax)
                _bits(xy, want[:, :2], f"ingest {w}x{h} t {t} {nonmax} xy")
                _bits(resp, want[:, 2], f"ingest {w}x{h} t {t} {nonmax} response")
        pyr.release()
        ing.close()


@pytest.mark.gpu
def test_capacities(hv, orc, imgs):
    img = imgs["frame752"]
    pyr = _pyr(hv, img)
    for nonmax in (True, False):
        want = orc.detect(img, 10, nonmax)
        n = len(want)
        for cap in (0, 1, n // 2, n - 1, n, n + 1, n + 100):
            what = f"capacity {cap} of {n} nonmax {nonmax}"
            d_xy, d_cnt, d_resp = _device_buffers(cap + 2)
            assert hv.lib.hv_fast_detect_device(hv.h, pyr.h, 10, int(nonmax), d_xy.data_ptr(), d_resp.data_ptr(), cap, d_cnt.data_ptr()) == 0
            hv.sync()
            _check_device(d_xy, d_cnt, d_resp, cap, want, what)
            # the host call: capacity slots, the full count
            xy = np.full((cap + 2, 2), SENT, np.float32)
            cnt = ctypes.c_int(-1)
            assert hv.lib.hv_fast_detect(hv.h, pyr.h, 10, int(nonmax), xy.ctypes.data if cap else None, None, cap, ctypes.byref(cnt)) == 0
            assert cnt.value == n
            m = min(n, cap)
            _bits(xy[:m], want[:m, :2], what + " host")
            assert np.all(xy[m:cap].view(np.uint32) == NONE.view(np.uint32)) and np.all(xy[cap:] == SENT), what + " host padding"
        xy, resp = pyr.fast_detect(10, nonmax, capacity=7)
        _bits(xy, want[:7, :2], "Pyramid.fast_detect capacity 7")
    pyr.release()


SIZES = [(752, 480), (512, 512), (751, 479), (333, 241), (6, 6), (97, 61), (1280, 720), (7, 7)]


@pytest.mark.gpu
@pytest.mark.parametrize("nonmax", [True, False], ids=["nms", "all"])
@pytest.mark.parametrize("S", [1, 2, 5, 64])
def test_batch_equals_per_frame_calls(hv, orc, S, nonmax):
    import torch
    t = 12
    frames, pyrs, single, batch, caps = [], [], [], [], []
    for j in range(S):
        w, h = SIZES[j % len(SIZES)]
        img = synth.stereo_frame(j + 1, w, h)[j % 2]
        frames.append(img)
        pyrs.append(_pyr(hv, img))
        n = len(orc.detect(img, t, nonmax))
        cap = (n + 9, n // 2, 0)[j % 3]
        caps.append(cap)
        single.append(_device_buffers(cap + 2))
        batch.append(_device_buffers(cap + 2))
    torch.cuda.synchronize()
    for p, (xy, cnt, resp), cap in zip(pyrs, single, caps):
        assert hv.lib.hv_fast_detect_device(hv.h, p.h, t, int(nonmax), xy.data_ptr(), resp.data_ptr(), cap, cnt.data_ptr()) == 0
    jobs = [capi.FastJob(p.h.value, xy.data_ptr(), resp.data_ptr() if j % 4 != 3 else None, cap, cnt.data_ptr())
            for j, (p, (xy, cnt, resp), cap) in enumerate(zip(pyrs, batch, caps))]
    before = hv.launches
    hv.fast_detect_batch_device(jobs, t, nonmax)
    assert hv.launches == before + 2
    hv.sync()
    for j in range(S):
        what = f"S {S} job {j} {frames[j].shape} capacity {caps[j]}"
        xs, cs, rs = (a.cpu().numpy() for a in single[j])
        xb, cb, rb = (a.cpu().numpy() for a in batch[j])
        assert xb.tobytes() == xs.tobytes() and cb.tobytes() == cs.tobytes(), what
        if j % 4 != 3:
            assert rb.tobytes() == rs.tobytes(), what + " response"
        else:
            assert np.all(rb == SENT), what + " NULL response written"
        _check_device(*single[j], caps[j], orc.detect(frames[j], t, nonmax), what + " per frame vs oracle")
    for p in pyrs:
        p.release()


@pytest.mark.gpu
def test_refusals(hv, imgs):
    import torch
    lib = hv.lib
    img = imgs["frame752"]
    pyr = _pyr(hv, img)
    other = capi.Context(0)
    opyr = _pyr(other, img)
    xy, cnt, resp = _device_buffers(100)
    host_xy = np.full((100, 2), SENT, np.float32)
    host_cnt = ctypes.c_int(-1)
    before = hv.launches
    dev = lambda c, p, x, r, cap, n: lib.hv_fast_detect_device(c, p, 10, 1, x, r, cap, n)
    hst = lambda c, p, x, r, cap, n: lib.hv_fast_detect(c, p, 10, 1, x, r, cap, n)
    X, R, N = xy.data_ptr(), resp.data_ptr(), cnt.data_ptr()
    for f, x, n in ((dev, X, N), (hst, host_xy.ctypes.data, ctypes.addressof(host_cnt))):
        assert f(None, pyr.h, x, R, 100, n) == HV_ERR_INVALID
        assert f(hv.h, None, x, R, 100, n) == HV_ERR_INVALID
        assert f(hv.h, opyr.h, x, R, 100, n) == HV_ERR_INVALID          # a pyramid of another context
        assert f(hv.h, pyr.h, x, R, -1, n) == HV_ERR_INVALID
        assert f(hv.h, pyr.h, None, R, 100, n) == HV_ERR_INVALID
        assert f(hv.h, pyr.h, x, R, 100, None) == HV_ERR_INVALID
    good = capi.FastJob(pyr.h.value, X, R, 100, N)
    bad_jobs = [[good, capi.FastJob(pyr.h.value, X, R, -3, N)], [good, capi.FastJob(opyr.h.value, X, R, 100, N)],
                [capi.FastJob(None, X, R, 100, N), good], [good, capi.FastJob(pyr.h.value, None, R, 100, N)],
                [good, capi.FastJob(pyr.h.value, X, R, 100, None)]]
    for jobs in bad_jobs:
        J = (capi.FastJob * len(jobs))(*jobs)
        assert lib.hv_fast_detect_batch_device(hv.h, J, len(jobs), 10, 1) == HV_ERR_INVALID
    J = (capi.FastJob * 65)(*([good] * 65))
    assert lib.hv_fast_detect_batch_device(hv.h, J, 65, 10, 1) == HV_ERR_INVALID
    assert lib.hv_fast_detect_batch_device(hv.h, J, 0, 10, 1) == HV_ERR_INVALID
    assert lib.hv_fast_detect_batch_device(hv.h, None, 1, 10, 1) == HV_ERR_INVALID
    assert lib.hv_fast_detect_batch_device(None, J, 1, 10, 1) == HV_ERR_INVALID
    torch.cuda.synchronize()
    assert hv.launches == before, "a refused call launched"
    assert np.all(xy.cpu().numpy() == SENT) and np.all(resp.cpu().numpy() == SENT) and int(cnt.cpu().numpy()[0]) == -1
    assert np.all(host_xy == SENT) and host_cnt.value == -1
    opyr.release(); other.close(); pyr.release()


@pytest.mark.gpu
@pytest.mark.parametrize("nonmax", [True, False], ids=["nms", "all"])
def test_chain_into_subpix_and_lk(hv, orc, nonmax):
    """fast_detect_device -> subpix_refine_device -> lk_track_device over the whole capacity (the padding included), compared with the
    same chain fed the oracle's list (padded the same way) from the host."""
    import torch
    L0, _ = synth.stereo_frame(0, 752, 480)
    L1, _ = synth.stereo_frame(1, 752, 480)
    p0, p1 = _pyr(hv, L0, 3), _pyr(hv, L1, 3)
    want = orc.detect(L0, 20, nonmax)
    cap = len(want) + 37
    outs = []
    for source in ("device", "oracle"):
        if source == "device":
            d_xy = torch.full((cap, 2), SENT, dtype=torch.float32, device="cuda")
            d_cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
            p0.fast_detect_device(d_xy, d_cnt, None, 20, nonmax)
        else:
            h_xy = np.full((cap, 2), NONE, np.float32)
            h_xy[:len(want)] = want[:, :2]
            d_xy = torch.from_numpy(h_xy).cuda()
        p0.subpix_refine_device(d_xy)
        d_next = torch.zeros((cap, 2), dtype=torch.float32, device="cuda")
        d_st = torch.zeros(cap, dtype=torch.uint8, device="cuda")
        d_ts = torch.zeros(cap, dtype=torch.int32, device="cuda")
        hv.lk_track_device(p0, p1, d_xy.data_ptr(), d_next.data_ptr(), d_st.data_ptr(), d_ts.data_ptr(), cap, False)
        hv.sync()
        outs.append([t.cpu().numpy() for t in (d_xy, d_next, d_st, d_ts)])
    for a, b, what in zip(outs[0], outs[1], ("refined", "tracked", "status", "track status")):
        assert a.tobytes() == b.tobytes(), f"nonmax {nonmax}: {what} differs"
    assert outs[0][2][:len(want)].sum() > len(want) // 2 and not outs[0][2][len(want):].any()
    p0.release(); p1.release()
