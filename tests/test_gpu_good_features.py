"""Shi-Tomasi corner detection on the device (csrc/good_features.cu): hv_good_features, hv_good_features_device and
hv_good_features_batch_device against the cv::goodFeaturesToTrack oracle (oracle/hv_oracle_good_features.c), bit for bit -- count, order,
(x, y), response and the HV_CORNER_NONE / 0 padding -- on level 0 of pyramids built by hv_pyr_build and by hv_ingest_frame, over the images
of good_features_common (752 x 480 noise at quality 1e-4 gives more candidates than a select round holds), 752 x 480 and 512 x 512
synthetic frames, every mask, min distance, corner budget and quality; capacities equal to and above max_corners with nothing written
past them; batches of 1, 2, 5 and 64 jobs of mixed sizes, budgets and masks against the per-frame calls, with launch counts; every refusal
before anything is launched; and the device chain good_features -> cornerSubPix -> LK over the whole capacity against the same chain fed
the oracle's list from the host."""
import ctypes

import numpy as np
import pytest

import good_features_common as gc
from hybvio_b200 import capi, synth
from oracle import good_features_oracle

HV_ERR_INVALID, HV_ERR_UNSUPPORTED = -1, -5
NONE = np.float32(-1.0e6)          # HV_CORNER_NONE
SENT = 777.0


@pytest.fixture(scope="module")
def orc(oracle_lk):
    return good_features_oracle.OracleGoodFeatures()


@pytest.fixture(scope="module")
def imgs():
    d = gc.images(large_noise=(480, 752))
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


def _device_buffers(slots):
    import torch
    return (torch.full((slots, 2), SENT, dtype=torch.float32, device="cuda"), torch.full((1,), -1, dtype=torch.int32, device="cuda"),
            torch.full((slots,), SENT, dtype=torch.float32, device="cuda"))


def _device_mask(mask):
    """The mask as a CUDA view whose row stride exceeds its width (None stays None)."""
    import torch
    if mask is None:
        return None
    h, w = mask.shape
    buf = torch.full((h, w + 13), 0xAB, dtype=torch.uint8, device="cuda")
    buf[:, :w] = torch.from_numpy(mask).cuda()
    return buf[:, :w]


def _check_device(xy, cnt, resp, cap, want, what):
    xy, resp, n = xy.cpu().numpy(), resp.cpu().numpy(), int(cnt.cpu().numpy()[0])
    assert n == len(want), f"{what}: count {n} vs oracle {len(want)}"
    _bits(xy[:n], want[:, :2], what + " xy")
    _bits(resp[:n], want[:, 2], what + " response")
    assert np.all(xy[n:cap].view(np.uint32) == NONE.view(np.uint32)), what + " xy padding"
    assert np.all(resp[n:cap] == 0.0), what + " response padding"
    assert np.all(xy[cap:] == SENT) and np.all(resp[cap:] == SENT), what + " written past the capacity"


def _budgets(orc, img, q, md, mask):
    """max_corners 1, 150 and one above the candidate count"""
    return (1, 150, len(orc.detect(img, 1 << 30, q, md, mask)) + 7)


@pytest.mark.gpu
@pytest.mark.parametrize("mask_kind", gc.MASKS)
def test_device_equals_oracle(hv, orc, imgs, mask_kind):
    longest = 0
    for name, img in imgs.items():
        pyr = _pyr(hv, img)
        mask = gc.mask_for(mask_kind, img, orc.eig(img))
        d_mask = _device_mask(mask)
        for q in gc.QUALITIES:
            for md in gc.MIN_DISTANCES:
                for mc in _budgets(orc, img, q, md, mask):
                    want = orc.detect(img, mc, q, md, mask)
                    longest = max(longest, len(want))
                    what = f"{name} mask {mask_kind} q {q} md {md} max {mc}"
                    cap = mc + (0 if mc == 1 else 5)         # the wrapper passes the buffer's length as the capacity
                    d_xy, d_cnt, d_resp = _device_buffers(cap)
                    before = hv.launches
                    pyr.good_features_device(d_xy, d_cnt, mc, q, md, d_resp, d_mask)
                    assert hv.launches == before + 3
                    hv.sync()
                    _check_device(d_xy, d_cnt, d_resp, cap, want, what + " device")
                    if md in (0.0, 10.0) and mc != 1:
                        xy, resp = pyr.good_features(mc, q, md, mask)
                        _bits(xy, want[:, :2], what + " host xy")
                        _bits(resp, want[:, 2], what + " host response")
        pyr.release()
    assert longest > 8192, "no list longer than one select round"


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
        for q, md, mc in ((0.01, 10.0, 150), (1e-4, 0.0, 100000), (0.01, 2.5, 1000)):
            want = orc.detect(gray, mc, q, md)
            xy, resp = pyr.good_features(mc, q, md)
            _bits(xy, want[:, :2], f"ingest {w}x{h} q {q} md {md} xy")
            _bits(resp, want[:, 2], f"ingest {w}x{h} q {q} md {md} response")
        pyr.release()
        ing.close()


@pytest.mark.gpu
def test_capacities(hv, orc, imgs):
    """capacity == max_corners and above it, on the device and through the host call; a NULL response buffer is never written."""
    import torch
    img = imgs["frame752"]
    pyr = _pyr(hv, img)
    for md in (0.0, 10.0):
        for mc in (1, 150, 4000):
            want = orc.detect(img, mc, 0.01, md)
            for cap in (mc, mc + 1, mc + 100):
                what = f"md {md} max {mc} capacity {cap}"
                d_xy, d_cnt, d_resp = _device_buffers(cap + 2)
                assert hv.lib.hv_good_features_device(hv.h, pyr.h, 3, mc, 0.01, md, None, 0, d_xy.data_ptr(), d_resp.data_ptr(), cap,
                                                      d_cnt.data_ptr()) == 0
                hv.sync()
                _check_device(d_xy, d_cnt, d_resp, cap, want, what)
                d_resp.fill_(SENT)
                torch.cuda.synchronize()
                assert hv.lib.hv_good_features_device(hv.h, pyr.h, 3, mc, 0.01, md, None, 0, d_xy.data_ptr(), None, cap,
                                                      d_cnt.data_ptr()) == 0
                hv.sync()
                assert np.all(d_resp.cpu().numpy() == SENT), what + " NULL response written"
                xy = np.full((cap + 2, 2), SENT, np.float32)
                resp = np.full(cap + 2, SENT, np.float32)
                cnt = ctypes.c_int(-1)
                assert hv.lib.hv_good_features(hv.h, pyr.h, 3, mc, 0.01, md, None, 0, xy.ctypes.data, resp.ctypes.data, cap, ctypes.byref(cnt)) == 0
                n = cnt.value
                assert n == len(want), what + " host count"
                _bits(xy[:n], want[:, :2], what + " host")
                _bits(resp[:n], want[:, 2], what + " host response")
                assert np.all(xy[n:cap].view(np.uint32) == NONE.view(np.uint32)) and np.all(resp[n:cap] == 0.0), what + " host padding"
                assert np.all(xy[cap:] == SENT) and np.all(resp[cap:] == SENT), what + " host past the capacity"
    pyr.release()


SIZES = [(752, 480), (512, 512), (751, 479), (333, 241), (2, 2), (97, 61), (1280, 720), (3, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("md", [0.0, 10.0])
@pytest.mark.parametrize("S", [1, 2, 5, 64])
def test_batch_equals_per_frame_calls(hv, orc, S, md):
    import torch
    q = 0.01
    frames, masks, pyrs, single, batch, caps, budgets = [], [], [], [], [], [], []
    for j in range(S):
        w, h = SIZES[j % len(SIZES)]
        img = synth.stereo_frame(j + 1, w, h)[j % 2]
        frames.append(img)
        masks.append(gc.mask_for(("none", "half", "hide_max")[j % 3], img, orc.eig(img)))
        pyrs.append(_pyr(hv, img))
        mc = (150, 1, 40, 100000)[j % 4]
        budgets.append(mc)
        caps.append(mc + (0, 9)[j % 2] if mc < 100000 else mc)
        single.append(_device_buffers(caps[-1] + 2))
        batch.append(_device_buffers(caps[-1] + 2))
    d_masks = [_device_mask(m) for m in masks]
    torch.cuda.synchronize()
    lib = hv.lib
    for p, (xy, cnt, resp), cap, mc, dm in zip(pyrs, single, caps, budgets, d_masks):
        mp, ms = (None, 0) if dm is None else (dm.data_ptr(), dm.stride(0))
        assert lib.hv_good_features_device(hv.h, p.h, 3, mc, q, md, mp, ms, xy.data_ptr(), resp.data_ptr(), cap, cnt.data_ptr()) == 0
    jobs = []
    for j, (p, (xy, cnt, resp), cap, mc, dm) in enumerate(zip(pyrs, batch, caps, budgets, d_masks)):
        mp, ms = (None, 0) if dm is None else (dm.data_ptr(), dm.stride(0))
        jobs.append(capi.GoodFeaturesJob(p.h.value, mc, mp, ms, xy.data_ptr(), resp.data_ptr() if j % 4 != 3 else None, cap, cnt.data_ptr()))
    before = hv.launches
    hv.good_features_batch_device(jobs, q, md)
    assert hv.launches == before + 3
    hv.sync()
    for j in range(S):
        what = f"S {S} job {j} {frames[j].shape} max {budgets[j]} capacity {caps[j]}"
        xs, cs, rs = (a.cpu().numpy() for a in single[j])
        xb, cb, rb = (a.cpu().numpy() for a in batch[j])
        assert xb.tobytes() == xs.tobytes() and cb.tobytes() == cs.tobytes(), what
        if j % 4 != 3:
            assert rb.tobytes() == rs.tobytes(), what + " response"
        else:
            assert np.all(rb == SENT), what + " NULL response written"
        _check_device(*single[j], caps[j], orc.detect(frames[j], budgets[j], q, md, masks[j]), what + " per frame vs oracle")
    for p in pyrs:
        p.release()


@pytest.mark.gpu
def test_refusals(hv, imgs):
    import torch
    lib = hv.lib
    img = imgs["frame752"]
    h, w = img.shape
    pyr = _pyr(hv, img)
    other = capi.Context(0)
    opyr = _pyr(other, img)
    xy, cnt, resp = _device_buffers(100)
    d_mask = torch.ones((h, w), dtype=torch.uint8, device="cuda")
    host_xy = np.full((100, 2), SENT, np.float32)
    host_cnt = ctypes.c_int(-1)
    host_mask = np.ones((h, w), np.uint8)
    before = hv.launches
    X, R, N, M = xy.data_ptr(), resp.data_ptr(), cnt.data_ptr(), d_mask.data_ptr()
    for f, x, n, m in ((lib.hv_good_features_device, X, N, M), (lib.hv_good_features, host_xy.ctypes.data, ctypes.addressof(host_cnt), host_mask.ctypes.data)):
        call = lambda c=hv.h, p=pyr.h, bs=3, mc=50, q=0.01, md=10.0, mk=m, ms=w, xx=x, cap=100, nn=n: f(c, p, bs, mc, q, md, mk, ms, xx, R if f is lib.hv_good_features_device else None, cap, nn)
        for rc, kw in ((HV_ERR_INVALID, dict(c=None)), (HV_ERR_INVALID, dict(p=None)), (HV_ERR_INVALID, dict(p=opyr.h)),
                       (HV_ERR_INVALID, dict(xx=None)), (HV_ERR_INVALID, dict(nn=None)), (HV_ERR_INVALID, dict(cap=49)),
                       (HV_ERR_INVALID, dict(q=0.0)), (HV_ERR_INVALID, dict(q=-0.5)), (HV_ERR_INVALID, dict(q=float("nan"))),
                       (HV_ERR_INVALID, dict(md=-1.0)), (HV_ERR_INVALID, dict(md=float("nan"))), (HV_ERR_INVALID, dict(md=float("inf"))),
                       (HV_ERR_INVALID, dict(ms=w - 1)),
                       (HV_ERR_UNSUPPORTED, dict(bs=5)), (HV_ERR_UNSUPPORTED, dict(mc=0)), (HV_ERR_UNSUPPORTED, dict(mc=-3, cap=100))):
            assert call(**kw) == rc, f"{f.__name__} {kw}"
    good = capi.GoodFeaturesJob(pyr.h.value, 50, M, w, X, R, 100, N)
    bad_jobs = [[good, capi.GoodFeaturesJob(pyr.h.value, 50, M, w, X, R, 49, N)], [good, capi.GoodFeaturesJob(opyr.h.value, 50, M, w, X, R, 100, N)],
                [capi.GoodFeaturesJob(None, 50, M, w, X, R, 100, N), good], [good, capi.GoodFeaturesJob(pyr.h.value, 50, M, w, None, R, 100, N)],
                [good, capi.GoodFeaturesJob(pyr.h.value, 50, M, w, X, R, 100, None)], [good, capi.GoodFeaturesJob(pyr.h.value, 50, M, w - 1, X, R, 100, N)]]
    for jobs in bad_jobs:
        J = (capi.GoodFeaturesJob * len(jobs))(*jobs)
        assert lib.hv_good_features_batch_device(hv.h, J, len(jobs), 3, 0.01, 10.0) == HV_ERR_INVALID
    J = (capi.GoodFeaturesJob * 2)(good, capi.GoodFeaturesJob(pyr.h.value, 0, M, w, X, R, 100, N))
    assert lib.hv_good_features_batch_device(hv.h, J, 2, 3, 0.01, 10.0) == HV_ERR_UNSUPPORTED
    J = (capi.GoodFeaturesJob * 65)(*([good] * 65))
    assert lib.hv_good_features_batch_device(hv.h, J, 65, 3, 0.01, 10.0) == HV_ERR_INVALID
    assert lib.hv_good_features_batch_device(hv.h, J, 0, 3, 0.01, 10.0) == HV_ERR_INVALID
    assert lib.hv_good_features_batch_device(hv.h, None, 1, 3, 0.01, 10.0) == HV_ERR_INVALID
    assert lib.hv_good_features_batch_device(None, J, 1, 3, 0.01, 10.0) == HV_ERR_INVALID
    assert lib.hv_good_features_batch_device(hv.h, J, 1, 5, 0.01, 10.0) == HV_ERR_UNSUPPORTED
    assert lib.hv_good_features_batch_device(hv.h, J, 1, 3, 0.0, 10.0) == HV_ERR_INVALID
    assert lib.hv_good_features_batch_device(hv.h, J, 1, 3, 0.01, -2.0) == HV_ERR_INVALID
    assert lib.hv_good_features_batch_device(hv.h, J, 1, 3, 0.01, float("inf")) == HV_ERR_INVALID
    torch.cuda.synchronize()
    assert hv.launches == before, "a refused call launched"
    assert np.all(xy.cpu().numpy() == SENT) and np.all(resp.cpu().numpy() == SENT) and int(cnt.cpu().numpy()[0]) == -1
    assert np.all(host_xy == SENT) and host_cnt.value == -1
    opyr.release(); other.close(); pyr.release()


@pytest.mark.gpu
@pytest.mark.parametrize("md", [0.0, 10.0])
def test_chain_into_subpix_and_lk(hv, orc, md):
    """good_features_device -> subpix_refine_device -> lk_track_device over the whole capacity (the padding included), compared with
    the same chain fed the oracle's list (padded the same way) from the host."""
    import torch
    L0, _ = synth.stereo_frame(0, 752, 480)
    L1, _ = synth.stereo_frame(1, 752, 480)
    p0, p1 = _pyr(hv, L0, 3), _pyr(hv, L1, 3)
    mc = 300
    want = orc.detect(L0, mc, 0.01, md)
    cap = mc + 37
    outs = []
    for source in ("device", "oracle"):
        if source == "device":
            d_xy = torch.full((cap, 2), SENT, dtype=torch.float32, device="cuda")
            d_cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
            p0.good_features_device(d_xy, d_cnt, mc, 0.01, md)
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
        assert a.tobytes() == b.tobytes(), f"md {md}: {what} differs"
    assert outs[0][2][:len(want)].sum() > len(want) // 2 and not outs[0][2][len(want):].any()
    p0.release(); p1.release()


@pytest.mark.gpu
def test_python_mask_shape(hv, imgs):
    """The Python wrappers refuse a mask that is not level 0's (h, w) before the C call can read past it."""
    import torch
    img = imgs["frame752"]
    h, w = img.shape
    pyr = _pyr(hv, img)
    d_xy, d_cnt, d_resp = _device_buffers(150)
    for shape in ((h - 1, w), (h, w - 1), (h + 1, w)):
        with pytest.raises(ValueError):
            pyr.good_features(150, 0.01, 10.0, np.ones(shape, np.uint8))
        with pytest.raises(ValueError):
            pyr.good_features_device(d_xy, d_cnt, 150, 0.01, 10.0, d_resp, torch.ones(shape, dtype=torch.uint8, device="cuda"))
        with pytest.raises(ValueError):
            capi.good_features_job(pyr, d_xy, d_cnt, 150, d_resp, torch.ones(shape, dtype=torch.uint8, device="cuda"))
    with pytest.raises(ValueError):
        pyr.good_features_device(d_xy, d_cnt, 150, 0.01, 10.0, d_resp, torch.ones((h, w), dtype=torch.int32, device="cuda"))
    pyr.release()
