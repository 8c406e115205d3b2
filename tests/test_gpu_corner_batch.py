"""The new-corner step of many sessions in one launch per step: hv_gftt_detect_batch_device, hv_gftt_select_batch_device and
hv_subpix_refine_batch_device (csrc/gftt.cu, gftt_select.cu, subpix.cu) against the per-session calls on the same context -- key
points, corner lists, counts, padding and refined points BYTE-identical, the lists equal to orc_gftt_corners (oracle/hv_oracle_gftt.c)
-- over mixed frame sizes, radii, max_tracks, previous corners and spare capacity; an image smaller than a cell; the whole chain into
hv_lk_track_batch_device; one launch per call; and every refusal before anything is launched."""
import ctypes

import numpy as np
import pytest

import gftt_select_common as gc
from hybvio_b200 import capi, synth
from oracle import gftt_oracle

HV_ERR_INVALID, HV_ERR_UNSUPPORTED = -1, -5
SIZES = [(752, 480), (512, 512), (751, 479)]
RADII = [0, 8, 50]
MAX_TRACKS = [150, 7, 100000]
SENT = 7.0


@pytest.fixture(scope="module")
def orc(oracle_lk):
    return gftt_oracle.OracleGftt()


class Session:
    """One session's frame, pyramid(s) and the buffers of the per-session ("s") and batched ("b") calls, all sentinel-filled."""

    def __init__(self, hv, j, cell, size=None, levels=1, stereo=False):
        import torch
        self.w, self.h = size or SIZES[j % 3]
        self.r, self.m = RADII[(j // 3) % 3], MAX_TRACKS[(j + j // 9) % 3]
        self.img, right = synth.stereo_frame(j + 1, self.w, self.h)
        self.pyr = hv.pyramid(self.w, self.h, 31, levels)
        self.pyr.build(np.ascontiguousarray(self.img))
        if stereo:
            self.right = hv.pyramid(self.w, self.h, 31, levels)
            self.right.build(np.ascontiguousarray(right))
        self.prev = gc.prev_points(100 if j % 2 else 0, 50 + j, self.w, self.h)
        self.nkp = int(np.prod(self.pyr.gftt_cells(cell)))
        self.cap = max(gc.capacity(self.nkp, self.r, self.m) + j % 4, 1)
        self.d_prev = torch.from_numpy(self.prev).cuda() if len(self.prev) else None
        self.buf = {}
        for k in "sb":
            self.buf[k] = (torch.full((max(self.nkp, 1), 3), SENT, dtype=torch.float32, device="cuda"),
                           torch.full((self.cap, 2), SENT, dtype=torch.float32, device="cuda"),
                           torch.full((1,), -1, dtype=torch.int32, device="cuda"))

    def job(self, k="b"):
        kp, cor, cnt = self.buf[k]
        return capi.corner_job(self.pyr, kp, cor, cnt, self.d_prev, self.r, self.m, nkp=self.nkp)

    def per_session_detect_select(self, hv, cell):
        kp, cor, cnt = self.buf["s"]
        self.pyr.gftt_detect_device(kp.data_ptr(), 3, cell, 1e-3)
        hv.lib.hv_gftt_select_device(hv.h, kp.data_ptr(), self.nkp, capi._ptr(self.d_prev), len(self.prev), self.r, self.m,
                                     cor.data_ptr(), self.cap, cnt.data_ptr())

    def host(self, k):
        return [t.cpu().numpy() for t in self.buf[k]]

    def release(self):
        self.pyr.release()
        if hasattr(self, "right"):
            self.right.release()


def _same(a, b, what):
    assert a.shape == b.shape and a.tobytes() == b.tobytes(), f"{what}: differs"


def _step(hv, fn, *args):
    before = hv.launches
    fn(*args)
    assert hv.launches == before + 1, f"{fn.__name__}: {hv.launches - before} launches"


@pytest.mark.gpu
@pytest.mark.parametrize("cell", [32, 8])
@pytest.mark.parametrize("S", [1, 2, 5, 16, 64])
def test_batch_equals_per_session_calls(hv, orc, S, cell):
    import torch
    ss = [Session(hv, j, cell) for j in range(S)]
    torch.cuda.synchronize()
    for s in ss:
        s.per_session_detect_select(hv, cell)
    jobs = [s.job() for s in ss]
    _step(hv, hv.gftt_detect_batch_device, jobs, 3, cell, 1e-3)
    _step(hv, hv.gftt_select_batch_device, jobs)
    hv.sync()
    for j, s in enumerate(ss):
        what = f"S {S} cell {cell} job {j} {s.w}x{s.h} r {s.r} max {s.m} nprev {len(s.prev)} cap {s.cap}"
        (kp_s, cor_s, cnt_s), (kp_b, cor_b, cnt_b) = s.host("s"), s.host("b")
        _same(kp_b, kp_s, what + " key points")
        _same(cnt_b, cnt_s, what + " count")
        _same(cor_b, cor_s, what + " corners and padding")
        n = int(cnt_b[0])
        want = orc.corners(orc.collect(orc.response(s.img), cell, 1e-3), s.prev, s.r, s.m)
        _same(cor_b[:n], want, what + " list vs oracle")
        assert np.all(cor_b[n:].view(np.uint32) == gc.NONE.view(np.uint32)), what + " padding"
    # refinement over the whole capacity (padding included), per session and batched
    for s in ss:
        s.pyr.subpix_refine_device(s.buf["s"][1])
    _step(hv, hv.subpix_refine_batch_device, [capi.subpix_job(s.pyr, s.buf["b"][1]) for s in ss])
    hv.sync()
    for j, s in enumerate(ss):
        _same(s.host("b")[1], s.host("s")[1], f"S {S} cell {cell} job {j} refined points")
    for s in ss:
        s.release()


@pytest.mark.gpu
def test_image_smaller_than_a_cell(hv):
    import torch
    ss = [Session(hv, 0, 32), Session(hv, 1, 32, size=(20, 24)), Session(hv, 2, 32)]
    small = ss[1]
    assert small.nkp == 0
    torch.cuda.synchronize()
    jobs = [s.job() for s in ss]
    _step(hv, hv.gftt_detect_batch_device, jobs, 3, 32, 1e-3)
    _step(hv, hv.gftt_select_batch_device, jobs)
    hv.sync()
    kp, cor, cnt = small.host("b")
    assert int(cnt[0]) == 0 and np.all(kp == SENT)                      # no cell: no key point written
    assert np.all(cor.view(np.uint32) == gc.NONE.view(np.uint32))
    for s in (ss[0], ss[2]):
        assert int(s.host("b")[2][0]) > 0
    # a batch of images without a cell launches nothing
    before = hv.launches
    hv.gftt_detect_batch_device([small.job()], 3, 32, 1e-3)
    assert hv.launches == before
    for s in ss:
        s.release()


def _lk_jobs(ss, k, nxt, st, ts):
    return [capi.LkJob(s.pyr.h.value, s.right.h.value, s.buf[k][1].data_ptr(), nxt[j].data_ptr(), st[j].data_ptr(), ts[j].data_ptr(),
                       s.cap, 0) for j, s in enumerate(ss)]


@pytest.mark.gpu
def test_chain_into_lk_batch_for_eleven_sessions(hv):
    """detect -> select -> refine -> stereo LK over every session's capacity: batched (3 + 2 launches) against 11 per-session chains."""
    import torch
    S = 11
    ss = [Session(hv, j, 32, levels=3, stereo=True) for j in range(S)]
    out = {k: ([torch.full((s.cap, 2), SENT, dtype=torch.float32, device="cuda") for s in ss],
               [torch.full((s.cap,), 9, dtype=torch.uint8, device="cuda") for s in ss],
               [torch.full((s.cap,), 9, dtype=torch.int32, device="cuda") for s in ss]) for k in "sb"}
    torch.cuda.synchronize()
    for j, s in enumerate(ss):
        s.per_session_detect_select(hv, 32)
        s.pyr.subpix_refine_device(s.buf["s"][1])
        nxt, st, ts = (x[j] for x in out["s"])
        hv.lk_track_device(s.pyr, s.right, s.buf["s"][1], nxt, st, ts, s.cap, False)
    jobs = [s.job() for s in ss]
    before = hv.launches
    hv.gftt_detect_batch_device(jobs, 3, 32, 1e-3)
    hv.gftt_select_batch_device(jobs)
    hv.subpix_refine_batch_device([capi.subpix_job(s.pyr, s.buf["b"][1]) for s in ss])
    L = (capi.LkJob * S)(*_lk_jobs(ss, "b", *out["b"]))
    capi.check(hv.lib.hv_lk_track_batch_device(hv.h, L, S, 20, 0.03, 1e-3), "hv_lk_track_batch_device")
    assert hv.launches - before == 3 + 2
    hv.sync()
    for j, s in enumerate(ss):
        for i, name in enumerate(("end points", "status", "track status")):
            _same(out["b"][i][j].cpu().numpy(), out["s"][i][j].cpu().numpy(), f"job {j} {name}")
        _same(s.host("b")[1], s.host("s")[1], f"job {j} refined corners")
        n = int(s.host("b")[2][0])
        assert n > 0 and np.all(out["b"][1][j].cpu().numpy()[n:] == 0)    # padding: status 0
    for s in ss:
        s.release()


@pytest.mark.gpu
def test_refusals_launch_nothing_and_touch_nothing(hv):
    import torch
    lib = hv.lib
    ss = [Session(hv, j, 32) for j in range(3)]
    other = capi.Context(0)
    foreign = other.pyramid(752, 480, 31, 1)
    tiny = hv.pyramid(14, 40, 31, 1)                                   # narrower than the 2 * 5 + 5 columns a half-window of 5 needs
    torch.cuda.synchronize()

    def detect(jobs, bs=3, cell=32, n=None):
        J = (capi.CornerJob * len(jobs))(*jobs)
        return lib.hv_gftt_detect_batch_device(hv.h, J, len(jobs) if n is None else n, bs, cell, 1e-3)

    def select(jobs, n=None):
        J = (capi.CornerJob * len(jobs))(*jobs)
        return lib.hv_gftt_select_batch_device(hv.h, J, len(jobs) if n is None else n)

    def refine(jobs, hw=5, hh=5, n=None):
        J = (capi.SubpixJob * len(jobs))(*jobs)
        return lib.hv_subpix_refine_batch_device(hv.h, J, len(jobs) if n is None else n, hw, hh, -1, -1, 3, 30, 0.01)

    def jobs_with_last(**kw):
        """the valid jobs with the LAST one changed: a refusal must come before the earlier jobs are launched"""
        js = [s.job() for s in ss]
        for k, v in kw.items():
            setattr(js[-1], k, v)
        return js

    def sjobs(last=None, **kw):
        js = [capi.subpix_job(s.pyr, s.buf["b"][1]) for s in ss]
        if last is not None:
            js[-1] = last
        for k, v in kw.items():
            setattr(js[-1], k, v)
        return js

    before = hv.launches
    ok = [s.job() for s in ss]
    assert lib.hv_gftt_detect_batch_device(None, (capi.CornerJob * 1)(ok[0]), 1, 3, 32, 1e-3) == HV_ERR_INVALID
    assert lib.hv_gftt_detect_batch_device(hv.h, None, 1, 3, 32, 1e-3) == HV_ERR_INVALID
    assert detect(ok, n=0) == HV_ERR_INVALID
    assert detect([ok[0]] * 65) == HV_ERR_INVALID
    assert detect(jobs_with_last(pyr=None)) == HV_ERR_INVALID
    assert detect(jobs_with_last(pyr=foreign.h.value)) == HV_ERR_INVALID
    assert detect(jobs_with_last(d_kp=None)) == HV_ERR_INVALID
    assert detect(ok, bs=5) == HV_ERR_UNSUPPORTED
    assert detect(ok, cell=64) == HV_ERR_UNSUPPORTED

    assert lib.hv_gftt_select_batch_device(hv.h, None, 1) == HV_ERR_INVALID
    assert select(ok, n=0) == HV_ERR_INVALID
    assert select([ok[0]] * 65) == HV_ERR_INVALID
    assert select(jobs_with_last(d_corners=None)) == HV_ERR_INVALID
    assert select(jobs_with_last(d_count=None)) == HV_ERR_INVALID
    assert select(jobs_with_last(d_kp=None)) == HV_ERR_INVALID
    assert select(jobs_with_last(nprev=4, d_prev_xy=None)) == HV_ERR_INVALID
    assert select(jobs_with_last(nkp=-1)) == HV_ERR_INVALID
    assert select(jobs_with_last(max_tracks=0)) == HV_ERR_INVALID
    last = ss[-1]
    assert select(jobs_with_last(capacity=gc.capacity(last.nkp, last.r, last.m) - 1)) == HV_ERR_INVALID
    assert select(jobs_with_last(nkp=gc.MAX_KP + 1, capacity=2 * gc.MAX_KP + 2)) == HV_ERR_UNSUPPORTED
    assert select(jobs_with_last(mask_radius=46341)) == HV_ERR_UNSUPPORTED

    assert lib.hv_subpix_refine_batch_device(hv.h, None, 1, 5, 5, -1, -1, 3, 30, 0.01) == HV_ERR_INVALID
    assert refine(sjobs(), n=0) == HV_ERR_INVALID
    assert refine(sjobs() * 22) == HV_ERR_INVALID                         # 66 jobs
    assert refine(sjobs(pyr=None)) == HV_ERR_INVALID
    assert refine(sjobs(pyr=foreign.h.value)) == HV_ERR_INVALID
    assert refine(sjobs(d_xy=None)) == HV_ERR_INVALID
    assert refine(sjobs(n=-1)) == HV_ERR_INVALID
    assert refine(sjobs(pyr=tiny.h.value)) == HV_ERR_INVALID
    assert refine(sjobs(), hw=0) == HV_ERR_UNSUPPORTED
    assert refine(sjobs(), hh=16) == HV_ERR_UNSUPPORTED
    assert hv.launches == before
    hv.sync()
    for s in ss:
        kp, cor, cnt = s.host("b")
        assert np.all(kp == SENT) and np.all(cor == SENT) and int(cnt[0]) == -1
    foreign.release(); other.close(); tiny.release()
    for s in ss:
        s.release()
