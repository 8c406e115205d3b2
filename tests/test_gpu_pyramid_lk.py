"""GPU parity tests (through the C ABI): CUDA pyramid + LK vs the oracle, the golden vectors of the compiled
reference, and size-independent properties at BASELINE sizes.

Tolerances (BASELINE.json north_star / SURVEY.md 8(c)):
  * pyramid gray + Scharr levels: bit-exact (incl. the reference's padding, reconstructed by the accessor)
  * LK vs the oracle in accum_mode 1 (the kernel's own exact-integer arithmetic): bit-exact end points + status
  * LK vs the reference (golden vectors / accum_mode 0): status and track status identical; end points <= 1e-3 px
    for >= 99.9% of tracked points (outliers listed) and < 3e-2 px for all (a flipped stop test moves a point by at most one step).
"""
import hashlib
import os

import numpy as np
import pytest

from hybvio_b200 import synth

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "lk_golden.npz")
TOL_PX = 1e-3
TOL_FLIP_PX = 3e-2


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


def build(hv, img, win=31, max_level=3):
    p = hv.pyramid(img.shape[1], img.shape[0], win, max_level)
    p.build(np.ascontiguousarray(img))
    return p


def assert_lk_close(n_gpu, ts_gpu, n_ref, ts_ref, what):
    assert np.array_equal(ts_gpu, ts_ref), f"{what}: track status differs at {np.nonzero(ts_gpu != ts_ref)[0][:10]}"
    ok = ts_ref == 0
    d = np.abs(n_gpu - n_ref).max(axis=1)[ok]
    if d.size:
        # SURVEY.md 8(c): >= 99.9 % of the end points within 1e-3 px (a flipped stop test moves a point by one step: at most
        # ceil(n / 1000) such points), every point within 3e-2 px; the outliers are listed
        idx = np.nonzero(ok)[0][d > TOL_PX]
        outliers = [(int(i), float(np.abs(n_gpu[i] - n_ref[i]).max())) for i in idx]
        if outliers:
            print(f"{what}: {len(outliers)} of {d.size} end points differ by more than {TOL_PX} px: {outliers[:20]}")
        assert len(outliers) <= -(-d.size // 1000), f"{what}: {len(outliers)} of {d.size} end points off by more than {TOL_PX} px: {outliers[:20]}"
        assert d.max() < TOL_FLIP_PX, f"{what}: end point off by {d.max():.3e} px"


@pytest.mark.parametrize("w,h,max_level", [(752, 480, 3), (512, 512, 3), (752, 480, 2), (751, 479, 3), (320, 240, 3),
                                           (100, 70, 3), (65, 129, 1), (64, 64, 0), (33, 40, 3), (1000, 37, 4), (1280, 720, 5)])
def test_pyramid_bit_exact_vs_oracle(hv, oracle_lk, w, h, max_level):
    img, _ = synth.stereo_frame(w % 17, w, h, seed=h)
    p = build(hv, img, 31, max_level)
    o = oracle_lk.pyramid(img, 31, max_level)
    assert p.levels == o.levels
    for lv in range(p.levels):
        assert p.level_size(lv) == o.level_size(lv)
        g, d = p.download(lv, padded=True)
        og, od = o.download(lv, padded=True)
        assert np.array_equal(g, og), f"gray level {lv} differs"
        assert np.array_equal(d, od), f"deriv level {lv} differs"
    p.release()


def test_pyramid_matches_reference_golden(hv, gold):
    p = build(hv, gold["A_I"])
    assert p.levels == int(gold["A_levels"])
    for lv in range(p.levels):
        g, d = p.download(lv, padded=True)
        assert np.array_equal(g, gold[f"A_gray{lv}"]) and sha(d) == str(gold[f"A_deriv_sha{lv}"])
    L0, _ = synth.stereo_frame(10)
    p2 = build(hv, L0)
    for lv in range(4):
        g, d = p2.download(lv, padded=True)
        assert sha(g) == str(gold[f"B_gray_sha{lv}"]) and sha(d) == str(gold[f"B_deriv_sha{lv}"])
    p.release(); p2.release()


def test_pyramid_batch_and_strided_input(hv, oracle_lk):
    """Stereo pair in one launch; host image with a row stride larger than its width (accelerated::Image ROI)."""
    L, R = synth.stereo_frame(5)
    big = np.zeros((480, 800), np.uint8); big[:, :752] = L
    view = big[:, :752]
    pl, pr = hv.pyramid(752, 480), hv.pyramid(752, 480)
    hv.build_pyramids([pl, pr], [view, R])
    for p, img in ((pl, L), (pr, R)):
        o = oracle_lk.pyramid(img)
        for lv in range(4):
            for a, b in zip(p.download(lv), o.download(lv, padded=False)):
                assert np.array_equal(a, b)
    pl.release(); pr.release()


def test_lk_matches_reference_golden(hv, gold):
    pa, pb = build(hv, gold["A_I"]), build(hv, gold["A_J"])
    n, st, ts = hv.lk_track(pa, pb, gold["A_pts"])
    assert np.array_equal(st, gold["A_status"])
    assert_lk_close(n, ts, gold["A_next"], gold["A_ts"], "golden A")
    n, st, ts = hv.lk_track(pa, pb, gold["A_pts"], gold["A_init"])
    assert np.array_equal(st, gold["A_status_init"])
    assert_lk_close(n, ts, gold["A_next_init"], gold["A_ts_init"], "golden A init")
    L0, R0 = synth.stereo_frame(10)
    L1, _ = synth.stereo_frame(11)
    p0, p1, pr = build(hv, L0), build(hv, L1), build(hv, R0)
    n, st, ts = hv.lk_track(p0, p1, gold["B_pts"])
    assert_lk_close(n, ts, gold["B_next_t"], gold["B_ts_t"], "golden B temporal")
    n, st, ts = hv.lk_track(p0, pr, gold["B_pts"])
    assert_lk_close(n, ts, gold["B_next_s"], gold["B_ts_s"], "golden B stereo")
    a, _ = synth.stereo_frame(20, 512, 512)
    b, _ = synth.stereo_frame(21, 512, 512)
    qa, qb = build(hv, a), build(hv, b)
    n, st, ts = hv.lk_track(qa, qb, gold["C_pts"], gold["C_init"])
    assert_lk_close(n, ts, gold["C_next"], gold["C_ts"], "golden C (512x512)")
    for p in (pa, pb, p0, p1, pr, qa, qb):
        p.release()


def _lk_vs_oracle(hv, oracle_lk, w, h, max_level, use_init, seed, win, pts):
    """LK on the GPU against the oracle: bit-exact in accum_mode 1, assert_lk_close in accum_mode 0. Returns the oracle pyramid and statuses."""
    I, _ = synth.stereo_frame(seed, w, h, seed=seed)
    J, _ = synth.stereo_frame(seed + 1, w, h, seed=seed)
    if w > 200:
        I = I.copy(); I[100:160, 100:160] = 77          # constant patch: minEig rejection
    fx, fy = synth.true_flow(seed, seed + 1)
    init = (pts + [fx, fy] + np.random.RandomState(seed).uniform(-4, 4, pts.shape)).astype(np.float32) if use_init else None
    pa, pb = build(hv, I, win, max_level), build(hv, J, win, max_level)
    oa, ob = oracle_lk.pyramid(I, win, max_level), oracle_lk.pyramid(J, win, max_level)
    assert pa.levels == oa.levels
    n_gpu, st_gpu, ts_gpu = hv.lk_track(pa, pb, pts, init)
    n1, s1, t1 = oracle_lk.lk(oa, ob, pts, init, max_level=max_level, accum_mode=1)
    assert np.array_equal(st_gpu, s1) and np.array_equal(ts_gpu, t1)
    assert np.array_equal(n_gpu.view(np.uint32), n1.view(np.uint32)), \
        f"not bit-exact vs oracle exact mode: max diff {np.abs(n_gpu - n1).max()}"
    n0, s0, t0 = oracle_lk.lk(oa, ob, pts, init, max_level=max_level, accum_mode=0)
    assert np.array_equal(st_gpu, s0)
    assert_lk_close(n_gpu, ts_gpu, n0, t0, "vs reference-order oracle")
    pa.release(); pb.release()
    return oa, s1


@pytest.mark.parametrize("w,h,max_level,n,use_init,seed", [
    (752, 480, 3, 600, False, 1), (752, 480, 3, 600, True, 2), (512, 512, 3, 400, True, 3), (752, 480, 2, 100, True, 8),
    (751, 479, 2, 200, False, 4), (100, 70, 3, 64, False, 5), (33, 40, 3, 20, True, 6), (64, 64, 0, 30, False, 7),
    (752, 480, 3, 1000, True, 9)])   # > 640 features: warp-per-feature kernel; <= 640: CTA-per-feature kernel
def test_lk_bit_exact_vs_oracle_exact_mode_and_close_to_reference_order(hv, oracle_lk, w, h, max_level, n, use_init, seed):
    pts = synth.feature_points(n, w, h, seed=seed, flat_fraction=0.1 if w > 200 else 0, flat_rect=(115, 115, 145, 145))
    _lk_vs_oracle(hv, oracle_lk, w, h, max_level, use_init, seed, 31, pts)


@pytest.mark.parametrize("w,h,max_level,n,use_init,seed,win", [
    (752, 480, 5, 600, True, 11, 11), (752, 480, 5, 1000, False, 12, 11), (1280, 720, 5, 400, True, 13, 11), (96, 100, 3, 60, True, 14, 11),
    (752, 480, 4, 500, False, 15, 15), (1280, 720, 5, 1200, True, 16, 15), (128, 140, 3, 60, False, 17, 15),
    (752, 480, 4, 640, True, 18, 21), (1280, 720, 4, 641, False, 19, 21), (176, 200, 3, 60, True, 20, 21)])
def test_lk_other_windows_bit_exact_vs_oracle_exact_mode_and_close_to_reference_order(hv, oracle_lk, w, h, max_level, n, use_init, seed, win):
    """The window templates other than 31 (hv_lk_cta_kernel / hv_lk_kernel<11, 15, 21>): both kernels (n <= 640 and n > 640), 5- and
    6-level pyramids, a coarsest level win + 1 pixels wide; uniform points (incl. the flat patch), points within `win` of every border and
    far-out points."""
    pts = synth.feature_points(n, w, h, seed=seed, flat_fraction=0.1 if w > 200 else 0, flat_rect=(115, 115, 145, 145))
    rng = np.random.RandomState(seed)
    k = 8
    xs = np.concatenate([rng.uniform(0, win, k), rng.uniform(w - win, w, k), rng.uniform(0, w, 2 * k)])
    ys = np.concatenate([rng.uniform(0, h, 2 * k), rng.uniform(0, win, k), rng.uniform(h - win, h, k)])
    far = [[-3 * win, h / 2], [w + 3 * win, h / 2], [w / 2, -1e4], [1e6, 1e6]]
    pts = np.concatenate([pts[:n - len(xs) - len(far)], np.stack([xs, ys], 1), far]).astype(np.float32)
    oa, s1 = _lk_vs_oracle(hv, oracle_lk, w, h, max_level, use_init, seed, win, pts)
    if w < 200:
        assert oa.level_size(oa.levels - 1)[0] == win + 1
    assert 0 < s1.sum() < len(s1)                      # the flat patch and far-out points fail, the rest track


@pytest.mark.parametrize("max_iter,eps,min_eig", [(m, 0.03, 1e-3) for m in (0, 1, 5, 100, 150)] +
                         [(20, e, 1e-3) for e in (0.0, 1e-6, 0.5, 20.0)] + [(20, 0.03, me) for me in (0.0, 1e-2)])
def test_lk_termination_criteria_bit_exact_vs_oracle(hv, oracle_lk, max_iter, eps, min_eig):
    """Other max_iter / eps / min_eig than the tracker's defaults, incl. values the criteria clamp (max_iter <= 100, eps <= 10) limits."""
    I, _ = synth.stereo_frame(40, 752, 480, seed=40)
    J, _ = synth.stereo_frame(41, 752, 480, seed=40)
    I = I.copy(); I[100:160, 100:160] = 77
    pts = synth.feature_points(300, 752, 480, seed=40, flat_fraction=0.1, flat_rect=(115, 115, 145, 145))
    pa, pb = build(hv, I), build(hv, J)
    oa, ob = oracle_lk.pyramid(I), oracle_lk.pyramid(J)
    n_gpu, st_gpu, ts_gpu = hv.lk_track(pa, pb, pts, None, max_iter=max_iter, eps=eps, min_eig=min_eig)
    n1, s1, t1 = oracle_lk.lk(oa, ob, pts, None, max_iter=max_iter, eps=eps, min_eig=min_eig, accum_mode=1)
    assert np.array_equal(st_gpu, s1) and np.array_equal(ts_gpu, t1)
    assert np.array_equal(n_gpu.view(np.uint32), n1.view(np.uint32)), np.abs(n_gpu - n1).max()
    pa.release(); pb.release()


def test_lk_batch_device_matches_single_jobs(hv):
    """hv_lk_track_batch_device: jobs of unequal n (incl. 0), 11 jobs (two launches of at most 8), totals above 640 with every job below
    it (the kernel is picked on the total): every job equals the same job issued alone through hv_lk_track_device, bit for bit; mixed
    window sizes are rejected."""
    import torch
    from hybvio_b200 import capi
    frames = [synth.stereo_frame(50 + k)[0] for k in range(4)]
    pyrs = [build(hv, f) for f in frames]

    def job_set(sizes):
        out = []
        for i, n in enumerate(sizes):
            pts = synth.feature_points(max(n, 1), seed=60 + i)[:n]
            out.append((pyrs[i % 3], pyrs[i % 3 + 1], torch.from_numpy(np.ascontiguousarray(pts)).cuda().reshape(n, 2), n))
        return out

    def run_batch(js):
        res = [(torch.full((n, 2), -1.0, device="cuda"), torch.zeros(n, dtype=torch.uint8, device="cuda"),
                torch.full((n,), -1, dtype=torch.int32, device="cuda")) for _, _, _, n in js]
        jobs = (capi.LkJob * len(js))()
        for k, ((a, b, d, n), (nx, st, ts)) in enumerate(zip(js, res)):
            jobs[k].prev, jobs[k].next, jobs[k].n, jobs[k].use_initial = a.h, b.h, n, 0
            jobs[k].d_prev_xy, jobs[k].d_next_xy, jobs[k].d_status, jobs[k].d_track_status = d.data_ptr(), nx.data_ptr(), st.data_ptr(), ts.data_ptr()
        torch.cuda.synchronize()
        capi.check(hv.lib.hv_lk_track_batch_device(hv.h, jobs, len(js), 20, 0.03, 1e-3), "hv_lk_track_batch_device")
        hv.sync()
        return [tuple(x.cpu().numpy() for x in r) for r in res]

    for sizes in ([150, 0, 37, 300, 1], [100, 90, 80, 70, 60, 50, 40, 30, 20, 10, 5], [600, 500, 100]):
        js = job_set(sizes)
        got = run_batch(js)
        for (a, b, d, n), (nx, st, ts) in zip(js, got):
            if n == 0:
                continue
            nx1 = torch.zeros((n, 2), device="cuda"); st1 = torch.zeros(n, dtype=torch.uint8, device="cuda"); ts1 = torch.zeros(n, dtype=torch.int32, device="cuda")
            hv.lk_track_device(a, b, d, nx1, st1, ts1, n, False)
            hv.sync()
            assert np.array_equal(nx.view(np.uint32), nx1.cpu().numpy().view(np.uint32)), sizes
            assert np.array_equal(st, st1.cpu().numpy()) and np.array_equal(ts, ts1.cpu().numpy()), sizes
    p11a, p11b = build(hv, frames[0], 11), build(hv, frames[1], 11)
    d = torch.from_numpy(synth.interior_points(10)).cuda()
    out = [torch.zeros((10, 2), device="cuda"), torch.zeros(10, dtype=torch.uint8, device="cuda"), torch.zeros(10, dtype=torch.int32, device="cuda")]
    jobs = (capi.LkJob * 2)()
    for k, (a, b) in enumerate(((pyrs[0], pyrs[1]), (p11a, p11b))):
        jobs[k].prev, jobs[k].next, jobs[k].n, jobs[k].use_initial = a.h, b.h, 10, 0
        jobs[k].d_prev_xy, jobs[k].d_next_xy, jobs[k].d_status, jobs[k].d_track_status = d.data_ptr(), out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr()
    assert hv.lib.hv_lk_track_batch_device(hv.h, jobs, 2, 20, 0.03, 1e-3) == -1          # HV_ERR_INVALID
    for p in pyrs + [p11a, p11b]:
        p.release()


def test_lk_edge_cases(hv):
    I, _ = synth.stereo_frame(0, 96, 80)
    p = build(hv, I)
    assert p.levels == 2
    n, st, ts = hv.lk_track(p, p, np.zeros((0, 2), np.float32))          # empty input -> empty output
    assert n.shape == (0, 2) and st.shape == (0,)
    n, st, ts = hv.lk_track(p, p, np.array([[40.5, 30.25]], np.float32))   # identical images: zero flow
    assert st[0] == 1 and ts[0] == 0 and np.abs(n - [[40.5, 30.25]]).max() < 1e-3
    far = np.array([[-500., 10.], [40., 9000.], [1e9, 1e9]], np.float32)    # far outside: FAILED -> FLOW_OUT_OF_RANGE
    n, st, ts = hv.lk_track(p, p, far)
    assert not st.any() and (ts == 4).all()
    p.release()


def test_lk_properties_at_baseline_size(hv):
    """Size-independent properties on the BASELINE config-2 shape: (1) determinism, (2) tracking a frame against
    itself returns the input points, (3) the synthetic stream's known flow / disparity is recovered, (4) the
    result does not depend on how the points are batched."""
    L0, R0 = synth.stereo_frame(30)
    L1, _ = synth.stereo_frame(31)
    p0, p1, pr = build(hv, L0), build(hv, L1), build(hv, R0)
    pts = synth.interior_points(150, seed=11)
    a = hv.lk_track(p0, p1, pts)
    b = hv.lk_track(p0, p1, pts)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    s = hv.lk_track(p0, p0, pts)
    assert s[1].all() and np.abs(s[0] - pts).max() < 1e-3
    fx, fy = synth.true_flow(30, 31)
    assert a[1].all() and np.abs(a[0] - pts - [fx, fy]).max() < 0.25
    st = hv.lk_track(p0, pr, pts)
    disp = synth.true_disparity(pts[:, 0], pts[:, 1])
    assert st[1].all() and np.abs(st[0][:, 0] - pts[:, 0] - disp).max() < 0.5 and np.abs(st[0][:, 1] - pts[:, 1]).max() < 0.25
    half = hv.lk_track(p0, p1, pts[:75])
    assert np.array_equal(half[0], a[0][:75])
    for p in (p0, p1, pr):
        p.release()


def test_pyramid_from_device_frame_and_device_lk(hv, oracle_lk):
    """Frame already in HBM (hv_pyr_build_batch src_is_device): aligned and odd-pitch sources; device-pointer LK."""
    import torch
    L, R = synth.stereo_frame(7)
    dL = torch.from_numpy(L).cuda()
    odd = torch.zeros((480, 757), dtype=torch.uint8, device="cuda")    # pitch 757: not a multiple of 4
    odd[:, :752] = torch.from_numpy(R).cuda()
    pl, pr = hv.pyramid(752, 480), hv.pyramid(752, 480)
    hv.build_pyramids([pl, pr], [dL, odd[:, :752]], device=True)
    for p, img in ((pl, L), (pr, R)):
        o = oracle_lk.pyramid(img)
        for lv in range(4):
            for a, b in zip(p.download(lv), o.download(lv, padded=False)):
                assert np.array_equal(a, b)
    pts = synth.interior_points(150, seed=5)
    d_prev = torch.from_numpy(pts).cuda()
    d_next = torch.zeros_like(d_prev)
    d_st = torch.zeros(150, dtype=torch.uint8, device="cuda"); d_ts = torch.zeros(150, dtype=torch.int32, device="cuda")
    hv.lk_track_device(pl, pr, d_prev, d_next, d_st, d_ts, 150, False)
    hv.sync()
    n_host, st_host, ts_host = hv.lk_track(pl, pr, pts)
    assert np.array_equal(d_next.cpu().numpy(), n_host) and np.array_equal(d_ts.cpu().numpy(), ts_host)
    # the same launch on a stream of the caller, with the initial guess in its own buffer: bit-identical to use_initial in place
    init = (pts + np.array([1.5, -0.75], dtype=np.float32)).astype(np.float32)
    d_init = torch.from_numpy(init).cuda()
    d_a = d_init.clone(); d_b = torch.zeros_like(d_prev)
    st2 = torch.zeros(150, dtype=torch.uint8, device="cuda"); ts2 = torch.zeros(150, dtype=torch.int32, device="cuda")
    hv.lk_track_device(pl, pr, d_prev, d_a, d_st, d_ts, 150, True)
    hv.sync()
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    hv.lk_track_device_on_stream(side.cuda_stream, pl, pr, d_prev, d_init, d_b, st2, ts2, 150)
    hv.lk_track_device_on_stream(side.cuda_stream, pl, pr, d_prev, None, d_next, st2, ts2, 150)      # no guess: starts at the previous points
    side.synchronize()
    assert np.array_equal(d_a.cpu().numpy(), d_b.cpu().numpy()) and np.array_equal(d_init.cpu().numpy(), init)
    assert np.array_equal(d_next.cpu().numpy(), n_host) and np.array_equal(ts2.cpu().numpy(), ts_host)
    pl.release(); pr.release()
