"""The tracker front end (frame ingest, pyramid, GFTT key points, batched LK) at the layouts its C ABI accepts beyond the benchmark's gray
752 x 480 frames, every case BIT for BIT against the C oracles (oracle/hv_oracle_gftt.c, oracle/hv_oracle_lk.c), which are pinned to the
compiled reference by their own tests:
  * hv_ingest_frame: widths of every residue mod 4 (tiny, below 256, ragged against the kernels' 256-wide x grid), 1 .. 4 channels, the
    default and explicit colour coefficients (incl. sums above 1 and negative entries: both clamps fire), random remap tables with taps on
    the last column / row and entries without a source, host frames that are views into wider buffers, a table dropped and set again;
    the pyramid built in place from the ingested image equals the oracle's pyramid of the oracle's image.
  * hv_pyr_build / hv_pyr_build_batch: windows 3, 5, 11 with levels under 8 px (level 0 included), batches above PYR_MAX_BATCH (32),
    pyramids of 1 .. 6 levels in one launch, device sources on every staging branch (TMA, 32-bit loads, byte loads, a 6-level pyramid
    whose box TMA refuses), host sources whose row stride is the level-0 pitch; all of it again with HV_PYR_NO_TMA=1.
  * hv_gftt_detect / hv_gftt_detect_batch_device: every cell size 2 .. 32, images smaller than a cell, min_response at the edges of the
    strict comparison.
  * hv_lk_track_batch_device: per job against the oracle in exact-integer mode over mixed pyramid sizes and depths, use_initial mixed,
    totals on both sides of the 640-feature kernel switch, more than LK_MAX_JOBS (8) jobs, every supported window; and
    hv_lk_track_device_on_stream with a separate initial-guess buffer on the warp-per-feature kernel."""
import os
import subprocess
import sys

import numpy as np
import pytest

from hybvio_b200 import synth
from oracle import gftt_oracle
from oracle import ingest_oracle as io

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HV_OK = 0


@pytest.fixture(scope="module")
def orc():
    subprocess.check_call(["make", "-C", ROOT, "oracle"], stdout=subprocess.DEVNULL)
    return io.OracleIngest()


@pytest.fixture(scope="module")
def orc_gftt(orc):
    return gftt_oracle.OracleGftt()


def assert_pyramid_equal(p, o, what):
    assert p.levels == o.levels, what
    for lv in range(p.levels):
        assert p.level_size(lv) == o.level_size(lv), (what, lv)
        g, d = p.download(lv, padded=True)
        og, od = o.download(lv, padded=True)
        assert np.array_equal(g, og), f"{what}: gray level {lv} differs"
        assert np.array_equal(d, od), f"{what}: deriv level {lv} differs"


def gpitch(w):
    """Row pitch of a pyramid's level-0 buffer (hv_pyr_create): w when w % 4 == 0, else w rounded up to 128."""
    return w if w % 4 == 0 else (w + 127) // 128 * 128


def padded_view(img, stride, rng):
    """img (h, w) or (h, w, c) uint8 as a view into a buffer of `stride` bytes per row whose padding holds non-zero bytes."""
    h, w = img.shape[:2]
    c = 1 if img.ndim == 2 else img.shape[2]
    buf = rng.randint(1, 256, (h, stride)).astype(np.uint8)
    view = buf[:, :w * c].reshape(img.shape)
    assert np.shares_memory(view, buf) and view.strides[0] == stride
    view[...] = img
    return view


# ------------------------------------------------------------------------------------------------ CPU: the oracle reads a view as laid out
def test_ingest_oracle_reads_a_view_with_its_own_stride(orc):
    """A remap tap right of the last column reads the byte after the row: the view's padding, or the next row of a contiguous image."""
    buf = np.array([[10, 100, 200, 1, 1], [30, 40, 2, 2, 2]], np.uint8)
    view, img = buf[:, :2], np.ascontiguousarray(buf[:, :2])
    t = np.zeros(4, io.REMAP_DTYPE)
    t["x0"], t["y0"], t["xfrac"], t["yfrac"] = 1, 0, 0.5, 0.0
    assert orc.remap(view, t)[0, 0] == 150 and orc.remap(img, t)[0, 0] == 65     # 0.5 * 100 + 0.5 * (200 | 30), rounded
    rng = np.random.RandomState(0)
    rgb = rng.randint(0, 256, (3, 4, 3)).astype(np.uint8)
    assert np.array_equal(orc.gray(padded_view(rgb, 13, rng)), orc.gray(rgb))


# ------------------------------------------------------------------------------------------------ ingest
# tiny, every residue mod 4 below 256, and around / across the 256-wide blocks of the ingest kernels' x grid
INGEST_WIDTHS = [1, 2, 3, 5, 6, 7, 13, 64, 97, 130, 255, 256, 257, 258, 259, 514, 771]
# coefficient sets: the default (NULL), a sum above 1 (clamp at 1), negative entries (clamp at 0)
COEFFS = [None, (0.9, 0.8, 0.7, 0.6), (-0.35, 1.3, 0.45, -0.2)]
INGEST_WIN, INGEST_LEVEL = 5, 3


def ingest_height(w):
    return 9 + (7 * w) % 29


def remap_table(rng, w, h, edge=0.01, invalid=0.05):
    """Random table; about `edge` of the entries each sample from the last column (x0 = w - 1, rows above the last), the last row
    (y0 = h - 1) and the last pixel, all with non-zero fractions; about `invalid` have no source."""
    n = w * h
    t = np.zeros(n, io.REMAP_DTYPE)
    t["x0"] = rng.randint(0, w, n); t["y0"] = rng.randint(0, h, n)
    t["xfrac"] = rng.rand(n).astype(np.float32); t["yfrac"] = rng.rand(n).astype(np.float32)
    m = max(1, int(round(edge * n)))
    i = rng.choice(n, m); t["x0"][i] = w - 1; t["y0"][i] = rng.randint(0, max(h - 1, 1), m)
    j = rng.choice(n, m); t["y0"][j] = h - 1
    k = rng.choice(n, m); t["x0"][k] = w - 1; t["y0"][k] = h - 1
    e = np.concatenate([i, j, k])
    t["xfrac"][e] = rng.uniform(0.05, 1.0, e.size).astype(np.float32)
    t["yfrac"][e] = rng.uniform(0.05, 1.0, e.size).astype(np.float32)
    t["x0"][rng.rand(n) < invalid] = io.INVALID
    return t


def check_ingest(ing, pyr, orc, oracle_lk, img, coeff, table, what):
    """One hv_ingest_frame call against the oracle: the image it returns and the pyramid built from it in place."""
    c = 1 if img.ndim == 2 else img.shape[2]
    got = ing.frame(img, pyr, coeff)
    gray = img if c == 1 else orc.gray(img, io.GRAY_COEFF if coeff is None else coeff)
    want = np.array(gray) if table is None else orc.remap(gray, table)
    assert np.array_equal(got, want), f"{what}: {np.count_nonzero(got != want)} of {got.size} pixels differ"
    assert_pyramid_equal(pyr, oracle_lk.pyramid(want, INGEST_WIN, INGEST_LEVEL), what)
    return want


@pytest.mark.gpu
@pytest.mark.parametrize("w", INGEST_WIDTHS)
def test_ingest_channels_coefficients_and_remap_bit_exact(hv, orc, oracle_lk, w):
    """Every channel count and coefficient set, without a table, with one, without again and with another."""
    from hybvio_b200 import capi
    h = ingest_height(w)
    rng = np.random.RandomState(w)
    ing, pyr = capi.Ingest(hv, w, h), hv.pyramid(w, h, INGEST_WIN, INGEST_LEVEL)
    for step, table in enumerate((None, remap_table(rng, w, h), None, remap_table(rng, w, h))):
        ing.set_remap(table)
        for c in (1, 2, 3, 4):
            img = rng.randint(0, 256, (h, w, c) if c > 1 else (h, w)).astype(np.uint8)
            for coeff in COEFFS if c > 1 else [None]:
                check_ingest(ing, pyr, orc, oracle_lk, img, coeff, table, f"{w}x{h} table step {step} channels {c} coeff {coeff}")
    ing.close(); pyr.release()


@pytest.mark.gpu
@pytest.mark.parametrize("w", [3, 61, 130, 255, 300])
def test_ingest_strided_host_frames_bit_exact(hv, orc, oracle_lk, w):
    """Host frames that are views into wider buffers (padding bytes non-zero): plain gray (row stride w + 3 and the level-0 pitch),
    gray + remap (last-column taps read the view's padding, as the reference reads its own image), colour, colour + remap."""
    from hybvio_b200 import capi
    h = ingest_height(w)
    rng = np.random.RandomState(100 + w)
    ing, pyr = capi.Ingest(hv, w, h), hv.pyramid(w, h, INGEST_WIN, INGEST_LEVEL)
    gray = rng.randint(0, 256, (h, w)).astype(np.uint8)
    table = remap_table(rng, w, h)
    for stride in sorted({w + 3, gpitch(w)}):
        check_ingest(ing, pyr, orc, oracle_lk, padded_view(gray, stride, rng), None, None, f"gray stride {stride}")
    ing.set_remap(table)
    check_ingest(ing, pyr, orc, oracle_lk, padded_view(gray, w + 5, rng), None, table, "gray + remap")
    for c, extra in ((2, 1), (3, 7), (4, 2)):
        img = rng.randint(0, 256, (h, w, c)).astype(np.uint8)
        ing.set_remap(None)
        check_ingest(ing, pyr, orc, oracle_lk, padded_view(img, w * c + extra, rng), COEFFS[c % 3], None, f"colour {c}")
        ing.set_remap(table)
        check_ingest(ing, pyr, orc, oracle_lk, padded_view(img, w * c + extra, rng), COEFFS[c % 3], table, f"colour {c} + remap")
    ing.close(); pyr.release()


# ------------------------------------------------------------------------------------------------ pyramid
# levels under 8 px, level 0 itself included
SMALL_SIZES = [(1, 1), (2, 5), (5, 9), (8, 8), (9, 17), (7, 300), (300, 7), (33, 12), (130, 70)]
DEV_W, DEV_H = 301, 203


def build_host(hv, img, win, max_level):
    p = hv.pyramid(img.shape[1], img.shape[0], win, max_level)
    p.build(img)
    return p


def pyramid_small_images(hv, oracle_lk, win):
    rng = np.random.RandomState(win)
    for w, h in SMALL_SIZES:
        for max_level in (0, 5):
            img = rng.randint(0, 256, (h, w)).astype(np.uint8)
            p = build_host(hv, img, win, max_level)
            assert_pyramid_equal(p, oracle_lk.pyramid(img, win, max_level), f"{w}x{h} win {win} max_level {max_level}")
            p.release()


def pyramid_big_batch(hv, oracle_lk, n=37):
    """n > PYR_MAX_BATCH host images in one hv_pyr_build_batch: two launches."""
    w, h = 203, 61
    rng = np.random.RandomState(n)
    imgs = [rng.randint(0, 256, (h, w)).astype(np.uint8) for _ in range(n)]
    pyrs = [hv.pyramid(w, h, 5, 3) for _ in range(n)]
    before = hv.launches
    hv.build_pyramids(pyrs, imgs)
    assert hv.launches - before == 2
    for i, (p, img) in enumerate(zip(pyrs, imgs)):
        assert_pyramid_equal(p, oracle_lk.pyramid(img, 5, 3), f"batch image {i}")
        p.release()


def pyramid_mixed_depths(hv, oracle_lk):
    """max_level 0 .. 5 at one size in one launch (shared memory for the deepest, a TMA box per image; the 6-level ones stage by loads)."""
    w, h = 320, 200
    rng = np.random.RandomState(6)
    levels = [5, 0, 3, 1, 4, 2, 5, 0]
    imgs = [rng.randint(0, 256, (h, w)).astype(np.uint8) for _ in levels]
    pyrs = [hv.pyramid(w, h, 3, ml) for ml in levels]
    hv.build_pyramids(pyrs, imgs)
    for p, img, ml in zip(pyrs, imgs, levels):
        assert p.levels == ml + 1
        assert_pyramid_equal(p, oracle_lk.pyramid(img, 3, ml), f"max_level {ml}")
        p.release()


# (pitch, byte offset of the base, max_level, win): the staging branch each takes with TMA available
DEVICE_SOURCES = [
    (320, 0, 3, 5),     # TMA: base and pitch 16-byte aligned
    (304, 0, 4, 3),     # TMA: 5 levels (box 192 wide)
    (308, 0, 3, 5),     # 32-bit loads: pitch = 4 (mod 16)
    (320, 1, 3, 5),     # byte loads: base 1 byte past alignment
    (321, 2, 3, 5),     # byte loads
    (320, 3, 3, 5),     # byte loads
    (320, 0, 5, 3),     # 32-bit loads: 6 levels, the box would be 288 wide and TMA refuses it
]


def device_source(img, pitch, offset):
    """img copied into a CUDA buffer with `pitch` bytes per row starting `offset` bytes past an allocation; the padding is non-zero."""
    import torch
    h, w = img.shape
    buf = torch.full((offset + h * pitch,), 0xA5, dtype=torch.uint8, device="cuda")
    view = buf[offset:].view(h, pitch)[:, :w]
    view.copy_(torch.from_numpy(img))
    assert view.data_ptr() % 16 == offset % 16 and view.stride(0) == pitch
    return view


def pyramid_device_sources(hv, oracle_lk):
    import torch
    rng = np.random.RandomState(11)
    imgs = [rng.randint(0, 256, (DEV_H, DEV_W)).astype(np.uint8) for _ in DEVICE_SOURCES]
    srcs = [device_source(img, pitch, off) for img, (pitch, off, _, _) in zip(imgs, DEVICE_SOURCES)]
    torch.cuda.synchronize()
    for img, src, (pitch, off, ml, win) in zip(imgs, srcs, DEVICE_SOURCES):
        p = hv.pyramid(DEV_W, DEV_H, win, ml)
        hv.build_pyramids([p], [src], device=True)
        assert_pyramid_equal(p, oracle_lk.pyramid(img, win, ml), f"device source pitch {pitch} offset {off} max_level {ml}")
        p.release()
    # one launch over every branch with one window: each image stages its own way
    sel = [i for i, s in enumerate(DEVICE_SOURCES) if s[3] == 5]
    pyrs = [hv.pyramid(DEV_W, DEV_H, 5, DEVICE_SOURCES[i][2]) for i in sel]
    hv.build_pyramids(pyrs, [srcs[i] for i in sel], device=True)
    for p, i in zip(pyrs, sel):
        assert_pyramid_equal(p, oracle_lk.pyramid(imgs[i], 5, DEVICE_SOURCES[i][2]), f"batched device source {DEVICE_SOURCES[i]}")
        p.release()
    hv.sync()


def pyramid_host_pitch_sources(hv, oracle_lk):
    """Host views whose row stride equals the level-0 pitch at w % 4 != 0 (one copy of the rows, padding included)."""
    rng = np.random.RandomState(12)
    for w, h in ((301, 203), (130, 70), (7, 300)):
        assert w % 4 and gpitch(w) > w
        imgs = [rng.randint(0, 256, (h, w)).astype(np.uint8) for _ in range(3)]
        views = [padded_view(img, gpitch(w), rng) for img in imgs]
        p = hv.pyramid(w, h, 5, 3)
        p.build(views[0])
        assert_pyramid_equal(p, oracle_lk.pyramid(imgs[0], 5, 3), f"{w}x{h} hv_pyr_build stride {gpitch(w)}")
        p.release()
        pyrs = [hv.pyramid(w, h, 5, 3) for _ in imgs]
        hv.build_pyramids(pyrs, views)
        for p, img in zip(pyrs, imgs):
            assert_pyramid_equal(p, oracle_lk.pyramid(img, 5, 3), f"{w}x{h} hv_pyr_build_batch stride {gpitch(w)}")
            p.release()


def pyramid_sweep(hv, oracle_lk):
    """Everything the pyramid tests below check, in one call (run again in a child process with HV_PYR_NO_TMA=1)."""
    for win in (3, 5, 11):
        pyramid_small_images(hv, oracle_lk, win)
    pyramid_big_batch(hv, oracle_lk)
    pyramid_mixed_depths(hv, oracle_lk)
    pyramid_device_sources(hv, oracle_lk)
    pyramid_host_pitch_sources(hv, oracle_lk)


@pytest.mark.gpu
@pytest.mark.parametrize("win", [3, 5, 11])
def test_pyramid_small_levels_bit_exact(hv, oracle_lk, win):
    pyramid_small_images(hv, oracle_lk, win)


@pytest.mark.gpu
def test_pyramid_batch_above_launch_capacity(hv, oracle_lk):
    pyramid_big_batch(hv, oracle_lk)


@pytest.mark.gpu
def test_pyramid_batch_of_mixed_depths(hv, oracle_lk):
    pyramid_mixed_depths(hv, oracle_lk)


@pytest.mark.gpu
def test_pyramid_device_sources_every_staging_branch(hv, oracle_lk):
    pyramid_device_sources(hv, oracle_lk)


@pytest.mark.gpu
def test_pyramid_host_stride_equal_to_level0_pitch(hv, oracle_lk):
    pyramid_host_pitch_sources(hv, oracle_lk)


_NO_TMA_CHILD = """
import sys
sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
import test_gpu_frontend_layouts as t
from hybvio_b200 import capi
from oracle import lk_oracle
hv = capi.Context(0)
t.pyramid_sweep(hv, lk_oracle.OracleLK())
hv.close()
"""


@pytest.mark.gpu
def test_pyramid_sweep_without_tma(oracle_lk):
    """HV_PYR_NO_TMA=1 (every source staged with loads) in a child process: the same sweep, the same bits."""
    env = dict(os.environ, HV_PYR_NO_TMA="1")
    r = subprocess.run([sys.executable, "-c", _NO_TMA_CHILD.format(root=ROOT, tests=os.path.join(ROOT, "tests"))], env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr


# ------------------------------------------------------------------------------------------------ GFTT key points
def gftt_image(w, h, k):
    img, _ = synth.stereo_frame(k, w, h)
    img = img.copy()
    img[:, : w // 5] = 90           # flat cells: every response 0
    return img


def assert_kp_equal(kp, want, what):
    assert kp.shape == want.shape, what
    assert np.array_equal(kp[:, :2], want[:, :2]), f"{what}: positions differ in cells {np.nonzero((kp[:, :2] != want[:, :2]).any(axis=1))[0][:10]}"
    assert np.array_equal(kp[:, 2].view(np.uint32), want[:, 2].view(np.uint32)), f"{what}: responses differ"


@pytest.mark.gpu
def test_gftt_every_cell_size(hv, orc_gftt):
    for w, h, k in ((211, 97, 3), (389, 151, 4)):
        img = gftt_image(w, h, k)
        resp = orc_gftt.response(img)
        p = build_host(hv, img, 31, 1)
        for cell in range(2, 33):
            assert_kp_equal(p.gftt_detect(3, cell, 1e-3), orc_gftt.collect(resp, cell, 1e-3), f"{w}x{h} cell {cell}")
        p.release()


@pytest.mark.gpu
def test_gftt_image_smaller_than_a_cell_writes_nothing(hv):
    import torch
    for w, h in ((20, 100), (100, 20), (31, 31)):
        p = build_host(hv, gftt_image(w, h, 1), 5, 0)
        assert p.gftt_cells(32)[0] * p.gftt_cells(32)[1] == 0
        kp = np.full(6, 7.0, np.float32)
        assert hv.lib.hv_gftt_detect(hv.h, p.h, 3, 32, 1e-3, kp.ctypes.data) == HV_OK
        assert (kp == 7.0).all()
        d = torch.full((6,), 7.0, device="cuda")
        p.gftt_detect_device(d.data_ptr(), 3, 32, 1e-3)
        hv.sync()
        assert (d.cpu() == 7.0).all()
        p.release()


@pytest.mark.gpu
def test_gftt_min_response_edges(hv, orc_gftt):
    """min_response 0 (flat cells have no candidate), -1 (every pixel is one), above every response, and exactly one cell's best response
    (the comparison is strict: that cell then reports its second best)."""
    w, h, cell = 211, 97, 16
    img = gftt_image(w, h, 5)
    resp = orc_gftt.response(img)
    p = build_host(hv, img, 31, 1)
    best = orc_gftt.collect(resp, cell, 0.0)
    pos = np.sort(best[best[:, 2] > 0, 2])
    r_eq = float(pos[len(pos) // 2])
    below = float(np.nextafter(np.float32(r_eq), np.float32(-np.inf)))
    for m in (0.0, -1.0, float(resp.max()) * gftt_oracle.GAIN * 2, r_eq, below):
        assert_kp_equal(p.gftt_detect(3, cell, m), orc_gftt.collect(resp, cell, m), f"min_response {m}")
    assert not np.array_equal(orc_gftt.collect(resp, cell, r_eq), orc_gftt.collect(resp, cell, below))
    p.release()


@pytest.mark.gpu
def test_gftt_detect_batch_non_power_of_two_cell(hv, orc_gftt):
    """hv_gftt_detect_batch_device, cell 12, 17 jobs of mixed sizes (two of them smaller than a cell: their buffers stay untouched)."""
    import torch
    from hybvio_b200 import capi
    cell = 12
    sizes = [(211, 97), (64, 64), (389, 151), (100, 37), (13, 40), (11, 50), (752, 480), (25, 25), (130, 70), (97, 130),
             (40, 11), (300, 7), (48, 48), (203, 61), (12, 12), (771, 33), (59, 201)]
    imgs = [gftt_image(w, h, 20 + i) for i, (w, h) in enumerate(sizes)]
    pyrs = [build_host(hv, img, 5, 0) for img in imgs]
    cells = [(w // cell) * (h // cell) for w, h in sizes]
    bufs = [torch.full((max(n, 1), 3), 7.0, device="cuda") for n in cells]
    jobs = [capi.corner_job(p, d_kp=b) for p, b in zip(pyrs, bufs)]
    torch.cuda.synchronize()
    hv.gftt_detect_batch_device(jobs, 3, cell, 1e-3)
    hv.sync()
    assert 0 in cells
    for (w, h), img, n, b, p in zip(sizes, imgs, cells, bufs, pyrs):
        got = b.cpu().numpy()
        if n == 0:
            assert (got == 7.0).all(), (w, h)
        else:
            assert_kp_equal(got, orc_gftt.collect(orc_gftt.response(img), cell, 1e-3), f"job {w}x{h}")
        p.release()


# ------------------------------------------------------------------------------------------------ batched LK
class LkPair:
    """A frame pair on the device and in the oracle, with points (and, for use_initial, predicted end points)."""

    def __init__(self, hv, oracle_lk, w, h, max_level, win, seed, n, use_initial):
        I, _ = synth.stereo_frame(seed, w, h, seed=seed)
        J, _ = synth.stereo_frame(seed + 1, w, h, seed=seed)
        self.pa, self.pb = build_host(hv, I, win, max_level), build_host(hv, J, win, max_level)
        self.oa, self.ob = oracle_lk.pyramid(I, win, max_level), oracle_lk.pyramid(J, win, max_level)
        assert self.pa.levels == self.oa.levels
        far = np.array([[-4.0 * win, h / 2], [w + 4.0 * win, h / 2]], np.float32)     # these two fail
        self.pts = np.concatenate([synth.feature_points(n - 2, w, h, seed=seed), far])
        fx, fy = synth.true_flow(seed, seed + 1)
        rng = np.random.RandomState(seed)
        self.init = (self.pts + [fx, fy] + rng.uniform(-3, 3, self.pts.shape)).astype(np.float32) if use_initial else None
        self.n = n

    def oracle(self, oracle_lk):
        return oracle_lk.lk(self.oa, self.ob, self.pts, self.init, max_level=self.oa.levels - 1, accum_mode=1)

    def release(self):
        self.pa.release(); self.pb.release()


def run_lk_batch(hv, pairs):
    """One hv_lk_track_batch_device call over the pairs; returns (next, status, track status) per job."""
    import torch
    from hybvio_b200 import capi
    res = []
    jobs = (capi.LkJob * len(pairs))()
    for k, q in enumerate(pairs):
        d_prev = torch.from_numpy(np.ascontiguousarray(q.pts, np.float32)).cuda().reshape(q.n, 2)
        d_next = torch.from_numpy(q.init).cuda() if q.init is not None else torch.full((q.n, 2), -1.0, device="cuda")
        st = torch.full((q.n,), 9, dtype=torch.uint8, device="cuda")
        ts = torch.full((q.n,), -1, dtype=torch.int32, device="cuda")
        res.append((d_prev, d_next, st, ts))
        jobs[k].prev, jobs[k].next, jobs[k].n, jobs[k].use_initial = q.pa.h, q.pb.h, q.n, int(q.init is not None)
        jobs[k].d_prev_xy, jobs[k].d_next_xy, jobs[k].d_status, jobs[k].d_track_status = d_prev.data_ptr(), d_next.data_ptr(), st.data_ptr(), ts.data_ptr()
    torch.cuda.synchronize()
    before = hv.launches
    capi.check(hv.lib.hv_lk_track_batch_device(hv.h, jobs, len(pairs), 20, 0.03, 1e-3), "hv_lk_track_batch_device")
    hv.sync()
    assert hv.launches - before == (len(pairs) + 7) // 8
    return [(nx.cpu().numpy(), st.cpu().numpy(), ts.cpu().numpy()) for _, nx, st, ts in res]


def assert_lk_batch(hv, oracle_lk, pairs, what):
    for k, (q, (nx, st, ts)) in enumerate(zip(pairs, run_lk_batch(hv, pairs))):
        n1, s1, t1 = q.oracle(oracle_lk)
        assert np.array_equal(st, s1) and np.array_equal(ts, t1), f"{what} job {k}: status differs"
        assert np.array_equal(nx.view(np.uint32), n1.view(np.uint32)), f"{what} job {k}: max diff {np.abs(nx - n1).max()}"
        assert 0 < s1.sum() < len(s1), f"{what} job {k}"


# (w, h, max_level): 4 levels, 3 levels, 2 levels, 1 level at window 31
LK_SHAPES = [(752, 480, 3), (320, 240, 3), (100, 70, 3), (64, 64, 0)]


@pytest.mark.gpu
@pytest.mark.parametrize("counts", [(200, 150, 100, 60), (300, 200, 150, 100)], ids=["total510", "total750"])
def test_lk_batch_mixed_sizes_depths_and_initial_guess(hv, oracle_lk, counts):
    """One launch over pyramids of four sizes and depths, use_initial mixed; a total on each side of the 640-feature kernel switch."""
    pairs = [LkPair(hv, oracle_lk, w, h, ml, 31, 70 + i, n, i % 2 == (sum(counts) > 640)) for i, ((w, h, ml), n) in enumerate(zip(LK_SHAPES, counts))]
    assert [q.pa.levels for q in pairs] == [4, 3, 2, 1]
    assert_lk_batch(hv, oracle_lk, pairs, f"total {sum(counts)}")
    for q in pairs:
        q.release()


@pytest.mark.gpu
def test_lk_batch_more_jobs_than_one_launch_takes(hv, oracle_lk):
    """11 jobs: a launch of 8 (730 features: warp kernel) and one of 3 (150 features: CTA kernel)."""
    counts = [150, 120, 100, 90, 80, 70, 60, 60, 50, 50, 50]
    pairs = [LkPair(hv, oracle_lk, *LK_SHAPES[i % 4], 31, 80 + i, n, i % 3 == 0) for i, n in enumerate(counts)]
    assert sum(counts[:8]) > 640 >= sum(counts[8:])
    assert_lk_batch(hv, oracle_lk, pairs, "11 jobs")
    for q in pairs:
        q.release()


@pytest.mark.gpu
@pytest.mark.parametrize("win", [11, 15, 21, 31])
def test_lk_batch_every_window(hv, oracle_lk, win):
    shapes = [(752, 480, 4), (176, 200, 3), (96, 100, 2)]
    pairs = [LkPair(hv, oracle_lk, w, h, ml, win, 90 + i + win, n, i == 1) for i, ((w, h, ml), n) in enumerate(zip(shapes, (250, 120, 60)))]
    assert_lk_batch(hv, oracle_lk, pairs, f"win {win}")
    for q in pairs:
        q.release()


@pytest.mark.gpu
def test_lk_on_stream_initial_guess_buffer_warp_kernel(hv, oracle_lk):
    """hv_lk_track_device_on_stream with d_init at n = 900 (warp-per-feature kernel): bit-identical to use_initial in place and to the
    oracle; d_init is only read."""
    import torch
    q = LkPair(hv, oracle_lk, 752, 480, 3, 31, 120, 900, True)
    d_prev = torch.from_numpy(q.pts.astype(np.float32)).cuda()
    d_init = torch.from_numpy(q.init).cuda()
    d_a = d_init.clone(); d_b = torch.zeros_like(d_prev)
    st_a = torch.zeros(q.n, dtype=torch.uint8, device="cuda"); ts_a = torch.zeros(q.n, dtype=torch.int32, device="cuda")
    st_b = torch.zeros_like(st_a); ts_b = torch.zeros_like(ts_a)
    torch.cuda.synchronize()
    hv.lk_track_device(q.pa, q.pb, d_prev, d_a, st_a, ts_a, q.n, True)
    hv.sync()
    side = torch.cuda.Stream()
    hv.lk_track_device_on_stream(side.cuda_stream, q.pa, q.pb, d_prev, d_init, d_b, st_b, ts_b, q.n)
    side.synchronize()
    n1, s1, t1 = q.oracle(oracle_lk)
    for nx, st, ts in ((d_a, st_a, ts_a), (d_b, st_b, ts_b)):
        assert np.array_equal(nx.cpu().numpy().view(np.uint32), n1.view(np.uint32))
        assert np.array_equal(st.cpu().numpy(), s1) and np.array_equal(ts.cpu().numpy(), t1)
    assert np.array_equal(d_init.cpu().numpy(), q.init)
    q.release()
