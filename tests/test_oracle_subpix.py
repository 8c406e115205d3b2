"""CPU: the cornerSubPix oracle (oracle/hv_oracle_subpix.c) against cv2.cornerSubPix / cv2.getRectSubPix with IPP off, BIT for bit,
over windows, zero zones, criteria, images and start points (incl. the border patch path, steps out of the image and the revert);
plus two checks that need no cv2: the refined corners of a blurred checkerboard lie at the analytic corners, and the comparison
rejects three injected faults of the restatement."""
import numpy as np
import pytest

import subpix_common as sc
from oracle import subpix_oracle as so


@pytest.fixture(scope="module")
def orc(oracle_lk):                 # oracle_lk builds oracle/libhv_oracle.so when it is missing
    return so.OracleSubpix()


@pytest.fixture(scope="module")
def cv2():
    cv2 = pytest.importorskip("cv2", reason="OpenCV (cv2) is not installed: nothing to compare the oracle with")
    cv2.ipp.setUseIPP(False)         # the reference builds OpenCV with -DWITH_IPP=OFF
    return cv2


@pytest.fixture(scope="module")
def imgs():
    return sc.images()


def cv_refine(cv2, img, pts, win, zero, crit):
    return cv2.cornerSubPix(img, pts.reshape(-1, 1, 2).copy(), win, zero, crit).reshape(-1, 2)


def assert_bits(got, want, what):
    bad = np.nonzero((got.view(np.uint32) != want.view(np.uint32)).any(axis=1))[0]
    assert len(bad) == 0, f"{what}: {len(bad)} corners differ, first {bad[:5]}: {got[bad[:3]]} vs {want[bad[:3]]}"


@pytest.mark.parametrize("zero", sc.ZERO_ZONES, ids=str)
@pytest.mark.parametrize("win", sc.WINDOWS, ids=str)
def test_oracle_bit_exact_vs_cv2_windows_and_zero_zones(orc, cv2, imgs, win, zero):
    z = sc.zero_zone(zero, win)
    for name, img in imgs.items():
        pts = sc.points(img, win, seed=len(name))
        assert_bits(orc.refine(img, pts, win, z, (3, 30, 0.01)), cv_refine(cv2, img, pts, win, z, (3, 30, 0.01)), f"{name} win {win} zero {z}")


@pytest.mark.parametrize("crit", sc.CRITERIA, ids=str)
def test_oracle_bit_exact_vs_cv2_criteria(orc, cv2, imgs, crit):
    for win in [(2, 3), (5, 5)]:
        for name, img in imgs.items():
            pts = sc.points(img, win, seed=3)
            assert_bits(orc.refine(img, pts, win, (-1, -1), crit), cv_refine(cv2, img, pts, win, (-1, -1), crit), f"{name} win {win} crit {crit}")


def test_rect_subpix_bit_exact_vs_cv2(orc, cv2, imgs):
    """getRectSubPix(8U -> 32F) alone, at centres inside, near and outside every border (the adjustRect path), all patch sizes used."""
    rng = np.random.RandomState(4)
    for name in ("texture", "frame751"):
        img = imgs[name]
        h, w = img.shape
        for _ in range(1500):
            size = (int(rng.randint(3, 34)), int(rng.randint(3, 34)))
            c = np.float32(rng.uniform(-20, w + 20)), np.float32(rng.uniform(-20, h + 20))
            want = cv2.getRectSubPix(img, size, (float(c[0]), float(c[1])), patchType=cv2.CV_32F)
            assert np.array_equal(orc.rect(img, size, c).view(np.uint32), want.view(np.uint32)), (name, size, c)


def test_sweep_reaches_every_stop_rule(orc, imgs):
    """The start points above do exercise the paths under test: some corners are reverted (moved more than the window), some stop
    outside the image, some stop on det == 0 (flat patches) and some run through the border patch path."""
    img = imgs["flat"]
    pts = np.array([[60, 50], [70.5, 40.25], [20, 120]], np.float32)         # flat patches: det == 0 at once, the point stays
    assert np.array_equal(orc.refine(img, pts, (5, 5), (-1, -1), (3, 30, 0.01)), pts)
    reverted = border = 0
    for name, img in imgs.items():
        for win in sc.WINDOWS:
            pts = sc.points(img, win, seed=len(name))
            ok = orc.refine(img, pts, win, (-1, -1), (3, 30, 0.01))
            reverted += int((orc.refine(img, pts, win, (-1, -1), (3, 30, 0.01), faults=so.NO_REVERT) != ok).any(axis=1).sum())
            border += int((orc.refine(img, pts, win, (-1, -1), (3, 30, 0.01), faults=so.CLAMP) != ok).any(axis=1).sum())
    assert reverted >= 10 and border >= 10, (reverted, border)


def test_injected_faults_are_rejected(orc, imgs):
    """Without cv2: float accumulators, a dropped revert rule and a plain clamp for the border patch each change the bits of some
    refinements of the sweep, so the bit-exact comparison above would reject each of them."""
    for fault in (so.FLOAT_ACC, so.NO_REVERT, so.CLAMP):
        differ = 0
        for name, img in imgs.items():
            for win in [(2, 3), (5, 5), (11, 11)]:
                pts = sc.points(img, win, seed=1)
                a = orc.refine(img, pts, win, (-1, -1), (3, 30, 0.01))
                b = orc.refine(img, pts, win, (-1, -1), (3, 30, 0.01), faults=fault)
                differ += int((a.view(np.uint32) != b.view(np.uint32)).any(axis=1).sum())
        assert differ > 0, f"fault {fault} is not visible in the sweep"


def test_checkerboard_corners_land_on_the_analytic_corners(orc):
    """Without cv2: blurred checkerboards with sub-pixel corner positions; from starts up to 2 px off, the refinement with a 5 x 5
    half-window ends within 0.05 px of the true corner on both axes (the residual is the 8-bit quantisation and the blur)."""
    rng = np.random.RandomState(8)
    for ox, oy in [(20.3, 17.6), (21.5, 19.0), (19.87, 18.25)]:
        img, truth = sc.checkerboard(200, 160, ox, oy)
        start = (truth + rng.uniform(-2, 2, truth.shape)).astype(np.float32)
        got = orc.refine(img, start, (5, 5), (-1, -1), (3, 40, 0.001))
        err = np.abs(got - truth).max()
        assert err < 0.05, (ox, oy, err)


def test_oracle_refuses_what_cv_asserts(orc, imgs):
    img = imgs["texture"]
    h, w = img.shape
    assert orc.refine(img, [[w, 5]], (5, 5)) is None                     # corner outside [0, w) x [0, h)
    assert orc.refine(img, [[5, -0.001]], (5, 5)) is None
    assert orc.refine(img[:14, :], [[5, 5]], (5, 5)) is None              # rows < 2 win + 5
    assert orc.refine(img, [[5, 5]], (0, 5)) is None                      # win > 0
    assert orc.refine(img[:15, :], [[5, 5]], (5, 5)) is not None
