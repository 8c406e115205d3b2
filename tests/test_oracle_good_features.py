"""CPU: the cv::goodFeaturesToTrack oracle (oracle/hv_oracle_good_features.c) against cv2, and checks that need no cv2.

With cv2.setUseOptimized(False) and IPP off, cv2 runs its baseline code (SSE2, no FMA), and the oracle must match it BIT for bit at every
stage: Sobel dx and dy (scale 1/3060, as cornerMinEigenVal forms them), boxFilter of their products, cornerMinEigenVal, and goodFeaturesToTrack's list (count, order,
x, y, cornersQuality) over the images of good_features_common, every mask, min distance, corner budget and quality. With cv2's defaults
(dispatch to AVX2 / FMA and IPP on) the response is only asserted within GPU-GFTT's tolerance, and the number of lists that differ is
printed. Without cv2 those tests skip. The numpy restatement of good_features_common equals the oracle, and each of its injected faults
changes the list on these inputs."""
import numpy as np
import pytest

import good_features_common as gc
from oracle import good_features_oracle


@pytest.fixture(scope="module")
def orc(oracle_lk):                 # oracle_lk builds oracle/libhv_oracle.so when it is missing
    return good_features_oracle.OracleGoodFeatures()


@pytest.fixture(scope="module")
def imgs():
    return gc.images()


@pytest.fixture(scope="module")
def cv2():
    return pytest.importorskip("cv2", reason="OpenCV (cv2) is not installed: nothing to compare the oracle with")


class _Baseline:
    """cv2's baseline path: no CPU dispatch, no IPP (restored afterwards)."""
    def __init__(self, cv2, optimized=False, ipp=False):
        self.cv2, self.want = cv2, (optimized, ipp)

    def __enter__(self):
        self.old = (self.cv2.useOptimized(), self.cv2.ipp.useIPP())
        self.cv2.setUseOptimized(self.want[0])
        self.cv2.ipp.setUseIPP(self.want[1])

    def __exit__(self, *exc):
        self.cv2.setUseOptimized(self.old[0])
        self.cv2.ipp.setUseIPP(self.old[1])


def cv_gftt(cv2, img, max_corners, quality, min_distance, mask):
    c, q = cv2.goodFeaturesToTrackWithQuality(np.ascontiguousarray(img), max_corners, quality, min_distance, mask, blockSize=3, gradientSize=3)
    if c is None:
        return np.zeros((0, 3), np.float32)
    return np.concatenate([c.reshape(-1, 2), q.reshape(-1, 1)], axis=1).astype(np.float32)


def _bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _sweep(imgs, orc):
    for name, img in imgs.items():
        eig = orc.eig(img)
        for mk in gc.MASKS:
            mask = gc.mask_for(mk, img, eig)
            for q in gc.QUALITIES:
                for md in gc.MIN_DISTANCES:
                    for mc in gc.MAX_CORNERS:
                        yield name, img, mask, mk, q, md, mc


def test_stages_bit_exact_vs_cv2_baseline(orc, cv2, imgs):
    print(f"cv2 {cv2.__version__}")
    with _Baseline(cv2):
        for name, img in imgs.items():
            dx, dy = orc.sobel(img)
            assert _bits(dx, cv2.Sobel(img, cv2.CV_32F, 1, 0, ksize=3, scale=1 / 3060)), f"{name}: Sobel dx"
            assert _bits(dy, cv2.Sobel(img, cv2.CV_32F, 0, 1, ksize=3, scale=1 / 3060)), f"{name}: Sobel dy"
            cov = np.stack([dx * dx, dx * dy, dy * dy], axis=2)
            box = cv2.boxFilter(cov, cv2.CV_32F, (3, 3), normalize=False, borderType=cv2.BORDER_REFLECT_101)
            assert _bits(orc.box(cov), box), f"{name}: boxFilter"
            assert _bits(orc.eig(img), cv2.cornerMinEigenVal(img, 3, ksize=3)), f"{name}: cornerMinEigenVal"


def test_list_bit_exact_vs_cv2_baseline(orc, cv2, imgs):
    with _Baseline(cv2):
        n = 0
        for name, img, mask, mk, q, md, mc in _sweep(imgs, orc):
            got, want = orc.detect(img, mc, q, md, mask), cv_gftt(cv2, img, mc, q, md, mask)
            assert _bits(got, want), f"{name} mask {mk} q {q} md {md} max {mc}: {len(got)} vs cv2 {len(want)}"
            n += 1
    print(f"cv2 {cv2.__version__}: {n} lists identical")


def test_response_within_tolerance_vs_cv2_defaults(orc, cv2, imgs):
    with _Baseline(cv2, optimized=True, ipp=True):
        worst, lists, differ = 0.0, 0, 0
        for name, img in imgs.items():
            r, e = cv2.cornerMinEigenVal(img, 3, ksize=3).astype(np.float64), orc.eig(img).astype(np.float64)
            d = np.abs(e - r)
            assert np.all(d <= 1e-6 + 1e-5 * np.abs(r)), f"{name}: response off by {d.max():.3g}"
            worst = max(worst, float(d.max()))
        for name, img, mask, mk, q, md, mc in _sweep(imgs, orc):
            lists += 1
            differ += not _bits(orc.detect(img, mc, q, md, mask), cv_gftt(cv2, img, mc, q, md, mask))
    print(f"cv2 {cv2.__version__} defaults: largest response difference {worst:.3g}; {differ} of {lists} lists differ")


def test_inputs_reach_every_branch(orc, imgs):
    """Thousands of candidates, lists cut by max_corners and by min_distance, equal responses, masks that change maxVal, and images
    without any candidate (the device tests add lists longer than a select round holds)."""
    big = orc.detect(imgs["noise"], 1 << 20, 1e-4, 0.0)
    assert len(big) > 4000
    per = orc.detect(imgs["periodic"], 1 << 20, 0.01, 0.0)
    assert len(per) - len(np.unique(per[:, 2])) > 100
    img = imgs["frame752"]
    eig = orc.eig(img)
    hide = gc.mask_for("hide_max", img, eig)
    assert eig[hide != 0].max() < eig.max()
    assert len(orc.detect(img, 150, 0.01, 10.0)) == 150 and len(orc.detect(img, 1 << 20, 0.01, 30.0)) < len(orc.detect(img, 1 << 20, 0.01, 0.0))
    assert len(orc.detect(imgs["flat"], 150, 0.01, 0.0)) == 0 and len(orc.detect(imgs["tiny1x1"], 150, 0.01, 0.0)) == 0


def test_numpy_restatement_equals_oracle(orc, imgs):
    for name, img in imgs.items():
        assert _bits(gc.eig_numpy(img), orc.eig(img)), f"{name}: response"
        eig = orc.eig(img)
        for mk in gc.MASKS:
            mask = gc.mask_for(mk, img, eig)
            for md in (0.0, 1.0, 10.0):
                assert _bits(gc.gftt_numpy(img, 150, 0.01, md, mask), orc.detect(img, 150, 0.01, md, mask)), f"{name} {mk} md {md}"


@pytest.mark.parametrize("fault", gc.FAULTS)
def test_inputs_catch_each_fault(orc, imgs, fault):
    """One injected fault at a time changes the list of at least one (image, mask, quality, min distance, budget) of the sweep."""
    caught = []
    for name, img in imgs.items():
        eig = orc.eig(img)
        for mk in gc.MASKS:
            mask = gc.mask_for(mk, img, eig)
            for q in (0.01, 1e-4, 1.0):
                for md in (0.0, 1.0, 10.0):
                    for mc in (150, 1 << 20):
                        if not _bits(gc.gftt_numpy(img, mc, q, md, mask, fault), orc.detect(img, mc, q, md, mask)):
                            caught.append((name, mk, q, md, mc))
            if caught:
                break
        if caught:
            break
    assert caught, f"no input tells the fault {fault} apart"
