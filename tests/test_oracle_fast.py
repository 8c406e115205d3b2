"""CPU: the cv::FAST oracle (oracle/hv_oracle_fast.c) against cv2.FastFeatureDetector_create(threshold, nonmax, TYPE_9_16) with IPP off
and on, BIT for bit -- count, order, x, y and response -- over the images of fast_common at every threshold of THRESHOLDS, with and
without suppression; plus checks that need no cv2: the numpy restatement of fast_common equals the oracle, and each of its injected faults
(>= in the suppression, a 4-pixel border, a score off by one, an arc of 8, column-major order) changes the list on these inputs.

cv2's vector loop reads the threshold as (char)threshold before FAST_t clamps it, so outside [0, 255] cv2 tests most columns at
threshold & 255 and only the last few (where its vector loop ends, which depends on the build's SIMD width) at the clamped value. The
oracle and the device clamp everywhere, so thresholds -5 and 300 are compared with cv2 at the clamped threshold."""
import numpy as np
import pytest

import fast_common as fc
from oracle import fast_oracle


@pytest.fixture(scope="module")
def orc(oracle_lk):                 # oracle_lk builds oracle/libhv_oracle.so when it is missing
    return fast_oracle.OracleFast()


@pytest.fixture(scope="module")
def imgs():
    return fc.images()


@pytest.fixture(scope="module")
def cv2():
    return pytest.importorskip("cv2", reason="OpenCV (cv2) is not installed: nothing to compare the oracle with")


def cv_fast(cv2, img, threshold, nonmax):
    det = cv2.FastFeatureDetector_create(threshold, nonmax, cv2.FAST_FEATURE_DETECTOR_TYPE_9_16)
    kp = det.detect(np.ascontiguousarray(img))
    return np.array([[k.pt[0], k.pt[1], k.response] for k in kp], np.float32).reshape(-1, 3)


def assert_same(got, want, what):
    assert got.shape == want.shape, f"{what}: {len(got)} keypoints, expected {len(want)}"
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"{what}: first difference at {np.nonzero((got != want).any(axis=1))[0][:5]}"


@pytest.mark.parametrize("ipp", [False, True], ids=["ipp_off", "ipp_on"])
@pytest.mark.parametrize("threshold", fc.THRESHOLDS)
def test_oracle_bit_exact_vs_cv2(orc, cv2, imgs, threshold, ipp):
    old = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(ipp)
    try:
        for name, img in imgs.items():
            for nonmax in (True, False):
                assert_same(orc.detect(img, threshold, nonmax), cv_fast(cv2, img, fc.clamp(threshold), nonmax), f"{name} t {threshold} nonmax {nonmax}")
    finally:
        cv2.ipp.setUseIPP(old)


def test_inputs_reach_every_branch(orc, imgs):
    """The sweep has corners of both polarities, suppressed and kept corners, keypoints on the first and last candidate rows and columns,
    responses from the threshold up to the top of the score range, and images without any keypoint."""
    total_kept = total_corners = 0
    first_last = set()
    resp = []
    for name, img in imgs.items():
        h, w = img.shape
        for t in fc.THRESHOLDS:
            kept, allc = orc.detect(img, t, True), orc.detect(img, t, False)
            total_kept += len(kept); total_corners += len(allc)
            resp += list(kept[:, 2])
            for x, y, _ in allc:
                first_last |= {("x3" if x == 3 else "xw" if x == w - 4 else ""), ("y3" if y == 3 else "yh" if y == h - 4 else "")}
    assert 0 < total_kept < total_corners
    assert {"x3", "xw", "y3", "yh"} <= first_last
    assert min(resp) <= 1 and max(resp) >= 150          # a score-0 corner never beats its neighbours (all >= 0)
    assert len(orc.detect(imgs["flat"], 0, True)) == 0 and len(orc.detect(imgs["tiny6x6"], 0, False)) == 0
    assert len(orc.detect(imgs["tiny7x7_corner"], 10, True)) == 1
    y, x = np.mgrid[-3:4, -3:4]
    bright = np.where(x * x + y * y >= 8, 220, 90).astype(np.uint8)    # a bright ring around a dark centre
    assert len(orc.detect(bright, 10, False)) == 1
    assert len(orc.detect(255 - bright, 10, False)) == 1              # and the opposite polarity


def test_oracle_reads_a_view_at_its_stride(orc, imgs):
    img = imgs["frame751x479"]
    padded = np.zeros((img.shape[0], img.shape[1] + 13), np.uint8)
    padded[:, :img.shape[1]] = img
    view = padded[:, :img.shape[1]]
    assert_same(orc.detect(view, 10, True), orc.detect(np.ascontiguousarray(view), 10, True), "strided view")


def test_numpy_restatement_equals_oracle(orc, imgs):
    for name, img in imgs.items():
        for t in fc.THRESHOLDS:
            for nonmax in (True, False):
                assert_same(fc.fast_numpy(img, t, nonmax), orc.detect(img, t, nonmax), f"{name} t {t} nonmax {nonmax}")


@pytest.mark.parametrize("fault", fc.FAULTS)
def test_inputs_catch_each_fault(orc, imgs, fault):
    """One injected fault at a time changes the list of at least one (image, threshold, suppression) of the sweep."""
    caught = []
    for name, img in imgs.items():
        for t in fc.THRESHOLDS:
            for nonmax in (True, False):
                got, want = fc.fast_numpy(img, t, nonmax, fault), orc.detect(img, t, nonmax)
                if got.shape != want.shape or not np.array_equal(got, want):
                    caught.append((name, t, nonmax))
    assert caught, f"no input tells the fault {fault} apart"
