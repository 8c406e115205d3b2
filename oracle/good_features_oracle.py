"""TEST INFRASTRUCTURE: ctypes wrapper of the cv::goodFeaturesToTrack (Shi-Tomasi) oracle (oracle/hv_oracle_good_features.c)."""
import ctypes

import numpy as np

from oracle.gftt_oracle import ORACLE_SO

_vp, _i, _d = ctypes.c_void_p, ctypes.c_int, ctypes.c_double


def _image(img):
    img = np.asarray(img)
    if img.dtype != np.uint8 or img.ndim != 2 or img.strides[1] != 1 or img.strides[0] < img.shape[1]:
        img = np.ascontiguousarray(img, np.uint8)
    return img


class OracleGoodFeatures:
    def __init__(self):
        self.lib = ctypes.CDLL(ORACLE_SO)
        self.lib.orc_gf_sobel.argtypes = [_vp, _i, _i, _i, _vp, _vp]
        self.lib.orc_gf_box.argtypes = [_vp, _i, _i, _vp]
        self.lib.orc_gf_box.restype = _i
        self.lib.orc_gf_eig.argtypes = [_vp, _i, _i, _i, _vp]
        self.lib.orc_gf_eig.restype = _i
        self.lib.orc_gf_detect.argtypes = [_vp, _i, _i, _i, _i, _d, _d, _vp, _i, _vp, _i]
        self.lib.orc_gf_detect.restype = _i

    def sobel(self, img):
        """(dx, dy) float32 maps: cv2.Sobel(img, CV_32F, 1, 0 / 0, 1, ksize=3, scale=1/3060)."""
        img = _image(img)
        h, w = img.shape
        dx, dy = np.zeros((h, w), np.float32), np.zeros((h, w), np.float32)
        self.lib.orc_gf_sobel(img.ctypes.data, img.strides[0], w, h, dx.ctypes.data, dy.ctypes.data)
        return dx, dy

    def box(self, cov):
        """cv2.boxFilter(cov, CV_32F, (3, 3), normalize=False) of an (h, w, 3) float32 image (reflect-101)."""
        cov = np.ascontiguousarray(cov, np.float32)
        h, w, _ = cov.shape
        out = np.zeros_like(cov)
        assert self.lib.orc_gf_box(cov.ctypes.data, w, h, out.ctypes.data) == 0, "orc_gf_box: out of memory"
        return out

    def eig(self, img):
        """cv2.cornerMinEigenVal(img, 3, 3) as a float32 map."""
        img = _image(img)
        h, w = img.shape
        out = np.zeros((h, w), np.float32)
        assert self.lib.orc_gf_eig(img.ctypes.data, img.strides[0], w, h, out.ctypes.data) == 0, "orc_gf_eig: out of memory"
        return out

    def detect(self, img, max_corners, quality_level, min_distance, mask=None):
        """cv2.goodFeaturesToTrack(img, max_corners, quality_level, min_distance, mask=mask, blockSize=3, gradientSize=3,
        useHarrisDetector=False) with cornersQuality, as (n, 3) float32 rows (x, y, response) in OpenCV's order."""
        img = _image(img)
        h, w = img.shape
        mp, ms = None, 0
        if mask is not None:
            mask = _image(mask)
            assert mask.shape == img.shape
            mp, ms = mask.ctypes.data, mask.strides[0]
        f = self.lib.orc_gf_detect
        n = f(img.ctypes.data, img.strides[0], w, h, max_corners, quality_level, min_distance, mp, ms, None, 0)
        assert n >= 0, "orc_gf_detect: out of memory"
        out = np.zeros((max(n, 1), 3), np.float32)
        assert f(img.ctypes.data, img.strides[0], w, h, max_corners, quality_level, min_distance, mp, ms, out.ctypes.data, n) == n
        return out[:n]
