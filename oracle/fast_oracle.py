"""TEST INFRASTRUCTURE: ctypes wrapper of the cv::FAST (TYPE_9_16) oracle (oracle/hv_oracle_fast.c)."""
import ctypes

import numpy as np

from oracle.gftt_oracle import ORACLE_SO


class OracleFast:
    def __init__(self):
        self.lib = ctypes.CDLL(ORACLE_SO)
        self.lib.orc_fast_detect.restype = ctypes.c_int
        self.lib.orc_fast_detect.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 5 + [ctypes.c_void_p, ctypes.c_int]

    def detect(self, img, threshold=10, nonmax=True):
        """cv2.FastFeatureDetector_create(threshold, nonmax, TYPE_9_16).detect(img) as (n, 3) float32 rows (x, y, response), in
        OpenCV's order. img: a 2-D uint8 array; a view with dense rows is read at its own row stride."""
        img = np.asarray(img)
        if img.dtype != np.uint8 or img.ndim != 2 or img.strides[1] != 1 or img.strides[0] < img.shape[1]:
            img = np.ascontiguousarray(img, np.uint8)
        h, w = img.shape
        f = self.lib.orc_fast_detect
        n = f(img.ctypes.data, img.strides[0], w, h, threshold, 1 if nonmax else 0, None, 0)
        assert n >= 0, "orc_fast_detect: out of memory"
        out = np.zeros((max(n, 1), 3), np.float32)
        assert f(img.ctypes.data, img.strides[0], w, h, threshold, 1 if nonmax else 0, out.ctypes.data, n) == n
        return out[:n]
