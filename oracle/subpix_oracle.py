"""TEST INFRASTRUCTURE: ctypes wrapper of the cornerSubPix oracle (oracle/hv_oracle_subpix.c)."""
import ctypes

import numpy as np

from oracle.gftt_oracle import ORACLE_SO

FLOAT_ACC, NO_REVERT, CLAMP = 1, 2, 4          # injectable faults (hv_oracle_subpix.c)
COUNT, EPS = 1, 2                              # cv::TermCriteria types


class OracleSubpix:
    def __init__(self):
        self.lib = ctypes.CDLL(ORACLE_SO)
        self.lib.orc_subpix_refine.restype = ctypes.c_int
        self.lib.orc_subpix_refine.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 3 + [ctypes.c_void_p] + [ctypes.c_int] * 7 + [ctypes.c_double, ctypes.c_int]
        self.lib.orc_rect_subpix.restype = None
        self.lib.orc_rect_subpix.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 5 + [ctypes.c_float] * 2 + [ctypes.c_void_p, ctypes.c_int]

    def refine(self, img, xy, win=(5, 5), zero_zone=(-1, -1), criteria=(COUNT | EPS, 30, 0.01), faults=0):
        """cv2.cornerSubPix(img, xy, win, zero_zone, criteria) with IPP off; returns a new (n, 2) float32 array, None where cv asserts."""
        img = np.ascontiguousarray(img, np.uint8)
        out = np.ascontiguousarray(xy, np.float32).reshape(-1, 2).copy()
        h, w = img.shape
        rc = self.lib.orc_subpix_refine(img.ctypes.data, w, w, h, out.ctypes.data, len(out), win[0], win[1], zero_zone[0], zero_zone[1],
                                        criteria[0], criteria[1], criteria[2], faults)
        return None if rc else out

    def rect(self, img, size, center, faults=0):
        """cv2.getRectSubPix(img, size, center, patchType=CV_32F)."""
        img = np.ascontiguousarray(img, np.uint8)
        h, w = img.shape
        out = np.zeros((size[1], size[0]), np.float32)
        self.lib.orc_rect_subpix(img.ctypes.data, w, w, h, size[0], size[1], center[0], center[1], out.ctypes.data, faults)
        return out
