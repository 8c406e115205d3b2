"""TEST INFRASTRUCTURE: ctypes wrapper of the cv::triangulatePoints oracle (oracle/hv_oracle_triangulate.c)."""
import ctypes

import numpy as np

from oracle.gftt_oracle import ORACLE_SO

_vp, _i = ctypes.c_void_p, ctypes.c_int


def _P(P):
    P = np.ascontiguousarray(np.asarray(P, np.float64).reshape(3, 4))
    return P


def _pts(a):
    return np.ascontiguousarray(a, np.float32).reshape(-1, 2)


def _u8(a):
    return None if a is None else np.ascontiguousarray(np.asarray(a).reshape(-1), np.uint8)


class OracleTriangulate:
    def __init__(self):
        self.lib = ctypes.CDLL(ORACLE_SO)
        L = self.lib
        L.orc_triangulate_points_ex.argtypes = [_vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _i]
        L.orc_triangulate_points_ex.restype = None
        L.orc_triangulate_one.argtypes = [_vp, _vp, _vp, _vp, _vp, _vp]
        L.orc_triangulate_one.restype = None

    def triangulate(self, P1, P2, xy1, xy2, status=None, status2=None, sort=True):
        """The whole call as the C ABI computes it: xy1, xy2 (n, 2) float32 (converted). Returns (X4 (4, n) float32, xyz (n, 3) float32,
        used (n,) uint8). sort=False leaves OpenCV's final selection sort out."""
        P1, P2, a, b = _P(P1), _P(P2), _pts(xy1), _pts(xy2)
        n = a.shape[0]
        assert b.shape[0] == n
        s1, s2 = _u8(status), _u8(status2)
        X4 = np.zeros((4, max(n, 1)), np.float32)
        xyz = np.zeros((max(n, 1), 3), np.float32)
        used = np.zeros(max(n, 1), np.uint8)
        self.lib.orc_triangulate_points_ex(P1.ctypes.data, P2.ctypes.data, a.ctypes.data, b.ctypes.data,
                                           None if s1 is None else s1.ctypes.data, None if s2 is None else s2.ctypes.data, n,
                                           X4.ctypes.data, xyz.ctypes.data, used.ctypes.data, 1 if sort else 0)
        return X4.reshape(-1)[:4 * n].reshape(4, n), xyz[:n], used[:n]

    def one(self, P1, P2, x1, x2):
        """One point's null vector in double (before rounding to float) and the number of Jacobi sweeps"""
        P1, P2 = _P(P1), _P(P2)
        a, b = np.ascontiguousarray(x1, np.float32).ravel(), np.ascontiguousarray(x2, np.float32).ravel()
        Q = np.zeros(4)
        sw = ctypes.c_int(-1)
        self.lib.orc_triangulate_one(P1.ctypes.data, P2.ctypes.data, a.ctypes.data, b.ctypes.data, Q.ctypes.data, ctypes.byref(sw))
        return Q, sw.value
