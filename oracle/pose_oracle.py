"""TEST INFRASTRUCTURE: ctypes wrapper of the cv::recoverPose oracle (oracle/hv_oracle_pose.c)."""
import ctypes

import numpy as np

from oracle.gftt_oracle import ORACLE_SO

_vp, _i, _d = ctypes.c_void_p, ctypes.c_int, ctypes.c_double


def _pts(a):
    return np.ascontiguousarray(a, np.float32).reshape(-1, 2)


class OraclePose:
    def __init__(self):
        self.lib = ctypes.CDLL(ORACLE_SO)
        L = self.lib
        L.orc_recover_pose_ex.argtypes = [_vp, _i, _vp, _vp, _vp, _i, _d, _d, _d, _d, _d, _vp, _vp, _vp, _vp, _vp, _vp]
        L.orc_recover_pose_ex.restype = _i
        L.orc_pose_decompose.argtypes = [_vp, _vp, _vp, _vp]
        L.orc_pose_decompose.restype = None

    def recover_pose(self, E, xy1, xy2, fx, fy, cx, cy, distance_thresh=50.0, mask=None, nsol=1, details=False):
        """The whole call as the C ABI computes it, E (3, 3) row-major. Returns (good, R (3, 3) row-major, t (3,), mask (n,) 0/1);
        details: also (flags (n, 4) per candidate before the input mask, Q (n, 4, 4) the candidates' null vectors)."""
        Ecm = np.ascontiguousarray(np.asarray(E, np.float64).reshape(3, 3).T).ravel()
        return self.recover_pose_cm(Ecm, xy1, xy2, fx, fy, cx, cy, distance_thresh, mask, nsol, details)

    def recover_pose_cm(self, Ecm, xy1, xy2, fx, fy, cx, cy, distance_thresh=50.0, mask=None, nsol=1, details=False):
        """As recover_pose, E as column-major doubles (the first 9 are used; the slots hv_find_essential writes)."""
        Ecm = np.ascontiguousarray(np.asarray(Ecm, np.float64).ravel()[:9])
        a, b = _pts(xy1), _pts(xy2)
        n = a.shape[0]
        mi = None if mask is None else np.ascontiguousarray(np.asarray(mask).reshape(-1), np.uint8)
        R, t = np.zeros(9), np.zeros(3)
        out = np.zeros(max(n, 1), np.uint8)
        good = ctypes.c_int(-1)
        flags = np.zeros((max(n, 1), 4), np.uint8) if details else None
        Q = np.zeros((max(n, 1), 4, 4)) if details else None
        rc = self.lib.orc_recover_pose_ex(Ecm.ctypes.data, nsol, a.ctypes.data, b.ctypes.data, None if mi is None else mi.ctypes.data, n,
                                          fx, fy, cx, cy, distance_thresh, R.ctypes.data, t.ctypes.data, out.ctypes.data,
                                          ctypes.byref(good), None if flags is None else flags.ctypes.data,
                                          None if Q is None else Q.ctypes.data)
        assert rc == 0, "orc_recover_pose_ex: out of memory"
        res = (good.value, R.reshape(3, 3).T.copy(), t, out[:n])
        return res + (flags[:n], Q[:n]) if details else res

    def decompose(self, E):
        """decomposeEssentialMat of a row-major (3, 3) E: (R1, R2, t)"""
        Ecm = np.ascontiguousarray(np.asarray(E, np.float64).reshape(3, 3).T).ravel()
        R1, R2, t = np.zeros(9), np.zeros(9), np.zeros(3)
        self.lib.orc_pose_decompose(Ecm.ctypes.data, R1.ctypes.data, R2.ctypes.data, t.ctypes.data)
        return R1.reshape(3, 3), R2.reshape(3, 3), t
