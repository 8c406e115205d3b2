"""TEST INFRASTRUCTURE: ctypes wrapper of the cv::findEssentialMat (RANSAC) oracle (oracle/hv_oracle_essential.c)."""
import ctypes

import numpy as np

from oracle.gftt_oracle import ORACLE_SO

_vp, _i, _d = ctypes.c_void_p, ctypes.c_int, ctypes.c_double
MAX_SOL = 10


def _pts(a):
    return np.ascontiguousarray(a, np.float32).reshape(-1, 2)


class OracleEssential:
    def __init__(self):
        self.lib = ctypes.CDLL(ORACLE_SO)
        L = self.lib
        L.orc_find_essential.argtypes = [_vp, _vp, _vp, _i, _d, _d, _d, _d, _d, _d, _i, _vp, _vp, _vp, _vp]
        L.orc_find_essential.restype = _i
        L.orc_ess_solve5.argtypes = [_vp, _vp]
        L.orc_ess_solve5.restype = _i
        L.orc_ess_compact.argtypes = [_vp, _vp, _vp, _i, _d, _d, _d, _d, _vp, _vp]
        L.orc_ess_compact.restype = _i
        L.orc_ess_subsets.argtypes = [_i, _i, _vp]
        L.orc_ess_subsets.restype = None
        L.orc_ess_hypotheses.argtypes = [_vp, _i, _vp, _i, _vp, _vp, _vp]
        L.orc_ess_hypotheses.restype = _i
        L.orc_ess_update_niters.argtypes = [_d, _d, _i]
        L.orc_ess_update_niters.restype = _i

    def find_essential(self, xy1, xy2, fx, fy, cx, cy, prob=0.999, threshold=1.0, max_iters=1000, status=None):
        """The whole call: (E (10, 3, 3) column-major slots as the C ABI writes them, nsol, mask (n,) u8, inliers)."""
        a, b = _pts(xy1), _pts(xy2)
        n = a.shape[0]
        st = None if status is None else np.ascontiguousarray(status, np.uint8)
        E = np.zeros(90, np.float64)
        nsol, inl = ctypes.c_int(), ctypes.c_int()
        mask = np.zeros(max(n, 1), np.uint8)
        rc = self.lib.orc_find_essential(a.ctypes.data, b.ctypes.data, None if st is None else st.ctypes.data, n, fx, fy, cx, cy, prob,
                                         threshold, max_iters, E.ctypes.data, ctypes.byref(nsol), mask.ctypes.data, ctypes.byref(inl))
        assert rc == 0, "orc_find_essential: out of memory"
        return E.reshape(10, 3, 3), nsol.value, mask[:n], inl.value

    def find_essential_cv(self, *args, **kw):
        """As cv2.findEssentialMat returns it: (E (nsol, 3, 3) row-major, mask (n,) u8)."""
        E, nsol, mask, _ = self.find_essential(*args, **kw)
        return np.ascontiguousarray(E[:nsol].transpose(0, 2, 1)), mask

    def compact(self, xy1, xy2, fx, fy, cx, cy, status=None):
        """(q (m, 4) normalised (x1, y1, x2, y2), original indices (m,))"""
        a, b = _pts(xy1), _pts(xy2)
        n = a.shape[0]
        st = None if status is None else np.ascontiguousarray(status, np.uint8)
        q = np.zeros((max(n, 1), 4), np.float64)
        idx = np.zeros(max(n, 1), np.int32)
        m = self.lib.orc_ess_compact(a.ctypes.data, b.ctypes.data, None if st is None else st.ctypes.data, n, fx, fy, cx, cy,
                                     q.ctypes.data, idx.ctypes.data)
        return q[:m], idx[:m]

    def solve5(self, q):
        """Every solution (k, 3, 3) row-major of five normalised correspondences q (5, 4)."""
        q = np.ascontiguousarray(q, np.float64)
        assert q.shape == (5, 4)
        S = np.zeros(90, np.float64)
        k = self.lib.orc_ess_solve5(q.ctypes.data, S.ctypes.data)
        return S[:9 * k].reshape(k, 3, 3)

    def subsets(self, m, iters):
        sub = np.zeros((max(iters, 1), 5), np.int32)
        self.lib.orc_ess_subsets(m, iters, sub.ctypes.data)
        return sub[:iters]

    def hypotheses(self, q, sub, errors=True):
        """Per subset: (nsols (iters,), solutions (iters, 10, 3, 3) row-major, Sampson errors (iters, 10, m) in double, inf past nsol)."""
        q = np.ascontiguousarray(q, np.float64)
        sub = np.ascontiguousarray(sub, np.int32)
        iters, m = sub.shape[0], q.shape[0]
        ns = np.zeros(iters, np.int32)
        S = np.zeros((iters, 10, 9), np.float64)
        err = np.zeros((iters, 10, m), np.float64) if errors else None
        self.lib.orc_ess_hypotheses(q.ctypes.data, m, sub.ctypes.data, iters, ns.ctypes.data, S.ctypes.data,
                                    None if err is None else err.ctypes.data)
        return ns, S.reshape(iters, 10, 3, 3), err

    def update_niters(self, p, ep, niters):
        return self.lib.orc_ess_update_niters(p, ep, niters)
