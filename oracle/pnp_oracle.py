"""TEST INFRASTRUCTURE: ctypes wrapper of the cv::solvePnPRansac (SOLVEPNP_P3P) oracle (oracle/hv_oracle_pnp.c)."""
import ctypes

import numpy as np

from oracle.gftt_oracle import ORACLE_SO

_vp, _i, _d, _f = ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_float


class OraclePnp:
    def __init__(self):
        self.lib = ctypes.CDLL(ORACLE_SO)
        L = self.lib
        L.orc_solve_pnp_ransac.argtypes = [_vp, _vp, _vp, _i, _d, _d, _d, _d, _i, _f, _d, _vp, _vp, _vp, _vp, _vp]
        L.orc_solve_pnp_ransac.restype = _i
        L.orc_pnp_p3p.argtypes = [_vp, _vp, _d, _d, _d, _d, _vp, _vp]
        L.orc_pnp_p3p.restype = _i
        L.orc_pnp_model4.argtypes = [_vp, _vp, _d, _d, _d, _d, _vp]
        L.orc_pnp_model4.restype = _i
        L.orc_pnp_epnp.argtypes = [_vp, _vp, _i, _d, _d, _d, _d, _vp, _vp]
        L.orc_pnp_epnp.restype = None
        L.orc_pnp_rodrigues_v2r.argtypes = [_vp, _vp]
        L.orc_pnp_rodrigues_r2v.argtypes = [_vp, _vp]
        L.orc_pnp_sincos.argtypes = [_d, _vp, _vp]
        L.orc_pnp_atan2.argtypes = [_d, _d]
        L.orc_pnp_atan2.restype = _d
        L.orc_pnp_subsets.argtypes = [_i, _i, _vp]
        L.orc_pnp_subsets.restype = None
        L.orc_pnp_update_niters.argtypes = [_d, _d, _i]
        L.orc_pnp_update_niters.restype = _i
        L.orc_pnp_grunert.argtypes = [_vp, _vp, _vp, _vp, _vp]
        L.orc_pnp_grunert.restype = _i

    def solve_pnp_ransac(self, xyz, xy, fx, fy, cx, cy, iterations=100, reproj_error=8.0, confidence=0.99, status=None):
        """The whole call as the C ABI computes it: (ok, rvec (3,), tvec (3,), mask (n,) u8, inliers)."""
        X = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
        x = np.ascontiguousarray(xy, np.float32).reshape(-1, 2)
        n = X.shape[0]
        st = None if status is None else np.ascontiguousarray(status, np.uint8)
        r, t = np.zeros(3), np.zeros(3)
        mask = np.zeros(max(n, 1), np.uint8)
        inl, ok = ctypes.c_int(), ctypes.c_int()
        rc = self.lib.orc_solve_pnp_ransac(X.ctypes.data, x.ctypes.data, None if st is None else st.ctypes.data, n, fx, fy, cx, cy,
                                           iterations, reproj_error, confidence, r.ctypes.data, t.ctypes.data, mask.ctypes.data,
                                           ctypes.byref(inl), ctypes.byref(ok))
        assert rc == 0, "orc_solve_pnp_ransac: out of memory"
        return ok.value, r, t, mask[:n], inl.value

    def p3p(self, X3, x3, fx, fy, cx, cy):
        """Every P3P pose of three world points (3, 3) at three pixels (3, 2): list of (R (3, 3), t (3,)), in ascending v = s3 / s1."""
        X = np.ascontiguousarray(X3, np.float64).reshape(9)
        x = np.ascontiguousarray(x3, np.float32).reshape(6)
        Rs, ts = np.zeros(36), np.zeros(12)
        k = self.lib.orc_pnp_p3p(X.ctypes.data, x.ctypes.data, fx, fy, cx, cy, Rs.ctypes.data, ts.ctypes.data)
        return [(Rs[9 * i:9 * i + 9].reshape(3, 3).copy(), ts[3 * i:3 * i + 3].copy()) for i in range(k)]

    def model4(self, X4, x4, fx, fy, cx, cy):
        """The RANSAC kernel on four points: (rvec, tvec) or None."""
        X = np.ascontiguousarray(X4, np.float64).reshape(12)
        x = np.ascontiguousarray(x4, np.float32).reshape(8)
        mdl = np.zeros(6)
        if not self.lib.orc_pnp_model4(X.ctypes.data, x.ctypes.data, fx, fy, cx, cy, mdl.ctypes.data):
            return None
        return mdl[:3].copy(), mdl[3:].copy()

    def epnp(self, X, x, fx, fy, cx, cy):
        """EPnP of (n, 3) world points at (n, 2) pixels (OpenCV's undistort round trip applied here): (rvec (3,), tvec (3,))."""
        pw = np.ascontiguousarray(X, np.float64).reshape(-1, 3)
        x = np.asarray(x, np.float64).reshape(-1, 2)
        us = np.ascontiguousarray(np.c_[((x[:, 0] - cx) * (1.0 / fx)) * fx + cx, ((x[:, 1] - cy) * (1.0 / fy)) * fy + cy])
        R, t, r = np.zeros(9), np.zeros(3), np.zeros(3)
        self.lib.orc_pnp_epnp(pw.ctypes.data, us.ctypes.data, pw.shape[0], fx, fy, cx, cy, R.ctypes.data, t.ctypes.data)
        self.lib.orc_pnp_rodrigues_r2v(R.ctypes.data, r.ctypes.data)
        return r, t

    def rodrigues(self, v):
        """rvec (3,) -> R (3, 3), or R (3, 3) -> rvec (3,)"""
        a = np.ascontiguousarray(v, np.float64)
        if a.size == 3:
            R = np.zeros(9)
            self.lib.orc_pnp_rodrigues_v2r(a.ctypes.data, R.ctypes.data)
            return R.reshape(3, 3)
        r = np.zeros(3)
        self.lib.orc_pnp_rodrigues_r2v(a.reshape(9).ctypes.data, r.ctypes.data)
        return r

    def sincos(self, th):
        s, c = ctypes.c_double(), ctypes.c_double()
        self.lib.orc_pnp_sincos(th, ctypes.byref(s), ctypes.byref(c))
        return s.value, c.value

    def atan2(self, y, x):
        return self.lib.orc_pnp_atan2(y, x)

    def grunert(self, X3, f3):
        """Grunert's quartic (5, 2) double-double (hi, lo), u's numerator (3,) and denominator (2,) for world points (3, 3) and unit rays (3, 3); None if degenerate."""
        X = np.ascontiguousarray(X3, np.float64).reshape(9)
        f = np.ascontiguousarray(f3, np.float64).reshape(9)
        P, N, D = np.zeros(10), np.zeros(3), np.zeros(2)
        if not self.lib.orc_pnp_grunert(X.ctypes.data, f.ctypes.data, P.ctypes.data, N.ctypes.data, D.ctypes.data):
            return None
        return P.reshape(5, 2), N, D

    def subsets(self, m, iters):
        sub = np.zeros((max(iters, 1), 4), np.int32)
        self.lib.orc_pnp_subsets(m, iters, sub.ctypes.data)
        return sub[:iters]

    def update_niters(self, p, ep, niters):
        return self.lib.orc_pnp_update_niters(p, ep, niters)
