"""TEST INFRASTRUCTURE: ctypes wrappers of the frame-ingest oracle (orc_gray / orc_remap in oracle/hv_oracle_gftt.c) and of the compiled
reference (oracle/_ref/libref_ingest.so: accelerated-arrays colour -> gray, src/tracker/undistorter.cpp)."""
import ctypes
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_SO = os.path.join(HERE, "libhv_oracle.so")
REF_SO = os.path.join(HERE, "_ref", "libref_ingest.so")
REMAP_DTYPE = np.dtype([("x0", np.int16), ("y0", np.int16), ("xfrac", np.float32), ("yfrac", np.float32)])
INVALID = -32768
GRAY_COEFF = (0.299, 0.587, 0.114, 0.0)


def have_ref():
    return os.path.exists(REF_SO)


def _rows(img, channels):
    """(image, row stride in bytes): a uint8 view whose rows are dense keeps its own stride (the reference reads its image as it lies in
    memory, padding bytes after a row included); any other layout is copied."""
    img = np.asarray(img)
    dense = (channels, 1) if img.ndim == 3 else (1,)
    if img.dtype != np.uint8 or img.strides[1:] != dense or img.strides[0] < img.shape[1] * channels:
        img = np.ascontiguousarray(img, np.uint8)
    return img, img.strides[0]


class OracleIngest:
    def __init__(self):
        self.lib = ctypes.CDLL(ORACLE_SO)

    def gray(self, img, coeff=GRAY_COEFF):
        h, w, c = np.shape(img)
        img, stride = _rows(img, c)
        cf = np.array([np.float32(x) for x in coeff[:c]], np.float32)      # the reference stores the coefficients as fp32
        out = np.zeros((h, w), np.uint8)
        self.lib.orc_gray(img.ctypes.data_as(ctypes.c_void_p), ctypes.c_int(stride), ctypes.c_int(c), ctypes.c_int(w), ctypes.c_int(h),
                          cf.ctypes.data_as(ctypes.c_void_p), out.ctypes.data_as(ctypes.c_void_p))
        return out

    def remap(self, img, table):
        """A tap right of the last column reads the first byte after the row in memory: for a view into a wider buffer that is the view's
        padding, for a contiguous image the first pixel of the next row."""
        h, w = np.shape(img)
        img, stride = _rows(img, 1)
        table = np.ascontiguousarray(table, REMAP_DTYPE)
        assert table.size == w * h and REMAP_DTYPE.itemsize == 12
        out = np.zeros((h, w), np.uint8)
        self.lib.orc_remap(img.ctypes.data_as(ctypes.c_void_p), ctypes.c_int(stride), ctypes.c_int(w), ctypes.c_int(h), table.ctypes.data_as(ctypes.c_void_p),
                           out.ctypes.data_as(ctypes.c_void_p))
        return out


class RefIngest:
    def __init__(self):
        self.lib = ctypes.CDLL(REF_SO)
        self.lib.hv_ref_undistort_mono.restype = ctypes.c_int

    def gray(self, img):
        img = np.ascontiguousarray(img, np.uint8)
        h, w, c = img.shape
        out = np.zeros((h, w), np.uint8)
        self.lib.hv_ref_gray(img.ctypes.data_as(ctypes.c_void_p), ctypes.c_int(w), ctypes.c_int(h), ctypes.c_int(c), out.ctypes.data_as(ctypes.c_void_p))
        return out

    def undistort(self, img, fisheye, fx, fy, cx, cy, dist, zoom=1.0):
        """Undistorter::buildMono(...)->undistort: returns (image, table of the same camera pair)."""
        img = np.ascontiguousarray(img, np.uint8)
        h, w = img.shape
        dist = np.ascontiguousarray(dist, np.float64)
        out = np.zeros((h, w), np.uint8)
        table = np.zeros(w * h, REMAP_DTYPE)
        rc = self.lib.hv_ref_undistort_mono(img.ctypes.data_as(ctypes.c_void_p), ctypes.c_int(w), ctypes.c_int(h), ctypes.c_int(int(fisheye)),
                                            ctypes.c_double(fx), ctypes.c_double(fy), ctypes.c_double(cx), ctypes.c_double(cy),
                                            dist.ctypes.data_as(ctypes.c_void_p), ctypes.c_int(len(dist)), ctypes.c_double(zoom),
                                            out.ctypes.data_as(ctypes.c_void_p), table.ctypes.data_as(ctypes.c_void_p))
        assert rc == 0
        return out, table
