"""Shared inputs of the FAST tests (test_oracle_fast.py on the CPU, test_gpu_fast.py on the device): images that reach every branch of
cv::FAST (TYPE_9_16) -- synthetic frames, noise, blurred noise, flat, checkerboard and step images, widths that are no multiple of 4 or
16, images smaller than 7 x 7 -- the thresholds to run them at, and a numpy restatement of the detector with one injectable fault at a
time, which shows that these inputs tell the mistakes a kernel could make apart from the right list."""
import numpy as np

from hybvio_b200 import synth

THRESHOLDS = (-5, 0, 1, 10, 20, 254, 255, 300)
FAULTS = ("ge_nms", "border4", "score_off", "arc8", "colmajor")
CIRCLE = ((0, 3), (1, 3), (2, 2), (3, 1), (3, 0), (3, -1), (2, -2), (1, -3),
          (0, -3), (-1, -3), (-2, -2), (-3, -1), (-3, 0), (-3, 1), (-2, 2), (-1, 3))     # makeOffsets(16) as (dx, dy)


def _blur(a, passes=2):
    """Separable [1 2 1] / 4 box passes with edge replication, in integers (no cv2 needed)."""
    a = a.astype(np.int32)
    for _ in range(passes):
        p = np.pad(a, 1, mode="edge")
        a = (p[1:-1, :-2] + 2 * p[1:-1, 1:-1] + p[1:-1, 2:] + 2) // 4
        p = np.pad(a, 1, mode="edge")
        a = (p[:-2, 1:-1] + 2 * p[1:-1, 1:-1] + p[2:, 1:-1] + 2) // 4
    return a.astype(np.uint8)


def images():
    rng = np.random.RandomState(11)
    out = {}
    out["frame752"] = synth.stereo_frame(2, 752, 480)[0]
    out["frame751x479"] = np.ascontiguousarray(synth.stereo_frame(5, 751, 479)[1])
    out["noise77x61"] = rng.randint(0, 256, (61, 77)).astype(np.uint8)
    out["blur_noise"] = _blur(rng.randint(0, 256, (240, 333)).astype(np.uint8))
    out["flat"] = np.full((40, 50), 97, np.uint8)
    y, x = np.mgrid[0:66, 0:70]
    out["checker"] = np.where(((x // 6) + (y // 6)) % 2 == 1, 210, 35).astype(np.uint8) + rng.randint(0, 4, (66, 70)).astype(np.uint8)
    step = np.full((45, 53), 60, np.uint8)
    step[:, 26:] = 190
    step[20:, :] //= 2
    step[np.arange(45)[:, None] > np.arange(53)[None, :] - 10] += 30     # a diagonal step as well
    out["step"] = step
    out["noise37x29"] = _blur(rng.randint(0, 256, (29, 37)).astype(np.uint8), 1)
    out["noise101x53"] = rng.randint(0, 256, (53, 101)).astype(np.uint8)
    for w, h in ((1, 1), (6, 6), (7, 7), (5, 9), (9, 5), (8, 7)):
        out[f"tiny{w}x{h}"] = rng.randint(0, 256, (h, w)).astype(np.uint8)
    out["tiny7x7_corner"] = np.full((7, 7), 200, np.uint8)
    out["tiny7x7_corner"][3, 3] = 20                                      # one dark-centre corner, the only candidate pixel
    return out


def clamp(t):
    return min(max(int(t), 0), 255)


def fast_numpy(img, threshold, nonmax, fault=None):
    """cv::FAST(img, threshold, nonmax, TYPE_9_16) as (n, 3) float32 rows (x, y, response) in OpenCV's order, with at most one of FAULTS."""
    img = np.asarray(img, np.uint8)
    h, w = img.shape
    t = clamp(threshold)
    b = 4 if fault == "border4" else 3
    arc = 8 if fault == "arc8" else 9
    if w < 2 * b + 1 or h < 2 * b + 1:
        return np.zeros((0, 3), np.float32)
    I = img.astype(np.int32)
    v = I[b:h - b, b:w - b]
    q = np.stack([I[b + dy:h - b + dy, b + dx:w - b + dx] for dx, dy in CIRCLE])
    corner = np.zeros(v.shape, bool)
    for m in (q < v - t, q > v + t):
        mm = np.concatenate([m, m[:arc - 1]])
        for k in range(16):
            corner |= mm[k:k + arc].all(axis=0)
    S = np.zeros((h, w), np.int32)
    C = np.zeros((h, w), bool)
    C[b:h - b, b:w - b] = corner
    if nonmax:
        d = v - q
        dd = np.concatenate([d, d[:8]])
        a0 = np.full(v.shape, t)
        b0 = np.full(v.shape, 255)
        for k in range(16):
            a0 = np.maximum(a0, dd[k:k + 9].min(axis=0))
            b0 = np.minimum(b0, dd[k:k + 9].max(axis=0))
        score = np.maximum(a0, -b0) - 1 + (1 if fault == "score_off" else 0)
        S[b:h - b, b:w - b] = np.where(corner, score, 0)
        P = np.pad(S, 1)
        keep = C.copy()
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                if dx or dy:
                    nb = P[1 + dy:h + 1 + dy, 1 + dx:w + 1 + dx]
                    keep &= (S >= nb) if fault == "ge_nms" else (S > nb)
    else:
        keep = C
    ys, xs = np.nonzero(keep)                       # row-major
    if fault == "colmajor":
        o = np.lexsort((ys, xs))
        ys, xs = ys[o], xs[o]
    return np.stack([xs, ys, S[ys, xs]], axis=1).astype(np.float32).reshape(-1, 3)
