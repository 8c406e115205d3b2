"""Shared inputs of the Shi-Tomasi (cv::goodFeaturesToTrack) tests (test_oracle_good_features.py on the CPU, test_gpu_good_features.py
on the device): the images of fast_common plus a linear ramp (every response is rounding noise: the sharpest test of operation order), a
periodic pattern (thousands of equal responses: tie order, and more keys of one value than a select round holds), raw noise to run
at quality 1e-4 (a very large candidate count) and dark noise under bright bars (dy of rounding noise below bright rows, where
boxFilter's running column sum differs from the exact 9-term sum); the masks, min distances and corner budgets to run them at; and a numpy restatement of
the detector with one injectable fault at a time, which shows that these inputs tell the mistakes a kernel could make apart from the
right list."""
import numpy as np

import fast_common

MIN_DISTANCES = (0.0, 0.5, 1.0, 2.5, 10.0, 30.0)
MAX_CORNERS = (1, 150, 1 << 20)          # the last is above every candidate count here
QUALITIES = (0.01, 1e-4, 1.0)        # 1.0: the threshold equals maxVal, so `>` leaves no candidate
MASKS = ("none", "half", "hide_max")
FAULTS = ("ties_ascending", "ge_threshold", "le_distance", "unmasked_max", "border", "fp32_box", "exact_box")


def images(large_noise=(240, 320)):
    out = dict(fast_common.images())
    y, x = np.mgrid[0:120, 0:160]
    out["ramp"] = (x + 2 * y).astype(np.uint8)
    out["periodic"] = np.where(((x // 4) + (y // 4)) % 2 == 1, 200, 50).astype(np.uint8)
    out["noise"] = np.random.RandomState(21).randint(0, 256, large_noise).astype(np.uint8)
    rng = np.random.RandomState(23)
    for k in range(6):
        img = rng.randint(0, 6, (120, 160)).astype(np.uint8)
        for _ in range(3):
            y0, x0 = rng.randint(0, 110), rng.randint(0, 150)
            img[y0:y0 + rng.randint(2, 10), x0:x0 + rng.randint(2, 40)] = rng.randint(150, 256)
        out[f"dark_bars{k}"] = img
    return out


def mask_for(kind, img, eig):
    """None, the left half, or everything but a 9 x 9 block around the global maximum of eig (a maxVal taken without the mask then
    sets a threshold no unmasked pixel's response may reach)."""
    h, w = img.shape
    if kind == "none":
        return None
    m = np.zeros((h, w), np.uint8)
    if kind == "half":
        m[:, :w // 2] = 255
        return m
    m[:] = 1
    by, bx = np.unravel_index(int(np.argmax(eig)), eig.shape)
    m[max(by - 4, 0):by + 5, max(bx - 4, 0):bx + 5] = 0
    return m


def _reflect(n, lo, hi):
    """indices lo .. hi - 1 reflected (BORDER_REFLECT_101) into [0, n)"""
    i = np.arange(lo, hi)
    if n == 1:
        return np.zeros_like(i)
    while True:
        neg, big = i < 0, i >= n
        if not (neg.any() or big.any()):
            return i
        i = np.where(neg, -i, np.where(big, 2 * n - 2 - i, i))


def eig_numpy(img, fault=None):
    """cv::cornerMinEigenVal(img, 3, 3) in OpenCV's operation order (numpy float32 rounds every operation; float64 for boxFilter's row sums
    and running column sums)."""
    img = np.asarray(img, np.uint8)
    h, w = img.shape
    I = img.astype(np.float32)
    k1 = np.float32(1.0 / 3060.0)
    k0 = np.float32(2.0) * k1
    P = I[_reflect(h, -1, h + 1)][:, _reflect(w, -1, w + 1)]
    L, C, R = P[:, :-2], P[:, 1:-1], P[:, 2:]
    rdx = R - L
    rdy = (k1 * L + k0 * C) + k1 * R
    dx = rdx[1:-1] * k0 + (rdx[:-2] + rdx[2:]) * k1
    dy = rdy[2:] - rdy[:-2]
    cov = [dx * dx, dx * dy, dy * dy]
    ry, rx = _reflect(h, -1, h + 1), _reflect(w, -1, w + 1)
    sums = []
    for c in cov:
        Q = c[ry][:, rx]
        if fault == "fp32_box":              # GPU-GFTT's box: rows of rounded fp32 adds, then the rows
            rows = (Q[:, :-2] + Q[:, 1:-1]) + Q[:, 2:]
            sums.append((rows[:-2] + rows[1:-1]) + rows[2:])
        elif fault == "exact_box":           # the 9 products summed in double, not boxFilter's running column sum
            Q = Q.astype(np.float64)
            sums.append(sum(Q[dy_:dy_ + h, dx_:dx_ + w] for dy_ in range(3) for dx_ in range(3)).astype(np.float32))
        else:                                # RowSum ((a + b) + c) in double, then ColumnSum's running double sum from the top
            Q = Q.astype(np.float64)
            R = (Q[:, :-2] + Q[:, 1:-1]) + Q[:, 2:]          # rows -1 .. h (reflected)
            run = (0.0 + R[0]) + R[1]
            out = np.zeros((h, w), np.float32)
            for y in range(h):
                s0 = run + R[y + 2]
                out[y] = s0.astype(np.float32)
                run = s0 - R[y]
            sums.append(out)
    a, b, c = sums[0] * np.float32(0.5), sums[1], sums[2] * np.float32(0.5)
    t = a - c
    return (a + c) - np.sqrt(t * t + b * b)


def gftt_numpy(img, max_corners, quality, min_distance, mask=None, fault=None):
    """cv::goodFeaturesToTrack(img, max_corners, quality, min_distance, mask, 3, 3) as (n, 3) float32 rows (x, y, response), with at
    most one of FAULTS."""
    img = np.asarray(img, np.uint8)
    h, w = img.shape
    eig = eig_numpy(img, fault)
    sel = np.ones((h, w), bool) if mask is None or fault == "unmasked_max" else mask != 0
    max_val = float(eig[sel].max()) if sel.any() else 0.0
    thresh = np.float32(max_val * quality)
    e = np.where(eig >= thresh if fault == "ge_threshold" else eig > thresh, eig, np.float32(0))
    if h < 3 or w < 3:
        return np.zeros((0, 3), np.float32)
    P = np.pad(e, 1, constant_values=-np.inf)
    dil = np.max(np.stack([P[dy:dy + h, dx:dx + w] for dy in range(3) for dx in range(3)]), axis=0)
    cand = (e != 0) & (e == dil)
    if fault != "border":
        inner = np.zeros((h, w), bool)
        inner[1:-1, 1:-1] = True
        cand &= inner
    if mask is not None:
        cand &= mask != 0
    idx = np.flatnonzero(cand)
    v = e.ravel()[idx]
    order = np.lexsort((idx if fault == "ties_ascending" else -idx, -v.astype(np.float64)))
    idx, v = idx[order], v[order]
    ys, xs = idx // w, idx % w
    out = []
    if min_distance >= 1:
        md2 = min_distance * min_distance
        cell = int(np.rint(min_distance))
        grid = {}
        for x, y, val in zip(xs.tolist(), ys.tolist(), v.tolist()):
            cx, cy = x // cell, y // cell
            good = True
            for yy in range(cy - 1, cy + 2):
                for xx in range(cx - 1, cx + 2):
                    for kx, ky in grid.get((xx, yy), ()):
                        d2 = float(np.float32(np.float32(x - kx) ** 2 + np.float32(y - ky) ** 2))
                        if (d2 <= md2) if fault == "le_distance" else (d2 < md2):
                            good = False
                            break
                    if not good:
                        break
                if not good:
                    break
            if good:
                grid.setdefault((cx, cy), []).append((x, y))
                out.append((x, y, val))
                if len(out) == max_corners:
                    break
    else:
        out = list(zip(xs.tolist(), ys.tolist(), v.tolist()))[:max_corners]
    return np.array(out, np.float32).reshape(-1, 3)
