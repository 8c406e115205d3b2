"""Shared inputs of the cornerSubPix tests (test_oracle_subpix.py on the CPU, test_gpu_subpix.py on the device): images, start points
and the parameter sweep."""
import numpy as np

from hybvio_b200 import synth

WINDOWS = [(1, 1), (2, 3), (5, 5), (7, 7), (11, 11), (15, 15)]
# none; (0, 0); (1, 2); one that does not fit into the window (2 zero + 1 >= 2 win + 1 on an axis), which cv ignores
ZERO_ZONES = [(-1, -1), (0, 0), (1, 2), "too_large"]
# (type, max_count, epsilon): COUNT only, EPS only, both; max_count 0, 1, 100, 150 (clamped to 1..100); epsilon 0
CRITERIA = [(1, 0, 0.0), (1, 1, 0.0), (1, 100, 0.0), (1, 150, 0.0), (2, 30, 0.0), (2, 30, 0.01), (3, 30, 0.01), (3, 150, 0.0), (3, 0, 0.001)]
SQUARE = 16.0


def zero_zone(z, win):
    return (win[0], 0) if z == "too_large" else z


def blur(a, sigma):
    r = int(3 * sigma + 1)
    k = np.exp(-0.5 * (np.arange(-r, r + 1) / sigma) ** 2)
    k /= k.sum()
    p = np.pad(a, r, mode="edge")
    p = np.apply_along_axis(lambda v: np.convolve(v, k, mode="valid"), 1, p)
    return np.apply_along_axis(lambda v: np.convolve(v, k, mode="valid"), 0, p)


def checkerboard(w, h, ox, oy, sigma=1.2):
    """Blurred checkerboard of SQUARE-pixel squares whose corners lie at (ox + i SQUARE, oy + j SQUARE) (pixel centres at integer
    coordinates). The squares are the XOR of vertical and horizontal stripes, so a pixel's covered area is fx (1 - fy) + (1 - fx) fy with
    fx, fy the stripe fractions of its two unit intervals (1-D sampling at 1/256 px). Returns (image, inner corners (n, 2))."""
    s = 256
    off = (np.arange(s) + 0.5) / s - 0.5

    def stripe(n, o):
        u = np.arange(n)[:, None] + off[None, :]
        return (np.floor((u - o) / SQUARE).astype(int) & 1).mean(axis=1)

    fx, fy = stripe(w, ox), stripe(h, oy)
    img = (fx[None, :] * (1 - fy[:, None]) + (1 - fx[None, :]) * fy[:, None]) * 180.0 + 40.0
    img = np.clip(np.floor(blur(img, sigma) + 0.5), 0, 255).astype(np.uint8)
    gx = ox + SQUARE * np.arange(-2, int(w / SQUARE) + 2)
    gy = oy + SQUARE * np.arange(-2, int(h / SQUARE) + 2)
    pts = np.array([(x, y) for y in gy for x in gx if 20 <= x <= w - 21 and 20 <= y <= h - 21])
    return img, pts


def images():
    """name -> uint8 image: the synthetic camera frames (752 x 480 and 751 x 479: a level-0 pitch that is not the width), random texture,
    an image with flat patches (the det == 0 stop) and a blurred checkerboard."""
    rng = np.random.RandomState(11)
    flat = synth.stereo_frame(3, 200, 150)[0].copy()
    flat[20:90, 30:120] = 77
    flat[100:, :60] = 200
    return {
        "frame752": synth.stereo_frame(2, 752, 480)[0],
        "frame751": synth.stereo_frame(5, 751, 479)[1],
        "texture": rng.randint(0, 256, (97, 131)).astype(np.uint8),
        "flat": flat,
        "checker": checkerboard(160, 120, 20.3, 17.6)[0],
    }


def points(img, win, seed=0, n_random=60):
    """Start points: random, within win + 1 of every border (the border patch path), the exact borders (0 and w - 1e-4), integer and
    half-integer positions; float32 (n, 2)."""
    h, w = img.shape
    rng = np.random.RandomState(seed)
    p = [rng.uniform([0, 0], [w, h], (n_random, 2))]
    for side in range(4):
        d = rng.uniform(0, max(win) + 1, 6)
        u = rng.uniform(0, 1, 6)
        if side == 0: p.append(np.stack([d, u * h], 1))
        if side == 1: p.append(np.stack([w - 1e-4 - d, u * h], 1))
        if side == 2: p.append(np.stack([u * w, d], 1))
        if side == 3: p.append(np.stack([u * w, h - 1e-4 - d], 1))
    p.append(np.array([[0, 0], [w - 1e-4, h - 1e-4], [0, h - 1e-4], [w - 1e-4, 0], [w // 2, h // 2], [w // 3 + 0.5, h // 3 + 0.5],
                       [17, 9.5], [w - 1e-4, h // 2]]))
    out = np.concatenate(p).astype(np.float32)
    out[:, 0] = np.minimum(out[:, 0], np.float32(w) - np.float32(1e-4))      # float32 rounding must not push a point onto the border
    out[:, 1] = np.minimum(out[:, 1], np.float32(h) - np.float32(1e-4))
    return out
