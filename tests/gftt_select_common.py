"""Shared inputs of the corner-selection tests (test_emu_gftt_select.py on the CPU, test_gpu_gftt_select.py on the device): crafted key
point lists that stress the stable sort, the quirk, the rounded distance test and the cap, and a numpy restatement of the selection
(FeatureDetector::detect's tail, feature_detector.cpp:625-638) with one injectable fault at a time, which shows that these inputs tell
the mistakes a kernel could make apart from the right list."""
import struct

import numpy as np

F32 = np.float32
NONE = F32(-1.0e6)
MAX_KP = 16384
EMPTY = F32(-1e10)        # response of a cell without a qualifying pixel
FAULTS = ("unstable_sort", "less_equal", "fma_distance", "no_quirk", "cap_without_radius")


def capacity(nkp, mask_radius, max_tracks):
    return min(max_tracks, 2 * nkp) if mask_radius > 0 else 2 * nkp


def _kp(xy, resp):
    return np.concatenate([np.asarray(xy, F32).reshape(-1, 2), np.asarray(resp, F32).reshape(-1, 1)], axis=1)


def _ulp_neighbours(v, steps=2):
    """v and its `steps` float32 neighbours on either side (v a float32 scalar or array)."""
    v = np.asarray(v, F32) if np.ndim(v) else F32(v)
    out = [v]
    up = dn = v
    for _ in range(steps):
        up, dn = np.nextafter(up, F32(np.inf)), np.nextafter(dn, F32(-np.inf))
        out += [up, dn]
    return out


def circle_case(r, seed):
    """Key points on a coarse grid with, next to each, a point whose offset is one of the float neighbours of a point on the circle of
    radius r around it: the fp32 rounding of the squared distance decides. Half of the companions are previous corners, the other half
    key points of lower response (decided by the greedy test against kept points). Pythagorean offsets give sums exactly equal to r^2."""
    rng = np.random.RandomState(seed)
    spacing = 4 * r + 16
    kp_xy, kp_r, prev = [], [], []
    triples = [(3, 4, 5), (5, 12, 13), (8, 15, 17), (6, 8, 10), (0, 1, 1)]
    cell = 0
    for ang in np.linspace(0, 2 * np.pi, 24, endpoint=False):
        base = np.array([(cell % 20) * spacing + 3.0, (cell // 20) * spacing + 5.0], np.float64)
        px, py = base + r * np.array([np.cos(ang), np.sin(ang)])
        for ox in _ulp_neighbours(F32(px)):
            for oy in _ulp_neighbours(F32(py), 1):
                c = np.array([(cell % 20) * spacing + 3.0, (cell // 20) * spacing + 5.0], np.float64)
                shift = np.array([float(ox), float(oy)]) - base
                kp_xy.append(c); kp_r.append(1.0 + rng.rand())
                if cell % 2 == 0:
                    prev.append(c + shift)
                else:
                    kp_xy.append(c + shift); kp_r.append(0.5 * rng.rand())
                cell += 1
    for a, b, c in triples:
        if r % c == 0:
            k = r // c
            for sx, sy in ((a, b), (b, a), (-a, b), (a, -b)):
                base = np.array([(cell % 20) * spacing + 3.0, (cell // 20) * spacing + 5.0])
                kp_xy.append(base); kp_r.append(1.0 + rng.rand())
                (prev if cell % 2 == 0 else kp_xy).append(base + k * np.array([sx, sy], np.float64))
                if cell % 2:
                    kp_r.append(0.25)
                cell += 1
    return _kp(np.array(kp_xy, F32), np.array(kp_r, F32)), np.array(prev, F32).reshape(-1, 2)


def fma_case(r, centres=12):
    """Key points with a companion (previous corner for even, lower-response key point for odd centres) at an offset whose squared
    distance falls on the other side of r^2 when the distance is formed with a fused multiply-add, found by a search over the float
    neighbours of points on the circle (such offsets exist for r = 8 and 50, not for r = 1)."""
    r2 = F32(r * r)
    ang = np.linspace(0, 2 * np.pi, 4000, endpoint=False)
    kp_xy, kp_r, prev = [], [], []
    for k in range(centres):
        cx, cy = F32(1003 + 300 * k), F32(1005 + 7 * k)
        xs = _ulp_neighbours((cx + r * np.cos(ang)).astype(F32), 3)
        ys = _ulp_neighbours((cy + r * np.sin(ang)).astype(F32), 3)
        ox = np.stack(xs, 1)[:, :, None].repeat(len(ys), 2)
        oy = np.stack(ys, 1)[:, None, :].repeat(len(xs), 1)
        dx, dy = ox - cx, oy - cy
        d2 = dx * dx + dy * dy
        d2f = (dx.astype(np.float64) * dx + (dy * dy).astype(np.float64)).astype(F32)
        hit = np.argwhere((d2 < r2) != (d2f < r2))
        if len(hit) == 0:
            continue
        i, a, b = hit[0]
        kp_xy.append((cx, cy)); kp_r.append(1.0 + 0.01 * k)
        if k % 2 == 0:
            prev.append((ox[i, a, b], oy[i, a, b]))
        else:
            kp_xy.append((ox[i, a, b], oy[i, a, b])); kp_r.append(0.5)
    return _kp(np.array(kp_xy, F32).reshape(-1, 2), np.array(kp_r, F32)), np.array(prev, F32).reshape(-1, 2)


def random_kp(n, seed, w=752, h=480, empty=0.0):
    rng = np.random.RandomState(seed)
    xy = np.stack([rng.randint(0, w, n), rng.randint(0, h, n)], 1).astype(F32)
    resp = (rng.rand(n) * 0.3).astype(F32)
    e = rng.rand(n) < empty
    xy[e] = 0
    resp[e] = EMPTY
    return _kp(xy, resp)


def prev_points(m, seed, w=752, h=480):
    """Random previous corners with duplicates and one next to (0, 0)."""
    rng = np.random.RandomState(seed)
    if m == 0:
        return np.zeros((0, 2), F32)
    p = rng.uniform([0, 0], [w, h], (m, 2)).astype(F32)
    p[m // 2:m // 2 + m // 10] = p[:m // 10]
    p[-1] = (0.75, 0.5)
    return p


def crafted_cases(big=False):
    """[(name, kp (n, 3) float32, prev (m, 2) float32, mask_radius, max_tracks)]"""
    rng = np.random.RandomState(17)
    cases = []
    eq = random_kp(400, 1)
    eq[:, 2] = 0.5
    for r, m in ((0, 150), (8, 100000), (8, 7), (50, 150)):
        cases.append((f"equal_responses_r{r}_max{m}", eq, prev_points(40, 2), r, m))
    sz = random_kp(300, 3)
    sz[:, 2] = rng.choice(np.array([0.0, -0.0, 1e-3, -1e-3, 0.25], F32), 300)
    for r in (0, 20):
        cases.append((f"signed_zero_r{r}", sz, np.zeros((0, 2), F32), r, 100000))
    em = random_kp(600, 4, empty=0.8)
    for r, m in ((0, 150), (8, 100000), (50, 150), (1, 3)):
        cases.append((f"empty_cells_r{r}_max{m}", em, prev_points(40, 5), r, m))
    one = random_kp(1, 6)
    for r, prev in ((0, None), (8, None), (8, one[:, :2] + F32(2)), (8, np.array([[0.5, 0.5]], F32))):
        cases.append((f"one_key_point_r{r}", one, np.zeros((0, 2), F32) if prev is None else prev, r, 150))
    cases.append(("no_key_points", np.zeros((0, 3), F32), prev_points(40, 7), 8, 150))
    for r in (1, 8, 50):
        kp, prev = circle_case(r, r)
        cases.append((f"circle_neighbours_r{r}", kp, prev, r, 100000))
    for r in (8, 50):
        kp, prev = fma_case(r)
        cases.append((f"fma_sensitive_r{r}", kp, prev, r, 100000))
    two = random_kp(2500, 8, 1280, 720, empty=0.1)
    for r, m in ((8, 100000), (8, 150), (1, 100000), (50, 7), (0, 1)):
        cases.append((f"two_chunks_r{r}_max{m}", two, prev_points(500, 9, 1280, 720), r, m))
    cases.append(("zero_blocked_by_prev", random_kp(200, 10), np.array([[3.0, 4.0], [3.0, 4.0]], F32), 8, 150))
    cases.append(("max_one_zero_kept", random_kp(200, 11), np.zeros((0, 2), F32), 8, 1))
    if big:
        full = random_kp(MAX_KP, 12, 1280, 720, empty=0.05)
        for r, m in ((0, 150), (8, 100000), (8, 150)):
            cases.append((f"max_key_points_r{r}_max{m}", full, prev_points(500, 13, 1280, 720), r, m))
    return cases


def write_cases(path, cases):
    with open(path, "wb") as f:
        f.write(struct.pack("<i", len(cases)))
        for _, kp, prev, r, m in cases:
            f.write(struct.pack("<4i", len(kp), len(prev), r, m))
            f.write(np.ascontiguousarray(kp, F32).tobytes())
            f.write(np.ascontiguousarray(prev, F32).reshape(-1, 2).tobytes())


def _near(others, c, r2, fault):
    """applyMinDistance's test of point c against the points `others`: (o.x - c.x)^2 + (o.y - c.y)^2 < r2 in fp32."""
    if len(others) == 0:
        return False
    dx = others[:, 0] - c[0]
    dy = others[:, 1] - c[1]
    if fault == "fma_distance":
        d2 = (dx.astype(np.float64) * dx + (dy * dy).astype(np.float64)).astype(F32)
    else:
        d2 = dx * dx + dy * dy
    return bool(np.any(d2 <= r2) if fault == "less_equal" else np.any(d2 < r2))


def select(kp, prev, mask_radius, max_tracks, fault=None):
    """The selection restated with numpy (fault=None) or with one of FAULTS injected. Returns (n, 2) float32."""
    kp = np.asarray(kp, F32).reshape(-1, 3)
    prev = np.asarray(prev, F32).reshape(-1, 2)
    n = len(kp)
    if fault == "unstable_sort":
        order = np.lexsort((-np.arange(n), -kp[:, 2]))          # equal responses in reverse cell order
    else:
        order = np.argsort(-kp[:, 2], kind="stable")
    pts = kp[order, :2]
    if fault != "no_quirk":
        pts = np.concatenate([np.zeros((n, 2), F32), pts])
    if mask_radius <= 0:
        return pts[:max_tracks] if fault == "cap_without_radius" else pts
    r2 = F32(mask_radius * mask_radius)
    out = np.zeros((len(pts), 2), F32)
    kept = 0
    for c in pts:
        if not _near(prev, c, r2, fault) and not _near(out[:kept], c, r2, fault):
            out[kept] = c
            kept += 1
        if kept >= max_tracks:
            break
    return out[:kept].copy()
