"""Plain extended-precision reference of the dense visual Kalman update (src/odometry/ekf.cpp:760-844, conventions as restated in
oracle/hv_oracle_ekf.c), and the tools the tests around it need: an input generator with a known condition number of S, the
comparator's tolerance, and a restatement of the launchers' predicates that says which kernel path a shape takes.

The reference is computed in np.longdouble (80-bit on x86-64, u = 2^-64) straight from the equations
    HP = H P[0:l, :],  S = HP[:, 0:l] H' + r^2 noiseScale I,  chi2 = noiseScale v' S^-1 v,
    m += HP' S^-1 v (then every quaternion normalised),  P -= HP' S^-1 HP
with a Cholesky factor of S. It does not use the kernels' algebra (no elimination tableau, no Z = L^-1 HP slices), so an error
in how the kernels organise that algebra cannot cancel out in the comparison."""
import numpy as np
from scipy.stats import chi2 as _chi2

LD = np.longdouble
U = 2.0 ** -53                  # unit roundoff of the fp64 implementations under test
C_TAU = 8.0                     # tolerance constant of tau() (see there)
CAM, POSE, ORI = 20, 7, 6


def chi2inv95(n):
    return float(_chi2.ppf(0.95, n))


def _chol(S):
    """Lower Cholesky factor of the symmetric positive definite S (longdouble); None if S is not positive definite."""
    n = S.shape[0]
    L = np.zeros_like(S)
    for j in range(n):
        d = S[j, j] - L[j, :j] @ L[j, :j]
        if not d > 0:
            return None
        L[j, j] = np.sqrt(d)
        L[j + 1:, j] = (S[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
    return L


def _chol_solve(L, B):
    """S^-1 B with S = L L' (B: n x k)."""
    n = L.shape[0]
    X = np.array(B, dtype=LD, copy=True)
    for i in range(n):
        X[i] = (X[i] - L[i, :i] @ X[:i]) / L[i, i]
    for i in range(n - 1, -1, -1):
        X[i] = (X[i] - L[i + 1:, i] @ X[i + 1:]) / L[i, i]
    return X


def normalize_quaternions(m, trail):
    """updateCommon after a visual update: the current and every trail quaternion (ekf.cpp:1024-1032)."""
    for o in [ORI] + [CAM + POSE * i + 3 for i in range(trail)]:
        q = m[o:o + 4]
        z = q @ q
        if z > 0:
            m[o:o + 4] = q / np.sqrt(z)


class Innovation:
    """HP, S, its Cholesky factor and the residual of one measurement against one state (all longdouble)."""

    def __init__(self, P, H, f, y, r, noise_scale, rdiag_scale=1.0, v_delta=None, transform_S=None):
        H = np.asarray(H, dtype=LD)
        n, l = H.shape
        self.ns = LD(noise_scale) ** 2                          # noiseScale = noise_scale^2 (ekf.cpp:190)
        self.v = np.asarray(y, dtype=LD) - np.asarray(f, dtype=LD)
        if v_delta is not None:
            self.v = self.v + np.asarray(v_delta, dtype=LD)
        self.HP = H @ np.asarray(P, dtype=LD)[:l, :]
        S = self.HP[:, :l] @ H.T
        S = 0.5 * (S + S.T)
        S[np.diag_indices(n)] += LD(r) * LD(r) * self.ns * LD(rdiag_scale)
        if transform_S is not None:
            S = transform_S(S)
        self.S = S
        self.L = _chol(S)


def check(P, H, f, y, r, noise_scale, rmse_thr=-1.0, **faults):
    """visualTrackOutlierCheck (ekf.cpp:760-819): (status, chi2) with status 0 INLIER, 2 RMSE, 3 CHI2."""
    n = np.asarray(H).shape[0]
    v = np.asarray(y, dtype=LD) - np.asarray(f, dtype=LD)
    if rmse_thr >= 0.0 and np.sqrt((v @ v) / n) > rmse_thr:
        return 2, 0.0
    if r < 0.0:
        return 0, 0.0
    inn = Innovation(P, H, f, y, r, noise_scale, **faults)
    if inn.L is None:
        return None, None
    x = _chol_solve(inn.L, inn.v[:, None])[:, 0]
    c2 = inn.ns * (x @ inn.v)
    return (3 if c2 > chi2inv95(n) else 0), c2


def update(m, P, H, f, y, r, noise_scale, trail, **faults):
    """updateVisualTrack (ekf.cpp:829-844): the new (m, P) in longdouble; None if S is not positive definite (the kernels report
    that as an error)."""
    inn = Innovation(P, H, f, y, r, noise_scale, **faults)
    if inn.L is None:
        return None
    W = _chol_solve(inn.L, inn.HP)                              # S^-1 HP = K'
    m1 = np.asarray(m, dtype=LD) + W.T @ inn.v
    P1 = np.asarray(P, dtype=LD) - inn.HP.T @ W
    normalize_quaternions(m1, trail)
    return m1, P1


def tau(n, kappa, c=C_TAU):
    """Tolerance of an fp64 implementation against the reference: c n u kappa_2(S)."""
    return c * n * U * kappa


def errors(ref_m, ref_P, m, P):
    """(|dm|_inf, max|dP| / max|P|) of (m, P) against the reference."""
    ref_m, ref_P = np.asarray(ref_m, dtype=LD), np.asarray(ref_P, dtype=LD)
    em = float(np.abs(np.asarray(m, dtype=LD) - ref_m).max())
    eP = float(np.abs(np.asarray(P, dtype=LD) - ref_P).max() / np.abs(ref_P).max())
    return em, eP


def chi2_error(ref_c2, c2):
    return float(abs(LD(c2) - LD(ref_c2)) / max(LD(1.0), abs(LD(ref_c2))))


# ---------------------------------------------------------------------------------------------------------- inputs
def state_dim(trail, map_size):
    return CAM + POSE * trail + 3 * map_size


def make_state(trail, map_size, n, l, kappa, seed):
    """A mean with unit quaternions and an SPD covariance P over the real state layout (inertial block, trail poses, map points),
    built so that S = H P[0:l, 0:l] H' + R of the measurement from make_measurement(seed) has condition number ~kappa: P = s I + a G G'
    with G of rank ceil(n / 2) < n, so that a (found by bisection) moves the large eigenvalues of S and leaves the small ones."""
    N = state_dim(trail, map_size)
    rng = np.random.RandomState(1000 + seed)
    m = rng.normal(0, 1.0, N)
    for o in [ORI] + [CAM + POSE * i + 3 for i in range(trail)]:
        m[o:o + 4] /= np.linalg.norm(m[o:o + 4])
    G = rng.normal(0, 1.0, (N, max(1, (n + 1) // 2)))
    H = make_measurement(n, l, seed)[0]
    R = 0.05 ** 2 * 1e4
    base = 1.0 * np.eye(N)

    def cond(a):
        P = base + a * (G @ G.T)
        return np.linalg.cond(H @ P[:l, :l] @ H.T + R * np.eye(n)), P

    lo, hi = 0.0, 1e6
    if n > 1:
        for _ in range(60):
            mid = np.sqrt(max(lo, 1e-3) * hi)
            if cond(mid)[0] < kappa:
                lo = mid
            else:
                hi = mid
    a = hi if n > 1 else 1.0
    P = base + a * (G @ G.T)
    P = 0.5 * (P + P.T)
    return m, P


def make_measurement(n, l, seed):
    """H ~ N(0, 0.1^2) (n x l) and a predicted measurement f; the residual is chosen by the caller."""
    rng = np.random.RandomState(2000 + seed)
    return np.asfortranarray(rng.normal(0, 0.1, (n, l))), rng.normal(0, 0.5, n)


def residual(P, H, r, noise_scale, scale, seed):
    """v ~ scale * N(0, S / noiseScale): chi2 ~ scale^2 chi2_n (0.5: inlier, 40: gross outlier)."""
    n, l = H.shape
    S = H @ P[:l, :l] @ H.T + (r * r) * noise_scale ** 2 * np.eye(n)
    z = np.random.RandomState(3000 + seed).normal(0, 1.0, n)
    return scale * np.linalg.cholesky(S) @ z / noise_scale


def kappa_S(P, H, r, noise_scale):
    n, l = H.shape
    inn = Innovation(P, H, np.zeros(n), np.zeros(n), r, noise_scale)
    return float(np.linalg.cond(np.asarray(inn.S, dtype=np.float64)))


# ---------------------------------------------------------------------------------------------------------- kernel paths
# Restatement of the launchers' predicates (hybvio_b200/csrc/ekf_cluster2.cu ekf_cluster2_fits, ekf_cluster2.cuh ek2_geom / ek2_body,
# ekf.cu ekf_update_smem_bytes / ekf_launch_update); joseph=True for the pose augmentation (the identity block in the tableau row and
# the EXTRA buffers of the Joseph product).
EK2_C, EK2_MAXN = 8, 768
EK2_STATIC_SMEM = 8 * (2 + 128 + 2 + EK2_MAXN) + 256
EK2_SMEM_LIMIT = 227 * 1024
SINGLE_SMEM_LIMIT = 200 * 1024


def _pad4mod16(w):
    return w + ((20 - (w & 15)) & 15)


def ek2_smem_bytes(n, l, N, joseph=False):
    C = EK2_C
    B = (N + C - 1) // C
    LDp = N + (((20 - (N & 15)) & 15) or 16)
    X = n * max(l, LDp)
    W = _pad4mod16(n + B + 1 + (n if joseph else 0))
    T = (n * W + 1) & ~1
    PB = LDp * B
    MTn = (n + 7) >> 3
    E = (64 * (MTn * (MTn + 1) // 2) + C - 1) // C
    RS = n * n if n * n <= 1024 else E
    EXTRA = N * 7 + 2 * 21 * LDp + N * B if joseph else 0
    SYM = N * B if n <= 8 else 0
    return (X + T + PB + RS + EXTRA + SYM) * 8, X


def cluster_fits(n, l, N, joseph=False):
    return N <= EK2_MAXN and ek2_smem_bytes(n, l, N, joseph)[0] + EK2_STATIC_SMEM <= EK2_SMEM_LIMIT


def kernel_path(n, l, N, h_aligned=True):
    """The path a dense visual update / check of shape (n, l) on an N-dimensional state takes:
    kernel in {cluster, single-smem, single-global}; for the cluster kernel also the S reduction (one-stage / two-stage through L2
    entry by entry / two-stage through L2 with bulk copies), where the gathered Z travels (dsmem / l2) and how H and P are staged
    (bulk / bulk-P loop-H / loop)."""
    if not cluster_fits(n, l, N):
        need = n * ((n + N + 1) | 1) * 8
        return ("single-global",) if need > SINGLE_SMEM_LIMIT else ("single-smem",)
    bulk = N % 2 == 0
    bulkH = bulk and (n * l) % 2 == 0 and h_aligned
    if n * n <= 1024:
        s = "one-stage"
    else:
        MT = (n + 7) >> 3
        ETOT = 64 * (MT * (MT + 1) // 2)
        X = ek2_smem_bytes(n, l, N)[1]
        if bulk and ETOT >= 2048 and ETOT % (2 * EK2_C) == 0 and 2 * ETOT <= X:
            s = "two-stage-l2-bulk"
        else:
            s = "two-stage-l2"
    z = "l2" if n * N >= 4096 else "dsmem"
    staging = "bulk" if bulkH else ("bulk-P-loop-H" if bulk else "loop")
    return ("cluster", s, z, staging)


KERNEL_NAME = {"cluster": "ekf_update_cluster2_kernel", "single-smem": "ekf_update_kernel", "single-global": "ekf_update_kernel"}


def visual_l(n, N):
    """Columns of H a visual measurement of n rows reaches (tests/ekf_script.visual_measurement)."""
    return min(N, 20 + 7 * max(1, n // 4))


def first(pred, lo, hi):
    """Smallest k in [lo, hi] with pred(k); None if none."""
    for k in range(lo, hi + 1):
        if pred(k):
            return k
    return None


# State layouts of the sweep, (camera trail length, map points): N = 61 (odd, trail 5 + 2 map points), 62, 160, 300, 163 (odd and
# large enough for the Z exchange through L2 without bulk copies)
CONFIGS = ((5, 2), (6, 0), (20, 0), (40, 0), (20, 1))
CHI2_MAX_N = 200                # the chi2 table of hv_ekf (ekf_capi.cu) ends at n = 200; updates go up to n = N


def reachable(trail, map_size):
    """{path: smallest (n, l)} over every dense visual shape a caller can issue on this state (l = visual_l(n) or l = N)."""
    N = state_dim(trail, map_size)
    out = {}
    for n in range(1, N + 1):
        for l in (visual_l(n, N), N):
            out.setdefault(kernel_path(n, l, N), (n, l))
    return out


def sweep_shapes():
    """(trail, map_size, n, l) of the GPU sweep, derived from the predicates: both sides of every boundary (n = 32 / 33 one- / two-stage
    S, n N = 4095 / 4096 Z through DSMEM / L2, the first n of the bulk S exchange, cluster / single-CTA, shared / global tableau), n = 1, 2, 3,
    n = N, the largest n a check can have, l = N at a small n, and for every other reachable path the smallest shape that takes it."""
    shapes = []
    for trail, ms in CONFIGS:
        N = state_dim(trail, ms)
        path = lambda n: kernel_path(n, visual_l(n, N), N)
        ns = {1, 2, 3, N, min(N, CHI2_MAX_N)}
        edges = [first(lambda n: n * n > 1024, 1, N),
                 first(lambda n: n * N >= 4096, 1, N),
                 first(lambda n: path(n)[0] == "cluster" and path(n)[1] == "two-stage-l2-bulk", 1, N),
                 first(lambda n: path(n)[0] != "cluster", 1, N),
                 first(lambda n: path(n)[0] == "single-global", 1, N)]
        for k in edges:
            if k is not None:
                ns |= {k - 1, k} if k > 1 else {k}
        sh = {(n, visual_l(n, N)) for n in ns if 1 <= n <= N} | {(8, N)}
        have = {kernel_path(n, l, N) for n, l in sh}
        sh |= {nl for p, nl in reachable(trail, ms).items() if p not in have}
        shapes += [(trail, ms, n, l) for n, l in sorted(sh)]
    return shapes
