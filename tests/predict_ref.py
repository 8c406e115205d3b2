"""Plain extended-precision reference of the IMU predict (src/odometry/ekf.cpp:320-514, conventions as restated in
oracle/hv_oracle_ekf.c:228-303), with a componentwise error bound carried along with the state, and the tools the tests around
it need: a restatement of the predict kernel's strip geometry and rotation branch, starting states and IMU input patterns.

The reference works sample by sample in np.longdouble (80-bit on x86-64, u = 2^-64): the host bookkeeping of one predict() call
(first sample, dt <= 0 dropped), the drift blocks of Q for this sample's dt, the rotation exp(-dt/2 Omega(w)) in closed form, the
mean, the Jacobians, P00 <- D P00 D' + G Q G', the two strips P[20:, :20] <- P[20:, :20] D' and P[:20, 20:] <- D P[:20, 20:], bias
decay and normalizeQuaternions(true) where the caller asks for it. The rest of P is never touched.

Error bound. For an fp64 implementation of the same operation, every computed entry gets, per sample,
    B <- |T| B |T|' + k (|T| |P| |T|' + |G| |Q| |G|'),   T = blockdiag(D, I),   k = C_P u + 2 delta,
where |.| of D and G is the absolute-value evaluation of their formulas (every sum replaced by the sum of the absolute values of its
terms), u = 2^-53 and delta is the relative error of the Jacobian entries caused by the error of the mean they are evaluated at
(see Reference.delta). The fresh term k (...) applies only to the entries the sample computes: P00 gets both products, a strip gets
k S_e+1 with S_e+1 = |P[20:, :20]_0| |D_0|' ... |D_e|' (and D's on the left for P[:20, 20:]), and the block P[20:, 20:] gets nothing,
so its bound stays 0 and it must come back bit for bit.

C_P is the tally of standard inner-product bounds (gamma_n ~ n u, Higham, Accuracy and Stability of Numerical Algorithms, 3.1):
  * the Jacobian entries themselves (C_D = 35): the worst is d vel / d gyro noise = (B A)(A dS q) -- the 3-term sums of B = dR' Tx dt
    (3u, times dt 1u, Tx = bat xa - baa 2u: 6u), the 4-term B A (4u) with 8u in A (sin / cos or the Taylor series, products with
    w and c), the 4-term A (dS q) (4u + 8u + 1u), and the 4-term product of the two (4u): 6 + 8 + 4 + 13 + 4 = 35;
  * D P00 D': the two 20-term products (20u + 21u, the second one adds W) and D's own error twice (70u): 111u;
  * G Q G': the two 12-term products (24u), the sum with D P00 D' (21u) and G's error twice (70u): 115u. The drift blocks of Q
    come from the host's fp64 (1 - exp(-2 dt rev)) / (2 rev), which cancels; their own bound EQ (Reference._sample) enters as
    |G| EQ |G|';
  * a strip: the kernel forms Dacc = D_e ... D_s of a launch first (one 20-term product per sample, gamma_20 |D_j| |Dacc|, plus D's
    error) and applies it once (one more 20-term product), so its error is at most (e - s + 2) (20 + 35)u |strip_s| |Dacc|' <=
    (e - s + 2) 55u S_e+1 whatever s is. The bound charges k S_e+1 at each of the e + 1 samples, at least 128 (e + 1)u S_e+1; this
    also covers the sample-by-sample evaluation, because S_e+1 >= |strip_e+1|. Where D is far from I (the 0.5 s gap: D[VEL, ORI] ~ 10)
    S grows with it, as the kernel's error can.
The largest, 115u, rounded up to a power of two gives C_P = 128. The mean bound is propagated in the same way, operation by
operation (Reference._mean). Where the bound of an entry is 0 (structural zeros, untouched blocks, constant biases), the comparator
requires the entry to be exact."""
import numpy as np

LD = np.longdouble
U = 2.0 ** -53                 # unit roundoff of the fp64 implementations under test
C_P = 128.0                    # per-sample covariance constant (tally above)
C_D = 35.0                     # Jacobian entries, relative to their absolute-value evaluation
C_A = 8.0                      # entries of the rotation exp(-dt/2 Omega(w))
INER, POS, VEL, ORI, BGA, BAA, BAT, SFT = 20, 0, 3, 6, 10, 13, 16, 19
Q_ACC, Q_GYRO, Q_BGA, Q_BAA = 0, 3, 6, 9
CAM, POSE, MAPPT = 20, 7, 3
EKF_NT = 512                   # threads of the predict CTA (hybvio_b200/csrc/ekf.cuh)
WARPS = EKF_NT // 32
TILE_STRIDE = 3 * WARPS        # tiles one pass of the strip loop covers (ekf_predict.cuh: tb += 3 * (EKF_NT / 32))
MAX_PREDICT = 16               # samples per launch (EKF_MAX_PREDICT)
BRANCH_X = 0.01                # x = (|w| dt / 2)^2 below which the kernel uses the Taylor series


# ------------------------------------------------------------------------------------------------ kernel geometry
def state_dim(trail, map_size):
    return INER + POSE * trail + MAPPT * map_size


def strip_geometry(N):
    """(rest, ntile) of the strip product: X = [P[20:, :20]; P[:20, 20:]'] has 2 rest rows, dealt to the warps in 8-row tiles.
    A tile straddles the two strips when rest % 8 != 0. Warp w takes tiles w, w + 16, w + 32 in one pass of its loop and
    TILE_STRIDE = 48 tiles later the next pass: ntile > 16, 32, 48, 96 ... adds a tile to some warp."""
    rest = N - INER
    return rest, (2 * rest + 7) // 8


def strip_passes(ntile):
    """Passes of the tile loop warp 0 makes."""
    return (ntile + TILE_STRIDE - 1) // TILE_STRIDE


def rotation_x(w, dt):
    """The kernel's x = (w0^2 + w1^2 + w2^2) (dt/2)^2 in fp64, in its order (ekf_predict.cuh). With at most one nonzero component of
    w, a contraction into FMAs cannot change it."""
    w0, w1, w2 = (np.float64(v) for v in w)
    c = -np.float64(dt) / np.float64(2)
    return np.float64((w0 * w0 + w1 * w1 + w2 * w2) * (c * c))


def closed_form_branch(x):
    """True where the kernel evaluates cos / sin(th) / th in closed form, False where it uses their Taylor series."""
    return not (x < BRANCH_X)


# ------------------------------------------------------------------------------------------------ rotation matrices
# R(q) (src/odometry/util.cpp:10-47) as sum_k coef q_a q_b per entry (row-major), so that R, dR / dq and their absolute-value
# evaluations come from one table
_R_TERMS = [[(1, 0, 0), (1, 1, 1), (-1, 2, 2), (-1, 3, 3)], [(2, 1, 2), (-2, 0, 3)], [(2, 1, 3), (2, 0, 2)],
            [(2, 1, 2), (2, 0, 3)], [(1, 0, 0), (-1, 1, 1), (1, 2, 2), (-1, 3, 3)], [(2, 2, 3), (-2, 0, 1)],
            [(2, 1, 3), (-2, 0, 2)], [(2, 2, 3), (2, 0, 1)], [(1, 0, 0), (-1, 1, 1), (-1, 2, 2), (1, 3, 3)]]


def rmat(q, absolute=False):
    """3 x 3 R(q) and dR[a] = dR / dq_a (4 x 3 x 3); absolute=True: their absolute-value evaluations at |q|."""
    q = np.abs(q) if absolute else q
    R = np.zeros((3, 3), dtype=LD)
    dR = np.zeros((4, 3, 3), dtype=LD)
    for e, terms in enumerate(_R_TERMS):
        i, j = divmod(e, 3)
        for coef, a, b in terms:
            cf = LD(abs(coef) if absolute else coef)
            R[i, j] += cf * q[a] * q[b]
            dR[a, i, j] += cf * q[b]
            dR[b, i, j] += cf * q[a]
    return R, dR


def omega(w):
    """Omega(w) (4 x 4), row-major as in the oracle."""
    return np.array([[0, -w[0], -w[1], -w[2]], [w[0], 0, -w[2], w[1]], [w[1], w[2], 0, -w[0]], [w[2], -w[1], w[0], 0]], dtype=LD)


def dS(h):
    """d(-dt/2 Omega(w)) / dw_j for j = 0, 1, 2 with h = dt / 2 (oracle dS)."""
    out = np.zeros((3, 4, 4), dtype=LD)
    out[0][[0, 1, 2, 3], [1, 0, 3, 2]] = [h, -h, h, -h]
    out[1][[0, 1, 2, 3], [2, 3, 0, 1]] = [h, -h, -h, h]
    out[2][[0, 1, 2, 3], [3, 2, 1, 0]] = [h, h, -h, -h]
    return out


def jacobians(A, q, qn, Tx, xa, dt, absolute=False):
    """dydx D (20 x 20) and dydq G (20 x 12) of one sample (ekf.cpp:450-498). absolute=True gives their absolute-value evaluation:
    every input replaced by its absolute value and every sum by the sum of the absolute values of its terms."""
    ab = np.abs if absolute else (lambda x: x)
    sg = (lambda x: x) if absolute else (lambda x: -x)
    A, q, qn, Tx, xa = ab(A), ab(q), ab(qn), ab(Tx), ab(xa)
    dt = LD(dt)
    R, dR = rmat(qn, absolute)
    D = np.eye(20, dtype=LD)
    G = np.zeros((20, 12), dtype=LD)
    D[POS:POS + 3, VEL:VEL + 3] = dt * np.eye(3, dtype=LD)
    Bq = np.stack([dR[a].T @ Tx for a in range(4)], axis=1) * dt          # 3 x 4: B[i, a] = (dR[a]' Tx)_i dt
    D[VEL:VEL + 3, ORI:ORI + 4] = Bq @ A
    D[ORI:ORI + 4, ORI:ORI + 4] = A
    G[VEL:VEL + 3, Q_ACC:Q_ACC + 3] = R.T * dt
    dSs = dS(dt / 2)
    for j in range(3):
        G[ORI:ORI + 4, Q_GYRO + j] = A @ (ab(dSs[j]) @ q)
    G[BGA:BGA + 3, Q_BGA:Q_BGA + 3] = np.eye(3, dtype=LD)
    G[BAA:BAA + 3, Q_BAA:Q_BAA + 3] = np.eye(3, dtype=LD)
    G[VEL:VEL + 3, Q_GYRO:Q_GYRO + 3] = D[VEL:VEL + 3, ORI:ORI + 4] @ G[ORI:ORI + 4, Q_GYRO:Q_GYRO + 3]
    D[VEL:VEL + 3, BGA:BGA + 3] = sg(G[VEL:VEL + 3, Q_GYRO:Q_GYRO + 3])
    D[ORI:ORI + 4, BGA:BGA + 3] = sg(G[ORI:ORI + 4, Q_GYRO:Q_GYRO + 3])
    D[VEL:VEL + 3, BAA:BAA + 3] = sg(R.T * dt)
    D[VEL:VEL + 3, BAT:BAT + 3] = R.T * xa[None, :] * dt
    return D, G


# ------------------------------------------------------------------------------------------------ the reference
FAULTS = ("p_vel_bat", "stale_drift_q", "strips_miss_last_d", "late_normalisation", "d_cols_16_19_dropped", "previous_sinc")


class Reference:
    """One filter: m, P, Q in longdouble with the bounds Bm, BP (and Bd of dydx). `params` has the fields of hv_ekf_params.
    faults: {name: sample index} (see FAULTS); a fault makes the reference compute something subtly wrong at that sample (counted
    over the samples that are not dropped), for the tests that show the comparator rejects it."""

    def __init__(self, params, m, P, faults=None):
        self.ns = LD(params.noise_scale) ** 2
        self.gravity = LD(params.gravity)
        self.walk = {"baa": (params.noise_process_baa, params.noise_process_baa_rev), "bga": (params.noise_process_bga, params.noise_process_bga_rev)}
        self.m = np.array(m, dtype=LD)
        self.P = np.array(P, dtype=LD)
        self.N = len(self.m)
        self.Q = np.zeros((12, 12), dtype=LD)
        for i in range(3):
            self.Q[Q_ACC + i, Q_ACC + i] = self.ns * LD(params.noise_process_acc) ** 2
            self.Q[Q_GYRO + i, Q_GYRO + i] = self.ns * LD(params.noise_process_gyro) ** 2
        self.EQ = np.zeros((12, 12), dtype=LD)     # error bound of the drift blocks the host computes in fp64
        self.Bm = np.zeros(self.N, dtype=LD)
        self.eq = LD(0)                             # bound on the 2-norm of the quaternion's error (Bm[ORI:ORI + 4] = eq each)
        self.BP = np.zeros((self.N, self.N), dtype=LD)
        # |P[20:, :20]| and |P[:20, 20:]| of the start carried through |D|: they bound |strip_s| |D_s|' ... |D_e|' for every s <= e
        self.S10, self.S01 = np.abs(self.P[20:, :20]), np.abs(self.P[:20, 20:])
        self.dydx = np.zeros((20, 20), dtype=LD)
        self.Bd = np.zeros((20, 20), dtype=LD)
        self.first, self.prev_t = True, -1.0
        self.k = 0                                  # samples processed (not dropped)
        self.faults = dict(faults or {})
        self._prev_sc = None
        self._late_norm = False

    # host bookkeeping (ekf.cpp:357-370, ekf_capi.cu predict_bookkeep): the first sample and dt <= 0 are dropped, prevSampleT moves
    def predict(self, t, xg, xa):
        dt = 0.0
        if not self.first:
            dt = t - self.prev_t                    # in fp64, as the host computes it: dt is an input of the fp64 implementations
        else:
            self.first = False
        self.prev_t = t
        if not dt > 0.0:
            return
        self._sample(dt, np.asarray(xg, dtype=LD), np.asarray(xa, dtype=LD))
        self.k += 1
        if self._late_norm:                         # fault: the normalisation asked for after the previous sample happens only now
            self._late_norm = False
            self._normalize()

    def normalize_quaternions(self):
        """normalizeQuaternions(true): the current orientation only."""
        if self.faults.get("late_normalisation") == self.k - 1:
            self._late_norm = True
            return
        self._normalize()

    def _fault(self, name):
        return self.faults.get(name) == self.k

    def _normalize(self):
        q = self.m[ORI:ORI + 4]
        n = np.sqrt(q @ q)
        if n > 0:
            # d(q / |q|) = (I - qh qh') dq / |q| and I - qh qh' has 2-norm 1, so the 2-norm bound only scales by 1 / |q| (plus the
            # second-order term); rounding of the sum of 4 squares, the sqrt and the division: 6u of |qh| = 1
            e = self.eq / n
            self._set_eq(e + e * e + 6 * U)
            self.m[ORI:ORI + 4] = q / n

    def _set_eq(self, eq):
        self.eq = eq
        self.Bm[ORI:ORI + 4] = eq

    def delta(self):
        """Relative error of the Jacobian entries caused by the error of the mean: they are at most quadratic in q (3 eps_q), A moves with
        the gyro bias by |dA / dw| <= 3 |dt / 2| per unit of w (eps_w, taken at dt = 1 s), Tx = bat xa - baa with the accelerometer bias
        (bat is constant in predict, so its bound stays 0)."""
        q = self.m[ORI:ORI + 4]
        eps_q = 2 * self.eq / np.sqrt(q @ q)        # sum_i |dq_i| <= 2 |dq|_2 for 4 components
        eps_w = 1.5 * self.Bm[BGA:BGA + 3].sum()
        eps_t = self.Bm[BAA:BAA + 3].sum() / (np.abs(self.m[BAT:BAT + 3]) + np.abs(self.m[BAA:BAA + 3])).min()
        return 3 * eps_q + eps_w + eps_t

    def _sample(self, dt, xg, xa):
        m, N, dtL = self.m, self.N, LD(dt)
        # drift blocks of Q in force at this sample (ekf.cpp:397-412)
        if not self._fault("stale_drift_q"):
            for key, off in (("baa", Q_BAA), ("bga", Q_BGA)):
                s, th = self.walk[key]
                if s > 0.0:
                    v = self.ns * LD(s) ** 2
                    eps = 4 * U
                    if th > 0.0:
                        x = 2 * dtL * LD(th)
                        v *= (1 - np.exp(-x)) / (2 * LD(th))
                        # the fp64 1 - exp(-x) cancels: exp's 1 ulp and the rounding of x cost 2 u e (1 + x) / (1 - e)
                        e = np.exp(-x)
                        eps = LD(6 * U) + 2 * U * e * (1 + x) / (1 - e)
                    self.Q[off:off + 3, off:off + 3] = v * np.eye(3, dtype=LD)
                    self.EQ[off:off + 3, off:off + 3] = eps * abs(v) * np.eye(3, dtype=LD)
        # rotation exp(-dt/2 Omega(w)) = cos(th) I + sin(th)/th S, S = -dt/2 Omega(w), th = |w| dt / 2
        w = xg - m[BGA:BGA + 3]
        c = -dtL / 2
        th = np.sqrt(w @ w) * abs(c)
        sc = np.sin(th) / th if th > 0 else LD(1)
        if self._fault("previous_sinc") and self._prev_sc is not None:
            sc = self._prev_sc
        self._prev_sc = np.sin(th) / th if th > 0 else LD(1)
        A = np.cos(th) * np.eye(4, dtype=LD) + sc * c * omega(w)
        q = m[ORI:ORI + 4].copy()
        qn = A @ q
        Tx = m[BAT:BAT + 3] * xa - m[BAA:BAA + 3]
        delta = self.delta()
        D, G = jacobians(A, q, qn, Tx, xa, dt)
        Da, Ga = jacobians(A, q, qn, Tx, xa, dt, absolute=True)
        self._mean(dt, xg, xa, A, q, qn, Tx)
        # covariance (ekf.cpp:504-508) and its bound
        k = LD(C_P * U) + 2 * delta
        P, BP = self.P, self.BP
        P00, P10, P01 = P[:20, :20], P[20:, :20], P[:20, 20:]
        aP00 = np.abs(P00)
        Dp = D.copy()
        if self._fault("d_cols_16_19_dropped"):
            Dp[:, 16:20] = 0
        W = G @ self.Q @ G.T
        new00 = Dp @ P00 @ D.T + W
        if self._fault("p_vel_bat"):
            new00[VEL:VEL + 3, BAT:BAT + 3] *= 1 + LD(1e-6)
            new00[BAT:BAT + 3, VEL:VEL + 3] *= 1 + LD(1e-6)
        B00 = Da @ BP[:20, :20] @ Da.T + k * (Da @ aP00 @ Da.T + Ga @ np.abs(self.Q) @ Ga.T) + Ga @ self.EQ @ Ga.T
        if N > INER and not self._fault("strips_miss_last_d"):
            self.S10, self.S01 = self.S10 @ Da.T, Da @ self.S01
            BP[20:, :20] = BP[20:, :20] @ Da.T + k * self.S10
            BP[:20, 20:] = Da @ BP[:20, 20:] + k * self.S01
            P[20:, :20] = P10 @ D.T
            P[:20, 20:] = D @ P01
        P[:20, :20] = new00
        BP[:20, :20] = B00
        self.dydx = D
        self.Bd = (LD(C_D * U) + delta) * Da

    def _mean(self, dt, xg, xa, A, q, qn, Tx):
        """Mean update (ekf.cpp:427-448) and its bound."""
        m, Bm, dtL = self.m, self.Bm, LD(dt)
        Ba = np.abs(A)
        Bw = Bm[BGA:BGA + 3] + U * np.abs(xg - m[BGA:BGA + 3])
        dA = C_A * U * Ba + 3 * abs(dtL / 2) * Bw.sum()
        # the exact A is orthogonal, so it carries the 2-norm of the error over unchanged; A's own error and the 4-term rounding add to it
        eqn = self.eq + np.linalg.norm(dA @ np.abs(q)) + 4 * U * np.linalg.norm(Ba @ np.abs(q))
        Bqn = np.full(4, eqn, dtype=LD)
        R, _ = rmat(qn)
        Ra, dRa = rmat(qn, absolute=True)
        Rerr = np.tensordot(Bqn, dRa, axes=1) + 2 * Bqn.sum() ** 2 + 5 * U * Ra          # |dR(q)| <= |dR|(|q|) |dq| + O(dq^2)
        BTx = Bm[BAT:BAT + 3] * np.abs(xa) + Bm[BAA:BAA + 3] + 2 * U * (np.abs(m[BAT:BAT + 3] * xa) + np.abs(m[BAA:BAA + 3]))
        g = np.array([0, 0, -self.gravity], dtype=LD)
        dv = (R.T @ Tx + g) * dtL
        Bdv = dtL * (Rerr.T @ np.abs(Tx) + Ra.T @ BTx + 4 * U * (Ra.T @ np.abs(Tx) + np.abs(g))) + U * np.abs(dv)
        p, v = m[POS:POS + 3].copy(), m[VEL:VEL + 3].copy()
        m[POS:POS + 3] = p + v * dtL
        Bm[POS:POS + 3] = Bm[POS:POS + 3] + dtL * Bm[VEL:VEL + 3] + 2 * U * (np.abs(p) + np.abs(v) * dtL)
        m[VEL:VEL + 3] = v + dv
        Bm[VEL:VEL + 3] = Bm[VEL:VEL + 3] + Bdv + U * (np.abs(v) + np.abs(dv))
        m[ORI:ORI + 4] = qn
        self._set_eq(eqn)
        for key, off in (("baa", BAA), ("bga", BGA)):
            s, th = self.walk[key]
            if s > 0.0:
                d = np.exp(-dtL * LD(th))
                m[off:off + 3] *= d
                Bm[off:off + 3] = d * Bm[off:off + 3] + 3 * U * np.abs(m[off:off + 3])


# ------------------------------------------------------------------------------------------------ comparison
def bound_ratio(got, ref, bound):
    """max |got - ref| / bound over the entries with a nonzero bound; inf if an entry with a zero bound is not exact."""
    got, ref, bound = np.asarray(got, dtype=LD), np.asarray(ref, dtype=LD), np.asarray(bound, dtype=LD)
    d = np.abs(got - ref)
    zero = bound == 0
    if (d[zero] != 0).any():
        return float("inf")
    return float((d[~zero] / bound[~zero]).max()) if (~zero).any() else 0.0


def ratios(ref, m, P, dydx=None):
    """{'m', 'P', 'dydx'}: bound_ratio of each against the reference."""
    out = {"m": bound_ratio(m, ref.m, ref.Bm), "P": bound_ratio(P, ref.P, ref.BP)}
    if dydx is not None:
        out["dydx"] = bound_ratio(dydx, ref.dydx, ref.Bd)
    return out


def scaled_error(P, ref):
    """max |P_ij - ref_ij| / sqrt(ref_ii ref_jj): the error of each entry on the scale of its own variables (0 / 0 counts as 0)."""
    ref = np.asarray(ref, dtype=LD)
    d = np.abs(np.asarray(P, dtype=LD) - ref)
    s = np.sqrt(np.abs(np.diag(ref)))
    den = s[:, None] * s[None, :]
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(den > 0, d / np.where(den > 0, den, 1), np.where(d > 0, np.inf, 0))
    return float(r.max())


# ------------------------------------------------------------------------------------------------ states and inputs
ACC0 = np.array([0.3, 0.2, 9.819])


def dense_state(N, seed=0):
    """(b): a mean with biases, a quaternion of norm 1.05 (so that where a normalisation happens is visible in the result) and a dense
    SPD P = Delta C Delta with the diagonal log-spread over 1e-12 .. 1e8 and correlations up to 0.999."""
    rng = np.random.RandomState(100 + seed)
    m = rng.normal(0, 1.0, N)
    m[ORI:ORI + 4] = [0.9, 0.1, -0.3, 0.2]
    m[ORI:ORI + 4] *= 1.05 / np.linalg.norm(m[ORI:ORI + 4])
    m[BGA:BGA + 3] = rng.normal(0, 1e-3, 3)
    m[BAA:BAA + 3] = rng.normal(0, 1e-2, 3)
    m[BAT:BAT + 3] = 1 + rng.normal(0, 1e-3, 3)
    m[SFT] = 1e-3
    Gm = rng.normal(0, 1.0, (N, 3))
    Cm = Gm @ Gm.T + 1e-3 * np.eye(N)
    s = 1 / np.sqrt(np.diag(Cm))
    Cm = Cm * s[:, None] * s[None, :]
    e = np.concatenate([np.linspace(-12, 8, 20), np.linspace(-12, 8, N - 20)])
    e[:20] = rng.permutation(e[:20])
    e[20:] = rng.permutation(e[20:])
    d = np.sqrt(10.0 ** e)
    P = Cm * d[:, None] * d[None, :]
    P = 0.5 * (P + P.T)
    return m, P


class Pattern:
    """A list of predict() calls (t, gyro, acc, normalise-after) and a few settings: random walks, batching, whether the mean launch is
    checked."""

    def __init__(self, name, calls, walk=None, batch=MAX_PREDICT, mean_launch=False):
        self.name, self.calls, self.walk, self.batch, self.mean_launch = name, calls, dict(walk or {}), batch, mean_launch


def _gyro_acc(rng, big=False):
    g = np.array([0.0, 0.0, 0.2]) + rng.normal(0, 0.05, 3)
    if big:
        g = g + rng.normal(0, 1.0, 3) * 2 + np.array([60.0, -10.0, 25.0])      # |w| ~ 66 rad/s: x ~ 0.027 at 5 ms
    a = np.array([0.3, 0.2, 9.819]) + rng.normal(0, 0.2, 3)
    return g, a


def _norm_flag(mode, i):
    return {"never": False, "every": True, "some": i % 3 == 1}[mode]


def burst(k, norm, seed=0, t0=1.0, dt=0.005):
    """k + 1 calls 5 ms apart: the first is dropped by the host (first sample), the next k form one burst."""
    rng = np.random.RandomState(50 + seed + 17 * k)
    calls = []
    for i in range(k + 1):
        g, a = _gyro_acc(rng)
        calls.append((t0 + i * dt, g, a, _norm_flag(norm, i)))
    return calls


def _rate_for(want, dt, b):
    """A gyro z rate whose x (with bias b) is the largest below, exactly at, or the smallest above 0.01 for this fp64 dt; None if no
    fp64 rate near the crossing gives x = 0.01 exactly."""
    x = lambda z: rotation_x([0.0, 0.0, z - np.float64(b)], dt)
    zs = [np.float64(np.sqrt(BRANCH_X) / (dt / 2)) + np.float64(b)]
    for _ in range(64):
        zs.insert(0, np.nextafter(zs[0], -np.inf))
        zs.append(np.nextafter(zs[-1], np.inf))
    for lo, hi in zip(zs, zs[1:]):
        if want == "below" and x(lo) < BRANCH_X <= x(hi):
            return lo
        if want == "above" and x(lo) <= BRANCH_X < x(hi):
            return hi
        if want == "at" and x(lo) == BRANCH_X:
            return lo
    return None


def boundary_calls(bg, t0=1.0):
    """Samples whose x (the kernel's fp64 expression, with the gyro bias bg the filter holds) lies just below, exactly at and just above
    0.01, each followed by an ordinary sample; w has one nonzero component so that FMA contraction cannot move x."""
    rng = np.random.RandomState(9)
    out = [(t0, *_gyro_acc(rng), False)]
    t = t0
    for want in ("below", "at", "above"):
        for i in range(200):
            tn = t + 0.005 + i * 1e-9
            z = _rate_for(want, tn - t, bg[2])
            if z is not None:
                break
        else:
            raise AssertionError(f"no gyro rate with x {want} {BRANCH_X}")
        out.append((tn, np.array([bg[0], bg[1], z]), ACC0.copy(), False))
        t = tn + 0.005
        out.append((t, *_gyro_acc(rng), True))
    return out


def irregular_calls(seed=0, t0=1.0):
    """dt jitter (5 +- 2 ms), a 0.1 s gap at 3 rad/s (closed form: x = 0.0225), a 0.5 s gap at 0.2 rad/s (series: x = 0.0025), a
    duplicate and a backwards timestamp (dropped; the next dt starts at the dropped sample's time)."""
    rng = np.random.RandomState(70 + seed)
    t, out = t0, []
    for i in range(15):
        g, a = _gyro_acc(rng)
        if i == 4:
            t += 0.1
            g = np.array([0.0, 3.0, 0.0])
        elif i == 7:
            t += 0.5
        elif i == 9:
            pass                                    # duplicate of the previous timestamp
        elif i == 11:
            t -= 0.003                              # backwards
        else:
            t += 0.005 + rng.uniform(-0.002, 0.002)
        out.append((t, g, a, _norm_flag("some", i)))
    return out


def rotation_calls(mode, seed=0, t0=1.0, n=17):
    """n + 1 calls: every sample a large rotation (|w| ~ 66 rad/s, closed form) or large and small ones alternating."""
    rng = np.random.RandomState(80 + seed)
    out = []
    for i in range(n + 1):
        g, a = _gyro_acc(rng, big=(mode == "large" or i % 2 == 0))
        out.append((t0 + i * 0.005, g, a, _norm_flag("some", i)))
    return out


def jitter_calls(n=17, seed=0, t0=1.0, big_every=0, norm="some"):
    """n + 1 calls with dt between 3 and 7 ms (the drift blocks of Q change every sample); every big_every-th sample a large rotation;
    normalisations as in burst()."""
    rng = np.random.RandomState(90 + seed)
    t, out = t0, []
    for i in range(n + 1):
        g, a = _gyro_acc(rng, big=big_every > 0 and i % big_every == 0)
        out.append((t, g, a, _norm_flag(norm, i)))
        t += 0.005 + rng.uniform(-0.002, 0.002)
    return out


WALKS = {"baa-rev0.1": {"noise_process_baa": 1e-4, "noise_process_baa_rev": 0.1},
         "baa-rev0": {"noise_process_baa": 1e-4, "noise_process_baa_rev": 0.0},
         "bga-rev0": {"noise_process_bga": 2e-5, "noise_process_bga_rev": 0.0},
         "bga-rev0.1": {"noise_process_bga": 2e-5, "noise_process_bga_rev": 0.1}}


def input_patterns(bg):
    """The inputs of the sweep at the base shape. bg: gyro bias of the starting state (for the boundary samples)."""
    pats = [Pattern("large", rotation_calls("large"), mean_launch=True),
            Pattern("large-small", rotation_calls("mixed"), mean_launch=True),
            Pattern("boundary", boundary_calls(bg), mean_launch=True),
            Pattern("irregular", irregular_calls()),
            Pattern("irregular-batch1", irregular_calls(1), batch=1)]
    for name, w in WALKS.items():
        pats.append(Pattern("walk-" + name, jitter_calls(seed=len(pats)), walk=w))
    return pats


PATTERN_NAMES = ["large", "large-small", "boundary", "irregular", "irregular-batch1"] + ["walk-" + w for w in WALKS]


def shape_pattern():
    """The input every shape of the sweep runs: 17 jittered samples with large rotations, both random walks on, some normalisations."""
    return Pattern("shape", jitter_calls(big_every=3), walk={**WALKS["baa-rev0.1"], **WALKS["bga-rev0.1"]}, mean_launch=True)


BASE_TRAIL = 6                 # N = 62
STARTS = ("default", "dense")  # (a) initialize_orientation on a new filter: 1e8 trail priors and structural zeros; (b) dense_state
BURST_NORMS = ("never", "every", "some")


def sweep_cases():
    """(id, start, trail, map_size, pattern name) of the sweep: at N = 62 bursts of 1..17 samples under each normalisation mode and every
    input pattern; at every shape of sweep_shapes the shape pattern. Each from both starting states."""
    out = []
    for start in STARTS:
        base = [f"burst{k}-{norm}" for norm in BURST_NORMS for k in range(1, 18)]
        base += PATTERN_NAMES
        out += [(f"{start}-N{state_dim(BASE_TRAIL, 0)}-{name}", start, BASE_TRAIL, 0, name) for name in base]
        out += [(f"{start}-N{state_dim(t, ms)}-shape", start, t, ms, "shape") for t, ms in sweep_shapes()]
    return out


def make_pattern(name, bg):
    """The Pattern called `name` in sweep_cases; bg: gyro bias of the starting state."""
    if name.startswith("burst"):
        k, norm = name[5:].split("-")
        return Pattern(name, burst(int(k), norm))
    if name == "shape":
        return shape_pattern()
    return {p.name: p for p in input_patterns(bg)}[name]


def start_state(start, backend):
    """Puts the starting state into a new filter of a back end (CUDA or oracle) and returns it as (m, P) in fp64."""
    if start == "default":
        backend.initialize_orientation(ACC0)
        return backend.download()
    m, P = dense_state(backend.N)
    backend.upload(m, P)
    return m, P


def sweep_shapes(max_trail=120, max_map=7):
    """(trail, map_size) of the GPU sweep, derived from strip_geometry: for each requirement the smallest state that meets it -- trail 1
    (N = 27), every rest % 8 (the tile that straddles the two strips at every offset), ntile on both sides of 16, 32 and 48 (one, two,
    three tiles per warp; a second pass of the loop), ntile > 96 (a third pass) and N >= 700."""
    cands = sorted(((state_dim(t, ms), ms, t) for t in range(1, max_trail + 1) for ms in range(max_map + 1)))
    need = [lambda t, ms, rest, nt: t == 1]
    need += [lambda t, ms, rest, nt, r=r: rest % 8 == r for r in range(8)]
    need += [lambda t, ms, rest, nt, v=v: nt == v for v in (16, 17, 32, 33, 48, 49)]
    need += [lambda t, ms, rest, nt: nt > 96, lambda t, ms, rest, nt: state_dim(t, ms) >= 700]
    out = []
    for pred in need:
        for N, ms, t in cands:
            if pred(t, ms, *strip_geometry(N)):
                if (t, ms) not in out:
                    out.append((t, ms))
                break
        else:
            raise AssertionError("no state layout meets a requirement of the sweep")
    return sorted(out, key=lambda s: state_dim(*s))


# ------------------------------------------------------------------------------------------------ running a case
def with_walk(params, walk):
    for k, v in walk.items():
        setattr(params, k, v)
    return params


def drive(backend, calls, ref=None):
    """Issues the calls to a back end (CUDA, oracle) and, if given, to the reference."""
    for t, g, a, norm in calls:
        backend.predict(t, g, a)
        if ref is not None:
            ref.predict(t, g, a)
        if norm:
            backend.normalize_quaternions(True)
            if ref is not None:
                ref.normalize_quaternions()


def reference_run(params, m, P, calls, faults=None):
    ref = Reference(params, m, P, faults)
    for t, g, a, norm in calls:
        ref.predict(t, g, a)
        if norm:
            ref.normalize_quaternions()
    return ref


def branches(calls, bg):
    """Rotation branch of every sample the host keeps (bias bg held constant, as in the sweep's boundary pattern)."""
    out, prev = [], None
    for t, g, a, _ in calls:
        if prev is not None and t - prev > 0:
            out.append(closed_form_branch(rotation_x(np.asarray(g) - bg, t - prev)))
        prev = t
    return out
