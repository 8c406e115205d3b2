"""Extended-precision reference of the dense visual Kalman update with a componentwise (per-entry) error bound, and the realistic
cases it is checked on: filter states that come out of a filter run and measurements from the per-track measurement model.

The reference is kalman_ref's: in np.longdouble from the equations, HP = H P[0:l, :], S = HP[:, 0:l] H' + r^2 noiseScale I,
m += HP' S^-1 v, P -= HP' S^-1 HP (v = y - f), then every quaternion normalised (updateCommon, ekf.cpp:1024-1032). The bound has the
form of ekf_ops_ref.Ops._update, with |K| = |P_l|' |H|' |S^-1| the absolute-value evaluation of the gain:
    B_P = C_VIS u kappa(S) (|P| + |K| |H| |P_l|),   B_m = C_VIS u kappa(S) (|m| + |K| (|v| + u (|y| + |f|))),
and the normalisation's bound (ekf_ops_ref._normalize) on top. An entry whose bound is 0 has no rounding in it (no nonzero term of
K H P or K v reaches it: blocks the measurement does not touch, structural zeros) and must be exact. chi2 stays with kalman_ref's
normwise tau: it is a scalar, so its relative error is already componentwise.

Tally of C_VIS(n, l_nz) (gamma_k ~ k u, Higham, Accuracy and Stability of Numerical Algorithms 3.1; l_nz: the nonzero columns of H --
a zero column adds exact zero products, however the kernel tiles it):
  * HP = H P[0:l, :]:                   l_nz terms                                  l_nz u
  * S = HP H' + R:                      l_nz terms and R                            (l_nz + 1) u
  * the cluster's split S sums:         8 partial slices (one per CTA) added        8 u
  * unpivoted elimination of n rows:    carried through kappa(S)                    (n + 1) u
  * Z = L^-1 HP (with D^-1/2):          n terms, sqrt and division                  (n + 3) u
  * Z'Z and the subtraction from P:     n terms, one subtraction                    (n + 1) u
  one pass: 2 l_nz + 3 n + 14.
  The row-chunked form (the rows eliminated h at a time, each chunk a downdate of what the earlier ones left) pays one pass of h rows
  per chunk, c = ceil(n / h) chunks, and forms each chunk's residual v_k = v_k(m_0) - H_k (m_cur - m_0): l_nz terms and a subtraction,
  with m_cur - m_0 accumulated over c chunks: c (2 l_nz + 3 h + 14) + l_nz + 1 + c.
C_VIS is that count rounded up to a power of two (n = 84, l_nz = 160: 586 -> 1024). It does not depend on what any kernel produces."""
import functools

import numpy as np

import ekf_ops_ref as E
import ekf_script
import kalman_ref as K

LD = np.longdouble
U = 2.0 ** -53
R_VIS, R_CHECK = 0.05, 0.07     # visualR, and a second noise level for the check of the speculative update
LAYOUTS = ((20, 0), (30, 0), (20, 14), (20, 47), (20, 80))      # N = 160, 230, 202, 301, 400
EK2_MIN_CHUNK = 8


# ------------------------------------------------------------------------------------------------ kernel form of a measurement
def chunk_rows(n, l, N):
    """Rows per chunk of the row-chunked cluster form (ekf_cluster2.cu ekf_cluster2_chunk_rows: the largest h whose working set fits,
    with ek2_geom_chunked's buffers: no symmetrisation buffer, N + n extra doubles); 0 if none fits."""
    if N > K.EK2_MAXN:
        return 0
    for h in range(n, max(0, min(n, EK2_MIN_CHUNK) - 1), -1):
        B = (N + K.EK2_C - 1) // K.EK2_C
        sym = N * B if h <= 8 else 0
        byts = K.ek2_smem_bytes(h, l, N)[0] - 8 * sym + 8 * ((N + n + 1) & ~1)
        if byts + K.EK2_STATIC_SMEM <= K.EK2_SMEM_LIMIT:
            return h
    return 0


def chain_chunks(n, l, N):
    """Chunks the device chain (hv_ekf_visual_tracks) runs an (n, l) update in: 1 where it fits the cluster kernel whole."""
    if K.cluster_fits(n, l, N):
        return 1
    h = chunk_rows(n, l, N)
    assert h > 0, (n, l, N)
    return -(-n // h)


def c_vis(n, l_nz, chunks=1):
    """C_VIS(n, l_nz) of the module docstring, for an update run in `chunks` row chunks."""
    if chunks <= 1:
        t = 2 * l_nz + 3 * n + 14
    else:
        h = -(-n // chunks)
        t = chunks * (2 * l_nz + 3 * h + 14) + l_nz + 1 + chunks
    return float(2 ** int(np.ceil(np.log2(t))))


# ------------------------------------------------------------------------------------------------ the reference
def _solve_ld(L, B):
    return K._chol_solve(L, B)


def update(m, P, H, f, y, r, noise_scale, trail, chunks=1, stale_residual=False):
    """The visual update of (m, P) as an ekf_ops_ref.Result (longdouble values, per-entry bounds); None if S is not positive definite.
    chunks > 1 computes the update as the row-chunked form does (a downdate per chunk of rows, residual v_k - H_k (m_cur - m_0)); in
    exact arithmetic that is the same update. stale_residual (a fault): every chunk's residual without the - H_k (m_cur - m_0) term."""
    H = np.asarray(H, dtype=LD)
    n, l = H.shape
    inn = K.Innovation(P, H, f, y, r, noise_scale)
    if inn.L is None:
        return None
    m0, P0 = np.asarray(m, dtype=LD), np.asarray(P, dtype=LD)
    if chunks <= 1:
        W = _solve_ld(inn.L, inn.HP)                          # S^-1 HP = K'
        m1 = m0 + W.T @ inn.v
        P1 = P0 - inn.HP.T @ W
    else:
        h = -(-n // chunks)
        m1, P1 = m0.copy(), P0.copy()
        for r0 in range(0, n, h):
            Hk = H[r0:r0 + h]
            vk = inn.v[r0:r0 + h] - (0 if stale_residual else Hk @ (m1[:l] - m0[:l]))
            k_inn = K.Innovation(P1, Hk, np.zeros(len(Hk)), np.zeros(len(Hk)), r, noise_scale)
            W = _solve_ld(k_inn.L, k_inn.HP)
            m1 = m1 + W.T @ vk
            P1 = P1 - k_inn.HP.T @ W
    kap = float(np.linalg.cond(np.asarray(inn.S, dtype=np.float64)))
    l_nz = int((np.abs(H).sum(axis=0) != 0).sum())
    C = c_vis(n, l_nz, chunks)
    aHP = np.abs(H) @ np.abs(P0[:l])
    aK = aHP.T @ np.abs(_solve_ld(inn.L, np.eye(n, dtype=LD)))     # |K| = |P_l|' |H|' |S^-1|
    X = aK @ aHP
    BP = np.where(X != 0, LD(C * U * kap) * (np.abs(P0) + X), LD(0))
    av = np.abs(inn.v) + LD(U) * (np.abs(np.asarray(y, dtype=LD)) + np.abs(np.asarray(f, dtype=LD)))
    Xm = aK @ av
    Bm = np.where(Xm != 0, LD(C * U * kap) * (np.abs(m0) + Xm), LD(0))
    res = E.Result(m1, P1, Bm, E._sym(BP))
    E._normalize(res.m, res.Bm, E.quaternion_offsets(trail, False))
    res.kappa, res.C = kap, C
    return res


def worst(res, m, P, trail, map_size):
    """(ratio, what) of the worst entry of m and P against the bound, with its index, block and 8-CTA column block."""
    N = len(res.m)
    B = (N + K.EK2_C - 1) // K.EK2_C
    rp, i, j = res.worst_entry(P)
    d = np.abs(np.asarray(m, dtype=LD) - res.m)
    zero = res.Bm == 0
    rm_all = np.where(zero, np.where(d > 0, LD(np.inf), LD(0)), d / np.where(zero, LD(1), res.Bm))
    k = int(np.argmax(rm_all))
    rm = float(rm_all[k])
    if rp >= rm:
        return rp, (f"P[{i},{j}] ({E.block_of(i, trail, map_size)} x {E.block_of(j, trail, map_size)}, column block {j // B} of 8)")
    return rm, f"m[{k}] ({E.block_of(k, trail, map_size)}, column block {k // B} of 8)"


# ------------------------------------------------------------------------------------------------ states
def oracle_params(trail, map_size):
    from oracle import ekf_oracle
    o = ekf_oracle.OracleEKF()
    p = o.default_params()
    o.close()
    p.camera_trail_length, p.hybrid_map_size = trail, map_size
    return p


def _map_points(o, map_size, seed):
    """Fills every map slot with insert_map_point, points a few metres around the current position."""
    m, _ = o.download()
    rng = np.random.RandomState(seed)
    for i in range(map_size):
        o.insert_map_point(i, m[0:3] + rng.normal(0, 3.0, 3))


STATES = ("fresh", "filled", "bench1", "bench20", "bench140", "trail30", "map14", "map47", "map80")


@functools.lru_cache(maxsize=None)
def _bench_states():
    """The filter of the benchmark's frame loop (config 2 with the frame pool of the driver runs, frame_loop_replay) at frames 1, 20, 140."""
    import torch
    import bench
    import frame_loop_replay as R
    out = {}
    with R.configured(2, 8):
        rep = R.FilterReplay(bench.Inputs(torch.device("cpu")))
        for k in range(1, 141):
            rep.step()
            if k in (1, 20, 140):
                out[k] = rep.o.download()
        rep.close()
    return out


@functools.lru_cache(maxsize=None)
def state(kind):
    """(trail, map_size, m, P) of a filter state, P exactly symmetric:
    fresh      initialize_orientation, seven predicts and one augmentation (slot 1 filled, slots 2..20 at the 1e8 priors);
    filled     a trail-20 filter after 60 frames of tests/ekf_script.run_frames (every slot filled);
    bench<k>   the benchmark's frame loop after frame k;
    trail30    a trail-30 filter filled the same way (N = 230);
    map<s>     the filled trail-20 filter with s hybrid-map points, every slot set by insert_map_point (N = 202, 301, 400)."""
    from oracle import ekf_oracle
    if kind.startswith("bench"):
        m, P = _bench_states()[int(kind[5:])]
        return 20, 0, m, E.symmetrize_fp64(P)
    trail, ms = {"trail30": (30, 0), "map14": (20, 14), "map47": (20, 47), "map80": (20, 80)}.get(kind, (20, 0))
    o = ekf_oracle.OracleEKF(oracle_params(trail, ms))
    if kind == "fresh":
        E.start_state(o, "fresh")
        o.augment(-1)
    else:
        ekf_script.run_frames(o, frames=60, n_list=(8, 20, 40))
    if ms:
        _map_points(o, ms, 5 + ms)
    m, P = o.download()
    o.close()
    return trail, ms, m, E.symmetrize_fp64(P)


# ------------------------------------------------------------------------------------------------ measurements
@functools.lru_cache(maxsize=None)
def rig():
    """imuToCamera / secondImuToCamera of a stereo rig (tests/tri_common.make_track): 11 cm baseline, camera along the IMU z axis."""
    t = __import__("tri_common").make_track(5)
    return t["T1"], t["T2"]


@functools.lru_cache(maxsize=None)
def _tri():
    from oracle import tri_oracle
    return tri_oracle.OracleTri()


def _camera(m, i, T):
    o = 0 if i == 0 else 20 + 7 * (i - 1)
    q = m[6:10] if i == 0 else m[o + 3:o + 7]
    R = T[:3, :3] @ __import__("tri_common").quat2rmat(q)
    return m[o:o + 3] - R.T @ T[:3, 3], R


class Track:
    """One track observed from the state's own mean: pose indices, observations ip / velocities (the chain's input) and the model's
    H, f from the C oracle (oracle/hv_oracle_tri.c)."""

    def __init__(self, m, trail, idx, stereo, time_shift, seed):
        T1, T2 = rig()
        rng = np.random.RandomState(seed)
        c0, R0 = _camera(m, 0, T1)
        depth = rng.uniform(2.0, 6.0)
        pf = c0 + R0.T @ np.array([rng.uniform(-0.3, 0.3) * depth, rng.uniform(-0.2, 0.2) * depth, depth])
        ip = __import__("tri_common").project(m, idx, T1, T2, stereo, pf)
        self.ip = ip + rng.normal(0, 1e-3, ip.shape)
        self.vel = rng.normal(0, 0.05, ip.shape)
        self.idx, self.stereo, self.time_shift = np.asarray(idx, np.int32), stereo, time_shift
        o = _tri().track_model(m, trail, stereo, self.idx, T1, T2, self.ip, self.vel, time_shift)
        self.ok = o["tri_status"] == 0 and o["vu_status"] == 0
        self.H, self.f = o["H"], o["f"]

    @property
    def obs(self):
        """(pose_trail_index, ip, velocities) as hv_ekf_visual_tracks takes a track."""
        return self.idx, self.ip, self.vel


def make_track(m, trail, npose, stereo, time_shift, seed):
    """A track of npose poses (the current one and npose - 1 of the first min(trail, 20) filled slots) that the model accepts."""
    top = 0
    while top < min(trail, 20) and np.abs(m[20 + 7 * top + 3:20 + 7 * top + 7]).sum() > 0:
        top += 1
    assert npose - 1 <= top, (npose, top)
    for k in range(50):
        rng = np.random.RandomState(seed * 100 + k)
        idx = np.concatenate([[0], np.sort(rng.choice(np.arange(1, top + 1), npose - 1, replace=False))])
        t = Track(m, trail, idx, stereo, time_shift, seed * 100 + k)
        if t.ok:
            return t
    raise AssertionError(f"no track of {npose} poses the model accepts (seed {seed})")


class Case:
    """One measurement against one state: H (n x l), f, an inlier y and a gross outlier y_out, the tracks it stacks and its kernel path."""

    def __init__(self, state_kind, spec, seed):
        self.state, self.spec = state_kind, spec
        self.trail, self.ms, self.m, self.P = state(state_kind)
        self.N = len(self.m)
        self.tracks = [make_track(self.m, self.trail, npose, stereo, ts, seed + 17 * i) for i, (npose, stereo, ts) in enumerate(spec)]
        n = sum(len(t.f) for t in self.tracks)
        l = max(t.H.shape[1] for t in self.tracks)
        self.H = np.zeros((n, l), order="F")
        r = 0
        for t in self.tracks:
            self.H[r:r + len(t.f), :t.H.shape[1]] = t.H
            r += len(t.f)
        self.f = np.concatenate([t.f for t in self.tracks])
        self.n, self.l = n, l
        rng = np.random.RandomState(seed + 5)
        S = np.asarray(K.Innovation(self.P, self.H, self.f, self.f, R_VIS, 100.0).S, dtype=np.float64) / 1e4
        Lc = np.linalg.cholesky(S)
        self.y = self.f + 0.5 * Lc @ rng.normal(0, 1.0, n)
        self.y_out = self.f + 40.0 * Lc @ rng.normal(0, 1.0, n)
        self.path = K.kernel_path(n, l, self.N)
        self.path_misaligned = K.kernel_path(n, l, self.N, h_aligned=False)

    @property
    def name(self):
        sp = "+".join(f"{'s' if st else 'm'}{p}{'' if ts else 'x'}" for p, st, ts in self.spec)
        return f"{self.state}-N{self.N}-n{self.n}-l{self.l}-{sp}"

    def reference(self, y=None, r=R_VIS, H=None, f=None, chunks=1, **kw):
        return update(self.m, self.P, self.H if H is None else H, self.f if f is None else f, self.y if y is None else y, r, 100.0,
                      self.trail, chunks, **kw)


# (npose, stereo, time shift) per stacked track: stereo tracks give 4 rows per pose, mono 2
_S = lambda p, ts=True: (p, True, ts)
_M = lambda p, ts=True: (p, False, ts)
SPECS = {
    # N = 160: n = 8 / 24 (Z through DSMEM) and 26 / 32 (L2) on either side of n N = 4096, 32 / 34 on either side of the two-stage S,
    # 56 / 60 on either side of the bulk S exchange, 84 (the longest track), 88 (single CTA, shared tableau), 96 / 100 on either side
    # of the global tableau, 160 = N
    "filled": [(_S(2),), (_M(5, False),), (_S(6),), (_M(13),), (_S(8, False),), (_M(17),), (_S(9),), (_S(10),), (_S(14),), (_S(15),), (_S(21),),
               (_S(21), _M(2)), (_S(21), _S(3)), (_S(21), _M(8, False)), (_S(21), _S(19)), (_M(2), _S(5), _M(3))],
    "fresh": [(_S(2),), (_S(2, False),), (_S(2), _S(2))],          # (one pose in the trail: only the stereo pair triangulates)
    "bench1": [(_S(2),), (_S(2), _S(2), _M(2))],
    "bench20": [(_S(9),), (_S(21),), (_S(14), _M(21))],
    "bench140": [(_S(14),), (_S(21), _S(4)), (_M(21, False), _S(21))],
    "trail30": [(_S(3),), (_M(8),), (_S(6),), (_S(12),), (_S(15),), (_S(17),), (_S(21),)],
    "map14": [(_M(2),), (_S(6),), (_S(9),), (_S(15),), (_S(21),), (_S(21), _S(2))],
    "map47": [(_M(2),), (_S(3),), (_M(10),), (_S(9),), (_S(12),), (_S(21),)],
    "map80": [(_M(2),), (_S(2),), (_M(5),), (_M(6),), (_S(9),), (_S(21),)],
}


@functools.lru_cache(maxsize=None)
def cases():
    out = []
    for kind in STATES:
        for i, spec in enumerate(SPECS[kind]):
            out.append(Case(kind, spec, 1000 * STATES.index(kind) + 10 * i))
    return tuple(out)


CHECK_BATCH_N = (8, 20, 40, 84)     # the rows of the benchmark's check batch (bench.N_ROWS of config 2)
