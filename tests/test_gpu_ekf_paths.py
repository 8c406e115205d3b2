"""GPU sweep of the dense visual update paths: every kernel / S reduction / Z exchange / staging combination the launchers pick
(shapes from tests/kalman_ref.sweep_shapes, derived from the predicates), through every entry point, against the extended-precision
reference (tolerance tau = 8 n u kappa(S), the observed error / tau is printed) and the C oracle (the 1e-9 gates of the other EKF tests);
which kernel ran at the cluster / single-CTA boundaries; and IMU bursts of every length the predict launch handles."""
import ctypes
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import ekf_common as C
import ekf_script
import kalman_ref as K
import visual_update_ref as V

pytestmark = pytest.mark.gpu
R, R_CHECK, NS = 0.05, 0.07, 100.0
KAPPA = 1e3


def default_params():
    from hybvio_b200 import capi
    p = capi.EkfParams()
    capi.load().hv_ekf_default_params(ctypes.byref(p))
    return p


def _params(trail, ms):
    return C.params_with(default_params, trail, ms)


class Case:
    """One shape: state, an inlier and a gross outlier measurement, and the reference results."""

    def __init__(self, trail, ms, n, l, seed):
        self.trail, self.ms, self.n, self.l = trail, ms, n, l
        self.N = K.state_dim(trail, ms)
        self.m, self.P = K.make_state(trail, ms, n, l, KAPPA, seed)
        self.H, self.f = K.make_measurement(n, l, seed)
        self.y = self.f + K.residual(self.P, self.H, R, NS, 0.5, seed)
        self.y_out = self.f + K.residual(self.P, self.H, R, NS, 40.0, seed + 1)
        self.kappa = K.kappa_S(self.P, self.H, R, NS)
        self.tau = K.tau(n, self.kappa)
        self.ref = K.update(self.m, self.P, self.H, self.f, self.y, R, NS, trail)
        self.ref_c = V.update(self.m, self.P, self.H, self.f, self.y, R, NS, trail)
        self.checkable = n <= K.CHI2_MAX_N
        if self.checkable:
            thr = K.chi2inv95(n)
            self.ref_in = K.check(self.P, self.H, self.f, self.y, R, NS)
            self.ref_in2 = K.check(self.P, self.H, self.f, self.y, R_CHECK, NS)
            self.ref_out = K.check(self.P, self.H, self.f, self.y_out, R, NS)
            assert self.ref_in[0] == 0 and self.ref_in2[0] == 0 and self.ref_out[0] == 3
            for _, c2 in (self.ref_in, self.ref_in2, self.ref_out):           # no decision within tau of the threshold
                assert abs(float(c2) - thr) > 1e-6 * thr
        self.worst = self.worst_c = 0.0

    def state_ratio(self, got):
        em, eP = K.errors(self.ref[0], self.ref[1], got[0], got[1])
        return max(em, eP) / self.tau

    def assert_state(self, got, what):
        r = self.state_ratio(got)
        self.worst = max(self.worst, r)
        assert r <= 1.0, f"{what}: error / tau = {r:.3g}"
        rc, where = V.worst(self.ref_c, got[0], got[1], self.trail, self.ms)
        self.worst_c = max(self.worst_c, rc)
        assert rc <= 1.0, f"{what}: per-entry ratio {rc:.3g} at {where}"

    def assert_check(self, st, c2, ref, what):
        assert st == ref[0], f"{what}: status {st} != {ref[0]}"
        r = K.chi2_error(ref[1], c2) / self.tau
        self.worst = max(self.worst, r)
        assert r <= 1.0, f"{what}: chi2 error / tau = {r:.3g}"


def _assert_oracle(got, ora, what):
    assert np.abs(got[0] - ora[0]).max() < C.TOL_M, what
    assert ekf_script.rel_err(got[1], ora[1]) < C.TOL_P_REL, what


SHAPES = K.sweep_shapes()


@pytest.mark.parametrize("trail,ms,n,l", SHAPES, ids=[f"N{K.state_dim(t, ms)}-n{n}-l{l}" for t, ms, n, l in SHAPES])
def test_update_path_matches_extended_precision_reference(hv, oracle_lk, trail, ms, n, l):
    """visual_check (inlier / gross outlier), visual_update, visual_check_update, a check followed by the update of the same measurement
    with another noise level (the speculative update adopted by pointer swap), and a device list whose H / f / y start 8 bytes past a
    16-byte boundary (no bulk copy of H), on an uploaded state."""
    import torch
    from hybvio_b200 import capi
    from oracle import ekf_oracle
    c = Case(trail, ms, n, l, seed=7 * n + l)
    p = _params(trail, ms)
    e, o = capi.Ekf(hv, p), ekf_oracle.OracleEKF(p)
    H, f, y = c.H, c.f, c.y
    o.upload(c.m, c.P)
    o.visual_update(H, f, y, R)
    ora = o.download()
    o.close()

    e.upload(c.m, c.P)
    e.visual_update(H, f, y, R)
    got = e.download()
    c.assert_state(got, "visual_update")
    _assert_oracle(got, ora, "visual_update vs oracle")

    if c.checkable:
        e.upload(c.m, c.P)
        c.assert_check(*e.visual_check(H, f, y, R), c.ref_in, "visual_check inlier")
        c.assert_check(*e.visual_check(H, f, c.y_out, R), c.ref_out, "visual_check outlier")
        m_, P_ = e.download()
        assert np.array_equal(m_, c.m) and np.array_equal(P_, c.P), "a check changed the state"

        e.upload(c.m, c.P)
        st, c2, m_out = e.visual_check_update(H, f, y, R)
        c.assert_check(st, c2, c.ref_in, "visual_check_update")
        got = e.download()
        assert np.array_equal(m_out, got[0])
        c.assert_state(got, "visual_check_update")
        _assert_oracle(got, ora, "visual_check_update vs oracle")
        e.upload(c.m, c.P)
        st, c2, _ = e.visual_check_update(H, f, c.y_out, R)
        c.assert_check(st, c2, c.ref_out, "visual_check_update outlier")
        m_, P_ = e.download()
        assert np.array_equal(m_, c.m) and np.array_equal(P_, c.P), "an outlier changed the state"

        # speculative two-R path: an update at R arms it, the check at R_CHECK computes the update at R into the second buffers
        e.upload(c.m, c.P)
        e.visual_update(H, f, y, R)
        e.upload(c.m, c.P)
        c.assert_check(*e.visual_check(H, f, y, R_CHECK), c.ref_in2, "check before the speculative update")
        e.visual_update(H, f, y, R)
        got = e.download()
        c.assert_state(got, "check + update (speculative)")
        _assert_oracle(got, ora, "check + update vs oracle")

        # device list, misaligned inputs: one check+update op
        nl = n * l
        buf = torch.zeros(nl + 2 * n + 2, dtype=torch.float64, device="cuda")
        assert buf.data_ptr() % 16 == 0
        buf[1:1 + nl] = torch.from_numpy(np.asfortranarray(H).ravel(order="F")).cuda()
        buf[1 + nl:1 + nl + n] = torch.from_numpy(f).cuda()
        buf[1 + nl + n:1 + nl + 2 * n] = torch.from_numpy(y).cuda()
        base = buf.data_ptr() + 8
        ops = (capi.EkfOp * 1)()
        ops[0].kind, ops[0].n, ops[0].l, ops[0].mode, ops[0].r, ops[0].rmse_thr = capi.OP_VISUAL, n, l, 2, R, -1.0
        ops[0].H, ops[0].f, ops[0].y = base, base + 8 * nl, base + 8 * (nl + n)
        torch.cuda.synchronize()
        e.upload(c.m, c.P)
        e.run_device(ops, 1)
        st, c2 = e.run_device_results(1)
        c.assert_check(int(st[0]), float(c2[0]), c.ref_in, "run_device (misaligned)")
        got = e.download()
        c.assert_state(got, "run_device (misaligned)")
        _assert_oracle(got, ora, "run_device vs oracle")
        del buf
    e.close()
    path = K.kernel_path(n, l, c.N)
    print(f"\nPATH N={c.N} n={n} l={l} {'/'.join(path)} (misaligned H: {'/'.join(K.kernel_path(n, l, c.N, h_aligned=False))}) "
          f"kappa={c.kappa:.3g} worst error / tau = {c.worst:.3g}, worst per-entry ratio = {c.worst_c:.3g}")


@pytest.mark.parametrize("trail,ms", K.CONFIGS)
def test_host_list_of_checks_across_batch_splits(hv, oracle_lk, trail, ms):
    """hv_ekf_run_host with 27 consecutive outlier checks (more than the 24 of one batch launch) of assorted shapes, with one check in the
    middle that does not fit the cluster kernel (it breaks the batch) where the state has one; statuses and chi2 against the reference."""
    from hybvio_b200 import capi
    N = K.state_dim(trail, ms)
    big = [n for t, m_, n, l in SHAPES if (t, m_) == (trail, ms) and n <= K.CHI2_MAX_N and K.kernel_path(n, l, N)[0] != "cluster"]
    small = [n for t, m_, n, l in SHAPES if (t, m_) == (trail, ms) and K.kernel_path(n, l, N)[0] == "cluster"]
    ns = [small[i % len(small)] for i in range(27)]
    if big:
        ns[13] = big[0]
    m, P = K.make_state(trail, ms, 16, K.visual_l(16, N), KAPPA, 5)
    ops = (capi.EkfOp * len(ns))()
    keep, exp = [], []
    for i, n in enumerate(ns):
        l = K.visual_l(n, N)
        H, f = K.make_measurement(n, l, 100 + i)
        y = f + K.residual(P, H, R, NS, 0.5 if i % 3 else 40.0, 100 + i)
        H, f, y = np.asfortranarray(H), np.ascontiguousarray(f), np.ascontiguousarray(y)
        keep += [H, f, y]
        ops[i].kind, ops[i].n, ops[i].l, ops[i].mode, ops[i].r, ops[i].rmse_thr = capi.OP_VISUAL, n, l, 0, R, -1.0
        ops[i].H, ops[i].f, ops[i].y = H.ctypes.data, f.ctypes.data, y.ctypes.data
        st, c2 = K.check(P, H, f, y, R, NS)
        assert abs(float(c2) - K.chi2inv95(n)) > 1e-6 * K.chi2inv95(n)
        exp.append((st, c2, K.tau(n, K.kappa_S(P, H, R, NS))))
    e = capi.Ekf(hv, _params(trail, ms))
    e.upload(m, P)
    st, c2, _ = e.run_host(ops, len(ns))
    for i, (s_, c_, t) in enumerate(exp):
        assert st[i] == s_, f"op {i} (n={ns[i]}): status {st[i]} != {s_}"
        assert K.chi2_error(c_, c2[i]) <= t, f"op {i} (n={ns[i]}): chi2 error / tau = {K.chi2_error(c_, c2[i]) / t:.3g}"
    m_, P_ = e.download()
    assert np.array_equal(m_, m) and np.array_equal(P_, P)
    e.close()


HV_RUN_MAX_OPS = 256


def _host_frames(capi, N, frames, seed):
    """`frames` frames of a host op list: 10 IMU predicts, one check + update, 8 outlier checks (every third a gross outlier), symmetrise,
    augment. Returns the ops, the ops per frame and the arrays they point into."""
    rng, irng = np.random.RandomState(seed), np.random.RandomState(seed + 1)
    per = 10 + 1 + 8 + 2
    ops = (capi.EkfOp * (per * frames))()
    keep, t, k = [], 0.0, 0
    for fr in range(frames):
        for s_ in range(10):
            t += 0.005
            g, a = ekf_script.imu_sample(irng, 10 * fr + s_ + 1)
            ops[k].kind, ops[k].t = capi.OP_PREDICT, t
            for q in range(3):
                ops[k].gyro[q], ops[k].acc[q] = g[q], a[q]
            k += 1
        for c in range(9):
            H, f, y = ekf_script.visual_measurement(rng, (8, 20)[c % 2], N, 40.0 if c % 3 == 2 else 0.02)
            H, f, y = np.asfortranarray(H), np.ascontiguousarray(f), np.ascontiguousarray(y)
            keep += [H, f, y]
            op = ops[k]
            op.kind, op.n, op.l, op.mode, op.r, op.rmse_thr = capi.OP_VISUAL, H.shape[0], H.shape[1], 2 if c == 0 else 0, ekf_script.VISUAL_R, -1.0
            op.H, op.f, op.y = H.ctypes.data, f.ctypes.data, y.ctypes.data
            k += 1
        ops[k].kind = capi.OP_SYMMETRIZE
        ops[k + 1].kind, ops[k + 1].index = capi.OP_AUGMENT, -1
        k += 2
    return ops, per, keep


def test_host_list_longer_than_one_async_list_matches_shorter_lists(hv):
    """hv_ekf_run_host with more ops than HV_RUN_MAX_OPS cannot take the asynchronous path (one synchronisation per list) and runs op by op:
    each check batch stages its inputs and polls its results, each check + update goes through the single-measurement host call. 15
    frames (315 ops) in one call, and the same ops in calls of at most 256 ops split at frame boundaries (each taken by the asynchronous
    path) on a clone of the same filter: statuses, chi2, the returned mean and the final m and P bit for bit."""
    from hybvio_b200 import capi
    lib = capi.load()
    one = capi.Ekf(hv, _params(20, 0))
    one.initialize_orientation(ekf_script.imu_sample(np.random.RandomState(1), 0)[1])
    split = one.clone()
    frames = 15
    ops, per, keep = _host_frames(capi, one.N, frames, 9)
    nops = per * frames
    assert nops > HV_RUN_MAX_OPS
    for i in range(nops):        # every check joins a check batch on both paths
        assert ops[i].kind != capi.OP_VISUAL or ops[i].mode != 0 or K.kernel_path(ops[i].n, ops[i].l, one.N)[0] == "cluster"

    def host_times(e):           # {issue, wait, total, ops} of the last list the asynchronous path ran
        t = (ctypes.c_double * 4)()
        assert lib.hv_ekf_debug_host_times(e.h, t) == 0
        return list(t)

    before = host_times(one)
    st, c2, m = one.run_host(ops, nops, want_m=True)
    assert host_times(one) == before, "the asynchronous path took a list longer than it accepts"

    step = HV_RUN_MAX_OPS // per * per
    parts = []
    for start in range(0, nops, step):
        cnt = min(step, nops - start)
        chunk = (capi.EkfOp * cnt).from_address(ctypes.addressof(ops) + start * ctypes.sizeof(capi.EkfOp))
        parts.append(split.run_host(chunk, cnt, want_m=True))
        assert host_times(split)[3] == cnt, f"ops {start}..{start + cnt}: not run by the asynchronous path"
    visual = [i for i in range(nops) if ops[i].kind == capi.OP_VISUAL]
    assert 0 in st[visual] and (st[visual] != 0).any()
    assert np.array_equal(st, np.concatenate([p[0] for p in parts]))
    assert np.array_equal(c2.view(np.uint64), np.concatenate([p[1] for p in parts]).view(np.uint64))
    assert np.array_equal(m.view(np.uint64), parts[-1][2].view(np.uint64))
    (m1, P1), (m2, P2) = one.download(), split.download()
    assert np.array_equal(m1.view(np.uint64), m.view(np.uint64))
    assert np.array_equal(m1.view(np.uint64), m2.view(np.uint64)) and np.array_equal(P1.view(np.uint64), P2.view(np.uint64))
    one.close(); split.close()


def _boundary_shapes():
    """One shape on each side of each cluster / single-CTA boundary (and of the shared / global tableau one)."""
    out = []
    for trail, ms in ((20, 0), (40, 0)):
        N = K.state_dim(trail, ms)
        path = lambda n: K.kernel_path(n, K.visual_l(n, N), N)[0]
        for k in (K.first(lambda n: path(n) != "cluster", 1, N), K.first(lambda n: path(n) == "single-global", 1, N)):
            out += [(trail, ms, k - 1), (trail, ms, k)]
    return out


@pytest.mark.parametrize("trail,ms,n", _boundary_shapes())
def test_kernel_identity_at_path_boundaries(hv, trail, ms, n):
    """torch.profiler (CUDA activities) sees the kernels of the ctypes-loaded library: the update launches the kernel the predicates name,
    and a host list of checks that all fit the cluster kernel runs as one ekf_check_batch_cluster2_kernel."""
    import torch
    from torch.profiler import profile, ProfilerActivity
    from hybvio_b200 import capi
    N = K.state_dim(trail, ms)
    l = K.visual_l(n, N)
    m, P = K.make_state(trail, ms, n, l, KAPPA, 3)
    H, f = K.make_measurement(n, l, 3)
    y = f + K.residual(P, H, R, NS, 0.5, 3)
    e = capi.Ekf(hv, _params(trail, ms))
    e.upload(m, P)
    e.visual_update(H, f, y, R)                 # warm-up: function attributes, first launch
    e.upload(m, P)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e.visual_update(H, f, y, R)
        e.download()
        torch.cuda.synchronize()
    names = {ev.key.split("(")[0] for ev in prof.key_averages() if ev.key.startswith("ekf_")}
    want = K.KERNEL_NAME[K.kernel_path(n, l, N)[0]]
    other = ({"ekf_update_cluster2_kernel", "ekf_update_kernel"} - {want})
    print(f"\nKERNELS N={N} n={n}: {sorted(names)} (predicate: {want})")
    assert want in names and not (names & other), names
    if K.kernel_path(n, l, N)[0] == "cluster":
        ops = (capi.EkfOp * 3)()
        keep = []
        for i in range(3):
            keep += [np.asfortranarray(H), np.ascontiguousarray(f), np.ascontiguousarray(y)]
            ops[i].kind, ops[i].n, ops[i].l, ops[i].mode, ops[i].r, ops[i].rmse_thr = capi.OP_VISUAL, n, l, 0, R, -1.0
            ops[i].H, ops[i].f, ops[i].y = keep[-3].ctypes.data, keep[-2].ctypes.data, keep[-1].ctypes.data
        e.run_host(ops, 3)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            e.run_host(ops, 3)
            torch.cuda.synchronize()
        names = {ev.key.split("(")[0] for ev in prof.key_averages() if ev.key.startswith("ekf_")}
        print(f"KERNELS N={N} n={n} host list of 3 checks: {sorted(names)}")
        assert "ekf_check_batch_cluster2_kernel" in names, names
    e.close()


def _op_boundary_shapes():
    """(trail, map points, op) on each side of the cluster / single-CTA boundary of the pose augmentation (Joseph form, N = 200 / 201)
    and of the fixed-H updates (N = 323 / 324 for three and four rows, 328 / 329 for one row), from kalman_ref.cluster_fits."""
    import ekf_ops_ref as E
    out = []
    for op, lo, hi in (("augment", (24, 4), (25, 2)), ("position", (42, 3), (43, 1)), ("orientation", (42, 3), (43, 1)),
                       ("zero_height", (44, 0), (42, 5))):
        assert E.update_kernel(op, K.state_dim(*lo)) == K.KERNEL_NAME["cluster"] and E.update_kernel(op, K.state_dim(*hi)) != K.KERNEL_NAME["cluster"]
        out += [(*lo, op), (*hi, op)]
    return out


@pytest.mark.parametrize("trail,ms,op", _op_boundary_shapes())
def test_kernel_identity_of_fixed_h_ops_at_path_boundaries(hv, trail, ms, op):
    """The augmentation and the fixed-H updates launch the kernel the predicate (with the Joseph form's buffers for the augmentation)
    names, on both sides of its boundary."""
    import torch
    from torch.profiler import profile, ProfilerActivity
    from hybvio_b200 import capi
    import ekf_ops_ref as E
    N = K.state_dim(trail, ms)
    m, P = K.make_state(trail, ms, 7, 27, KAPPA, 4)
    call = {"augment": lambda e: e.augment(-1), "position": lambda e: e.update_position([0.1, -0.2, 0.05], 1e-3),
            "orientation": lambda e: e.update_orientation([1.0, 0.0, 0.0, 0.0], 1e-2), "zero_height": lambda e: e.update_zero_height(1e-3)}[op]
    e = capi.Ekf(hv, _params(trail, ms))
    e.upload(m, P)
    call(e)                                     # warm-up: function attributes, first launch
    e.upload(m, P)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call(e)
        e.download()
        torch.cuda.synchronize()
    e.close()
    names = {ev.key.split("(")[0] for ev in prof.key_averages() if ev.key.startswith("ekf_")}
    want = E.update_kernel(op, N)
    other = {"ekf_update_cluster2_kernel", "ekf_update_kernel"} - {want}
    print(f"\nKERNELS N={N} {op}: {sorted(names)} (predicate: {want})")
    assert want in names and not (names & other), names


@pytest.mark.parametrize("norm", [False, True])
def test_predict_bursts_of_every_length(hv, oracle_lk, norm):
    """With set_imu_batching(16), bursts of k = 1..17 and 33 queued samples (one launch up to 16, then split), optionally with the
    normalizeQuaternions(true) after each sample: the state against the oracle (1e-9), against batching 1 (1e-12), and the mean launch
    (predicted_mean_device) equal to the first 20 entries of the state the full launch leaves, bit for bit."""
    import torch
    from hybvio_b200 import capi
    from oracle import ekf_oracle
    p = _params(6, 0)
    d = torch.zeros(20, dtype=torch.float64, device="cuda")
    for k in list(range(1, 18)) + [33]:
        a, b, o = capi.Ekf(hv, p), capi.Ekf(hv, p), ekf_oracle.OracleEKF(p)
        a.set_imu_batching(16); b.set_imu_batching(1)
        acc0 = ekf_script.imu_sample(np.random.RandomState(1), 0)[1]
        irng = np.random.RandomState(40 + k)
        t = 0.0
        for x in (a, b, o):
            x.initialize_orientation(acc0)
        for burst in range(2):
            for s_ in range(k):
                t += 0.005
                g, acc = ekf_script.imu_sample(irng, s_ + 1)
                for x in (a, b, o):
                    x.predict(t, g, acc)
                    if norm:
                        x.normalize_quaternions(True)
            a.predicted_mean_device(d.data_ptr())
            torch.cuda.synchronize()
            pred = d.cpu().numpy().copy()
            (ma, Pa), (mb, Pb), (mo, Po) = a.download(), b.download(), o.download()
            assert np.array_equal(pred, ma[:20]), (k, burst, np.abs(pred - ma[:20]).max())
            assert np.abs(ma - mo).max() < C.TOL_M and ekf_script.rel_err(Pa, Po) < C.TOL_P_REL, (k, burst)
            assert np.abs(ma - mb).max() < 1e-12 and ekf_script.rel_err(Pa, Pb) < 1e-12, (k, burst)
            for x in (a, b, o):
                x.symmetrize(); x.augment(-1)
        for x in (a, b, o):
            x.close()
