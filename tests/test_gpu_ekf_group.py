"""GPU tests of hv_ekf_group_run_device: a group of filters stepped with one launch per step must leave every filter exactly where
hv_ekf_run_device would have left it. Twin sets of filters: set A takes per-filter calls, set B the group call; every comparison is
exact (the float64 bits of m, P, chi2; statuses, pose counts, platform times)."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import kalman_ref as K

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TRAILS = (6, 20)            # N = 62 (BASELINE config 4) and N = 160 (config 2)
R = 0.05


def _params(trail):
    from hybvio_b200 import capi
    p = capi.EkfParams()
    capi.load().hv_ekf_default_params(ctypes.byref(p))
    p.camera_trail_length = trail
    return p


def _twins(hv, trail, count):
    """Sets A and B of `count` filters; filter i of both sets starts from its own orientation."""
    from hybvio_b200 import capi
    sets = []
    for _ in range(2):
        fs = [capi.Ekf(hv, _params(trail)) for _ in range(count)]
        for i, e in enumerate(fs):
            e.initialize_orientation([0.3 * np.sin(i), 0.2 * np.cos(i), 9.8])
            e.set_first_sample_time(0.999)           # (the first PREDICT of a fresh filter adds no sample: its NORMALIZE would stand alone)
        sets.append(fs)
    return sets


class Pool:
    """Measurements in device memory (kept alive by the pool): entry k = one frame's worth of (offset, n, l) slices."""

    def __init__(self, N, seed, entries=6, nvis=20, ns=None):
        import torch
        ns = ns or [n for n in (8, 20, 40, 84) if n <= N and K.cluster_fits(n, K.visual_l(n, N), N)]
        rng = np.random.RandomState(seed)
        self.N, self.entries = N, []
        for _ in range(entries):
            parts, slices, off = [], [], 0
            for c in range(nvis):
                n = ns[(c + rng.randint(len(ns))) % len(ns)]
                l = K.visual_l(n, N) if rng.rand() < 0.7 else min(N, K.visual_l(n, N) + 7)
                H = rng.normal(0, 0.02, (n, l)); f = rng.normal(0, 0.5, n); y = f + rng.normal(0, 0.05 if rng.rand() < 0.8 else 5.0, n)
                parts += [H.ravel(order="F"), f, y]
                slices.append((off, n, l))
                off += n * l + 2 * n
            t = torch.from_numpy(np.concatenate(parts)).cuda()
            self.entries.append((t, slices))


def frame(t0, rate_seed, pool_entry=None, imu=10, normalize=True, nvis=None, modes=None, tail=("sym", "aug"), drop=-1):
    """A bench-shaped op list: `imu` predicts (+ normalise), the visual ops of a pool entry (modes[c] per op; default: 5 check+update,
    then checks), then the tail ops."""
    from hybvio_b200 import capi
    rng = np.random.RandomState(rate_seed)
    spec = []
    for s in range(imu):
        spec.append(("p", t0 + 0.005 * (s + 1), rng.normal(0, 0.1, 3), np.array([0, 0, 9.81]) + rng.normal(0, 0.3, 3)))
        if normalize:
            spec.append(("norm",))
    if pool_entry is not None:
        t, slices = pool_entry
        slices = slices[:nvis] if nvis is not None else slices
        for c, (o, n, l) in enumerate(slices):
            mode = modes[c % len(modes)] if modes else (2 if c < 5 else 0)
            spec.append(("v", t.data_ptr() + 8 * o, n, l, mode))
    for k in tail:
        spec.append((k,))
    ops = (capi.EkfOp * len(spec))()
    for op, s in zip(ops, spec):
        if s[0] == "p":
            op.kind, op.t = capi.OP_PREDICT, s[1]
            for q in range(3):
                op.gyro[q], op.acc[q] = s[2][q], s[3][q]
        elif s[0] == "norm":
            op.kind, op.index = capi.OP_NORMALIZE, 1
        elif s[0] == "v":
            _, H, n, l, mode = s
            op.kind, op.n, op.l, op.mode, op.r, op.rmse_thr = capi.OP_VISUAL, n, l, mode, R, -1.0
            op.H, op.f, op.y = H, H + 8 * n * l, H + 8 * (n * l + n)
        elif s[0] == "sym":
            op.kind = capi.OP_SYMMETRIZE
        elif s[0] == "aug":
            op.kind, op.index = capi.OP_AUGMENT, drop
    return ops


def _bits(x):
    return np.ascontiguousarray(x).view(np.uint64)


def assert_same(a, b, what=""):
    ma, Pa = a.download(); mb, Pb = b.download()
    assert np.array_equal(_bits(ma), _bits(mb)), f"{what}: m differs"
    assert np.array_equal(_bits(Pa), _bits(Pb)), f"{what}: P differs (max |d| {np.max(np.abs(Pa - Pb)):.3g})"
    assert a.pose_count() == b.pose_count(), what
    assert _bits(np.array([a.platform_time()])) == _bits(np.array([b.platform_time()])), what
    for i in range(a.pose_count()):
        assert a.history_time(i) == b.history_time(i), what


def assert_same_results(a, b, nops, what=""):
    sa, ca = a.run_device_results(nops)
    sb, cb = b.run_device_results(nops)
    assert np.array_equal(sa, sb), f"{what}: statuses {sa} != {sb}"
    assert np.array_equal(_bits(ca), _bits(cb)), f"{what}: chi2 differs"
    return sa


def step_both(A, B, lists):
    """lists[i] for filter i: set A one by one, set B in one group call; then the result words of every filter."""
    from hybvio_b200 import capi
    for e, ops in zip(A, lists):
        e.run_device(ops, len(ops))
    capi.ekf_group_run_device(B, lists)
    sts = []
    for i, (a, b, ops) in enumerate(zip(A, B, lists)):
        sts.append(assert_same_results(a, b, len(ops), f"filter {i}"))
    return sts


@pytest.mark.parametrize("trail", TRAILS)
@pytest.mark.parametrize("S", (1, 2, 3, 8, 16, 24))
def test_bench_frames(hv, trail, S):
    """S filters, each with its own IMU stream and measurements, through 20 bench frames (10 predict + normalise, 5 check+update,
    15 checks, symmetrise, augment)."""
    N = K.state_dim(trail, 0)
    pool = Pool(N, 7 + trail)
    A, B = _twins(hv, trail, S)
    seen = set()
    for k in range(20):
        lists = [frame(1.0 + 0.05 * k + 0.001 * i, 1000 * i + k, pool.entries[(3 * i + k) % len(pool.entries)]) for i in range(S)]
        for st in step_both(A, B, lists):
            seen |= set(int(x) for x in st if x >= 0)
    for i in range(S):
        assert_same(A[i], B[i], f"filter {i}")
    assert A[0].pose_count() == trail + 1
    assert 0 in seen, seen


@pytest.mark.parametrize("trail", TRAILS)
def test_heterogeneous_lists(hv, trail):
    """Different lists per filter in one group: visual ops of different counts, n and l, mode 1 updates; a list that is only an IMU
    burst, one without IMU ops, an empty one; different discarded poses; an augmentation without symmetrisation; a lone check+update;
    a run of 30 checks (more than one batch) ahead of the augmentation; a burst of 20 samples (two launches)."""
    from hybvio_b200 import capi
    N = K.state_dim(trail, 0)
    pool = Pool(N, 99, entries=3, nvis=30)
    A, B = _twins(hv, trail, 8)
    for k in range(6):
        t = 1.0 + 0.06 * k
        P_ = pool.entries
        lists = [
            frame(t, k, P_[k % 3], nvis=12, modes=(1, 0, 2)),
            frame(t, 10 + k, P_[(k + 1) % 3], imu=0, nvis=3, modes=(0,), tail=("aug",), drop=min(2, trail - 1)),
            frame(t, 20 + k, imu=10, tail=()),
            (capi.EkfOp * 0)(),
            frame(t, 40 + k, P_[(k + 2) % 3], nvis=7, modes=(2, 1), drop=k % trail),
            frame(t, 50 + k, P_[k % 3], nvis=1, modes=(2,), tail=("aug",), drop=0),
            frame(t, 60 + k, P_[(k + 1) % 3], nvis=30, modes=(0,)),
            frame(t, 70 + k, imu=20, normalize=False, tail=("sym", "aug")),
        ]
        step_both(A, B, lists)
    for i in range(len(A)):
        assert_same(A[i], B[i], f"filter {i}")


def test_launch_count(hv):
    """A group of S bench frames adds as many launches as one filter's frame (7; per filter in throughput mode as well)."""
    from hybvio_b200 import capi
    trail = 20
    pool = Pool(K.state_dim(trail, 0), 3)
    A, B = _twins(hv, trail, 8)
    for k in range(3):
        lists = [frame(1.0 + 0.05 * k + 0.001 * i, 10 * i + k, pool.entries[(i + k) % len(pool.entries)]) for i in range(8)]
        c0 = hv.launches
        capi.ekf_group_run_device(A[:1], lists[:1])
        c1 = hv.launches
        capi.ekf_group_run_device(B, lists)
        c2 = hv.launches
        assert c1 - c0 == 7 and c2 - c1 == 7, (c1 - c0, c2 - c1)
    hv.sync()


_INTERLEAVE = r"""
import ctypes, os, sys
import numpy as np
sys.path.insert(0, {root!r}); sys.path.insert(0, os.path.join({root!r}, "tests"))
import test_gpu_ekf_group as G
import kalman_ref as K
import torch
from hybvio_b200 import capi
hv = capi.Context(0)
trail = 20
N = K.state_dim(trail, 0)
pool = G.Pool(N, 5)
A, B = G._twins(hv, trail, 3)
d_mean = torch.zeros(20, dtype=torch.float64, device="cuda")
rng = np.random.RandomState(0)
def both(fn):
    for e in A + B:
        fn(e)
t = 1.0
for k in range(6):
    # per-filter calls before the group call: queued IMU samples (+ the mean launch of the burst), a deferred symmetrisation,
    # a list whose checks go to the side stream (latency mode), a speculative check (host-buffer check after an update)
    H, f = K.make_measurement(8, 34, k); y = f + 0.01
    both(lambda e: e.visual_update(H, f, y, G.R))
    both(lambda e: e.visual_check(H, f, y, G.R))
    lst = [G.frame(t + 0.001 * i, 7 * i + k, pool.entries[(i + k) % len(pool.entries)]) for i in range(3)]
    for e, ops in zip(A, lst):
        e.run_device(ops, len(ops))
    for e, ops in zip(B, lst):
        e.run_device(ops, len(ops))
    for i in range(3):
        G.assert_same_results(A[i], B[i], len(lst[i]), "per-filter list")
    t += 0.05
    for s in range(4):
        g, a = rng.normal(0, 0.1, 3), np.array([0, 0, 9.81]) + rng.normal(0, 0.3, 3)
        both(lambda e: e.predict(t + 0.005 * s, g, a))
    both(lambda e: e.predicted_mean_device(d_mean.data_ptr()))
    if k % 2:
        both(lambda e: e.symmetrize())
    lst = [G.frame(t + 0.02 + 0.001 * i, 11 * i + k, pool.entries[(2 * i + k) % len(pool.entries)]) for i in range(3)]
    G.step_both(A, B, lst)
    H, f = K.make_measurement(20, 55, 50 + k); y = f + 0.01
    both(lambda e: e.visual_update(H, f, y, G.R))
    t += 0.08
for i in range(3):
    G.assert_same(A[i], B[i], "filter %d" % i)
hv.sync()
print("interleave ok")
"""


@pytest.mark.parametrize("no_pdl", (False, True))
def test_interleaving_with_per_filter_calls(no_pdl):
    """Per-filter calls before and after group calls (queued IMU samples and their mean launch, a deferred symmetrisation, checks on
    the side stream, a speculative check), in latency mode and in throughput mode (HV_EKF_NO_PDL=1; read once per process)."""
    env = dict(os.environ)
    env.pop("HV_EKF_NO_PDL", None)
    if no_pdl:
        env["HV_EKF_NO_PDL"] = "1"
    r = subprocess.run([sys.executable, "-c", _INTERLEAVE.format(root=ROOT)], capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0 and "interleave ok" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]


def _raw(ekfs, lists, count=None):
    from hybvio_b200 import capi
    n = len(ekfs)
    E = (ctypes.c_void_p * max(n, 1))(*[e.h if e else None for e in ekfs])
    O = (ctypes.POINTER(capi.EkfOp) * max(n, 1))(*[ctypes.cast(x, ctypes.POINTER(capi.EkfOp)) if x is not None else None for x in lists])
    Kn = (ctypes.c_int * max(n, 1))(*[len(x) if x is not None else 0 for x in lists])
    return capi.load().hv_ekf_group_run_device(E, n if count is None else count, O, Kn)


def _snapshot(e):
    m, P = e.download()
    return _bits(m).copy(), _bits(P).copy(), e.pose_count(), e.platform_time()


def test_refusals(hv):
    """Every refusal returns its code before anything is issued: m, P, pose count and time bookkeeping of every filter unchanged."""
    from hybvio_b200 import capi
    lib = capi.load()
    trail = 20
    N = K.state_dim(trail, 0)
    pool = Pool(N, 11, entries=1)
    A, _ = _twins(hv, trail, 3)
    other = capi.Ekf(hv, _params(6))
    hv2 = capi.Context(0)
    foreign = capi.Ekf(hv2, _params(trail))
    big = capi.Ekf(hv, _params(26))                 # N = 202: the augmentation no longer fits the cluster kernel
    big2 = capi.Ekf(hv, _params(26))
    ok = lambda i: frame(1.0 + 0.001 * i, i, pool.entries[0])

    def with_op(kind, **kw):
        ops = ok(0)
        lst = (capi.EkfOp * (len(ops) + 1))(*ops)
        o = lst[len(ops)]
        o.kind = kind
        for k, v in kw.items():
            setattr(o, k, v)
        return lst

    nfit = K.first(lambda n: not K.cluster_fits(n, N, N), 1, N)
    H = pool.entries[0][0].data_ptr()
    too_long = frame(1.0, 3, imu=17)                          # NORMALIZE right after the 16th sample: a launch of its own
    bad = ok(0)
    bad[25].mode = 3
    nullm = ok(0)
    nullm[25].f = None
    drop = ok(0)
    drop[len(drop) - 1].index = trail
    cases = [
        ("UNAUGMENT", [A[0], A[1]], [ok(0), with_op(capi.OP_UNAUGMENT)], -5),
        ("standalone SYMMETRIZE", [A[0], A[1]], [ok(0), frame(1.0, 1, pool.entries[0], tail=("sym",))], -5),
        ("SYMMETRIZE before VISUAL", [A[0]], [with_op(capi.OP_SYMMETRIZE)], -5),
        ("standalone NORMALIZE", [A[0]], [(capi.EkfOp * 1)(capi.EkfOp(kind=capi.OP_NORMALIZE, index=1))], -5),
        ("NORMALIZE all", [A[0], A[1]], [ok(0), with_op(capi.OP_NORMALIZE, index=0)], -5),
        ("NORMALIZE after a full burst", [A[0]], [too_long], -5),
        ("measurement too large", [A[0], A[1]], [ok(0), with_op(capi.OP_VISUAL, n=nfit, l=N, mode=0, r=R, rmse_thr=-1.0, H=H, f=H, y=H)], -5),
        ("N = 202 augmentation", [big, big2], [frame(1.0, 1, imu=0, tail=("aug",)), frame(1.0, 2, imu=0, tail=())], -5),
        ("unknown kind", [A[0]], [with_op(77)], -1),
        ("bad mode", [A[0], A[1]], [ok(0), bad], -1),
        ("NULL measurement", [A[0], A[1]], [ok(0), nullm], -1),
        ("discarded pose out of range", [A[0], A[1]], [ok(0), drop], -1),
        ("other context", [A[0], foreign], [ok(0), ok(1)], -1),
        ("unequal state dimension", [A[0], other], [ok(0), frame(1.0, 1, tail=())], -1),
        ("filter twice", [A[0], A[1], A[0]], [ok(0), ok(1), ok(2)], -1),
        ("NULL filter", [A[0], None], [ok(0), ok(1)], -1),
        ("NULL list", [A[0], A[1]], [ok(0), None], -1),
    ]
    snaps = {id(e): _snapshot(e) for e in A + [other, foreign, big, big2]}
    for name, ekfs, lists, code in cases:
        assert _raw(ekfs, lists) == code, (name, lib.hv_last_error())
        for e in set(x for x in ekfs if x is not None):
            s = _snapshot(e)
            ref = snaps[id(e)]
            assert np.array_equal(s[0], ref[0]) and np.array_equal(s[1], ref[1]) and s[2:] == ref[2:], name
    E = (ctypes.c_void_p * 1)(A[0].h)
    O = (ctypes.POINTER(capi.EkfOp) * 1)(ctypes.cast(ok(0), ctypes.POINTER(capi.EkfOp)))
    Kn = (ctypes.c_int * 1)(1)
    assert lib.hv_ekf_group_run_device(E, 0, O, Kn) == -1
    assert _raw([A[0]] * 65, [ok(0)] * 65) == -1                             # count > HV_EKF_GROUP_MAX (also a duplicate)
    assert lib.hv_ekf_group_run_device(None, 1, O, Kn) == -1
    assert lib.hv_ekf_group_run_device(E, 1, None, Kn) == -1
    assert lib.hv_ekf_group_run_device(E, 1, O, None) == -1
    s = _snapshot(A[0])
    assert np.array_equal(s[0], snaps[id(A[0])][0]) and np.array_equal(s[1], snaps[id(A[0])][1])
    hv2.sync()
