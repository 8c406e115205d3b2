"""GPU sweep of the pose augmentation, the fixed-H updates and the structural operations against the extended-precision reference
(tests/ekf_ops_ref.py), through the C ABI only: state layouts on both sides of the cluster / single-CTA boundaries of the augmentation
(N = 200 / 201) and of the fixed-H updates (N = 323 / 324, 328 / 329) up to N = 768, fresh (1e8 trail priors), filled and dense states,
the fused deferred symmetrisation, the augmentation as the extra cluster of a check batch, chained augmentations, and the no-ops. Every
entry of m and P must lie within the reference's componentwise bound (entries with a zero bound exact); the worst error / bound is printed
per case with the block it falls in and the kernel that ran."""
import ctypes
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import ekf_common as C
import ekf_ops_ref as E
import kalman_ref as K

pytestmark = pytest.mark.gpu
LAYOUTS = ((5, 2), (6, 0), (20, 0), (24, 4), (25, 2), (40, 0), (42, 3), (43, 1), (44, 0), (42, 5), (106, 2))
STATES = ("fresh", "filled", "dense")


def _params(trail, ms):
    from hybvio_b200 import capi
    p = capi.EkfParams()
    capi.load().hv_ekf_default_params(ctypes.byref(p))
    return C.params_with(lambda: p, trail, ms)


def _check(ops, name, ref, got, kernel, worst):
    r = ref.ratios(*got)
    _, i, j = ref.worst_entry(got[1])
    worst.append((max(r.values()), name))
    print(f"OPS N={ops.N} {name} [{kernel}]: error / bound m {r['m']:.3g} P {r['P']:.3g} "
          f"(worst P entry: {E.block_of(i, ops.trail, ops.map_size)} / {E.block_of(j, ops.trail, ops.map_size)})")
    assert max(r.values()) <= 1.0, (name, r)


@pytest.mark.parametrize("state", STATES)
@pytest.mark.parametrize("trail,ms", LAYOUTS, ids=[f"N{E.state_dim(t, m)}" for t, m in LAYOUTS])
def test_ops_match_extended_precision_reference(hv, trail, ms, state):
    """Augmentation at drop -1, 0, 1, trail - 1 (below capacity, and at capacity on the filled state), after hv_ekf_symmetrize of an
    asymmetric P (the fused symFirst), every fixed-H update, transform_to at pose -1, 0, trail - 1, insert_map_point at every index,
    condition_on_last_pose (no map), lock_biases / unaugment / translate_to bit for bit."""
    from hybvio_b200 import capi
    p = _params(trail, ms)
    base = capi.Ekf(hv, p)
    m, P, time = E.start_state(base, state)
    ops = E.Ops(p)
    N, worst = ops.N, []
    print()

    def run(name, call):
        e = base.clone()
        e.upload(m, P)
        call(e)
        got = e.download()
        e.close()
        return got

    aug_kernel = E.update_kernel("augment", N)
    for drop in sorted({-1, 0, 1, trail - 1}):
        _check(ops, f"augment[{drop}] ({base.pose_count()} poses)", ops.augment(m, P, drop), run("aug", lambda e, d=drop: e.augment(d)),
               aug_kernel, worst)
    Pa = P * (1 + 1e-9 * np.triu(np.random.RandomState(trail).uniform(-1, 1, P.shape), 1))
    e = base.clone()
    e.upload(m, Pa)
    e.symmetrize()
    e.augment(-1)
    _check(ops, "symmetrize + augment[-1]", ops.augment(m, Pa, -1, sym_first=True), e.download(), aug_kernel, worst)
    e.close()
    for name, call, ref in E.fixed_h_ops(ops, m, P, time):
        op = "zupt" if name == "zupt_initialization" else name
        kern = E.update_kernel(op, N) if op in E.FIXED_H else "ekf_ew_kernel / ekf_ew_heavy_kernel"
        _check(ops, name, ref(), run(name, call), kern, worst)
    for k in range(ms):
        got = run("ins", lambda e, k=k: e.insert_map_point(k, [3.0, -2.0, 8.0]))
        want = ops.insert_map_point_fp64(m, P, k, [3.0, -2.0, 8.0])
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), f"insert_map_point[{k}]"
    got = run("lock", lambda e: e.lock_biases())
    assert all(np.array_equal(a, b) for a, b in zip(got, ops.lock_biases_fp64(m, P))), "lock_biases"
    got = run("tr", lambda e: e.translate_to([1.0, 2.0, 3.0]))
    assert np.array_equal(got[0], ops.translate_to_fp64(m, [1.0, 2.0, 3.0])) and np.array_equal(got[1], P), "translate_to"
    if state == "filled":
        got = run("unaug", lambda e: e.unaugment())
        assert all(np.array_equal(a, b) for a, b in zip(got, ops.unaugment_fp64(m, P))), "unaugment"
    base.close()
    print(f"OPS N={N} {state}: worst " + ", ".join(f"{n} {w:.3g}" for w, n in sorted(worst)[-3:]))


def test_chained_augmentations_from_fresh_filter(hv):
    """Twelve augmentations in a row from a fresh filter (trail 6: past capacity), each compared with the reference applied to the
    previous result, with a few predicts in between: the new slot's error must not build up."""
    from hybvio_b200 import capi
    import ekf_script
    p = _params(6, 0)
    e = capi.Ekf(hv, p)
    E.start_state(e, "fresh")
    ops = E.Ops(p)
    rng = np.random.RandomState(9)
    t, worst = 0.035, []
    print()
    for k in range(12):
        for _ in range(3):
            t += 0.005
            e.predict(t, *ekf_script.imu_sample(rng, k))
        m, P = e.download()
        P = E.symmetrize_fp64(P)
        e.upload(m, P)
        e.augment(-1 if k % 3 else k % 6)
        _check(ops, f"chain {k}", ops.augment(m, P, -1 if k % 3 else k % 6), e.download(), E.update_kernel("augment", ops.N), worst)
    e.close()


@pytest.mark.parametrize("trail,ms", [(t, m) for t, m in LAYOUTS if E.state_dim(t, m) <= 200])
def test_augmentation_in_check_batch(hv, trail, ms):
    """[3 outlier checks, SYMMETRIZE, AUGMENT] through hv_ekf_run_host and hv_ekf_run_device: the augmentation runs as the extra cluster of
    the check batch, into the second buffers, with the deferred symmetrisation fused."""
    import torch
    from hybvio_b200 import capi
    p = _params(trail, ms)
    base = capi.Ekf(hv, p)
    m, P, _ = E.start_state(base, "filled")
    N = base.N
    Pa = P * (1 + 1e-9 * np.triu(np.random.RandomState(5).uniform(-1, 1, P.shape), 1))
    ref = E.Ops(p).augment(m, Pa, 2, sym_first=True)
    keep = []
    for device in (False, True):
        ops = (capi.EkfOp * 5)()
        for i in range(3):
            n = 4 + 4 * i
            l = K.visual_l(n, N)
            H, f = K.make_measurement(n, l, 50 + i)
            arrs = [np.asfortranarray(H), np.ascontiguousarray(f), np.ascontiguousarray(f + 0.01)]
            if device:
                arrs = [torch.from_numpy(np.asarray(a).ravel(order="F")).cuda() for a in arrs]
            keep += arrs
            ptr = (lambda a: a.data_ptr()) if device else (lambda a: a.ctypes.data)
            ops[i].kind, ops[i].n, ops[i].l, ops[i].mode, ops[i].r, ops[i].rmse_thr = capi.OP_VISUAL, n, l, 0, 0.05, -1.0
            ops[i].H, ops[i].f, ops[i].y = ptr(arrs[0]), ptr(arrs[1]), ptr(arrs[2])
        ops[3].kind = capi.OP_SYMMETRIZE
        ops[4].kind, ops[4].index = capi.OP_AUGMENT, 2
        e = base.clone()
        e.upload(m, Pa)
        torch.cuda.synchronize()
        if device:
            e.run_device(ops, 5)
        else:
            e.run_host(ops, 5)
        got = e.download()
        e.close()
        _check(E.Ops(p), f"check batch + augment ({'run_device' if device else 'run_host'})", ref, got, "ekf_check_batch_cluster2_kernel", [])
    base.close()


@pytest.mark.parametrize("trail,ms", ((6, 0), (43, 1)))
def test_rate_limited_and_zero_speed_updates_are_no_ops(hv, trail, ms):
    """A rate-limited zupt / zrupt / zupt-initialisation leaves the state bit-identical and, after a flush, issues no launch of its own.
    A pseudo-velocity update at horizontal speed <= 1e-7 leaves the state bit-identical (that decision reads the device-resident mean, so
    the kernel makes it)."""
    from hybvio_b200 import capi
    p = _params(trail, ms)
    e = capi.Ekf(hv, p)
    m, P, _ = E.start_state(e, "fresh")
    e.update_zupt(1e-2)
    e.update_zrupt([0.0, 0.0, 0.1])
    e.update_zupt_initialization()          # wasStationary after the zupt: a no-op from now on
    e.flush()
    before = e.download()
    n0 = hv.launches
    e.update_zupt(1e-2)
    e.update_zrupt([0.0, 0.0, 0.1])
    e.update_zupt_initialization()
    assert hv.launches == n0, "a rate-limited update launched a kernel"
    after = e.download()
    assert all(np.array_equal(a, b) for a, b in zip(before, after))
    f = capi.Ekf(hv, p)
    m2 = m.copy()
    m2[E.VEL:E.VEL + 3] = [6e-8, -7e-8, 0.5]
    f.upload(m2, P)
    f.update_pseudo_velocity(0.7, 1.0)
    got = f.download()
    assert np.array_equal(got[0], m2) and np.array_equal(got[1], P)
    e.close(); f.close()
