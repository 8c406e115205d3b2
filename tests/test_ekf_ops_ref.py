"""CPU tests of the extended-precision reference of the EKF's non-visual operations (tests/ekf_ops_ref.py): the Joseph and closed
forms of the augmentation agree, the C oracle lies within the componentwise bound for every operation on fresh, filled and dense
states, the compiled reference's golden snapshots chain within it, the bit-exact operations are bit exact, the comparator rejects
subtly wrong results that the max|dP| / max|P| < 1e-9 gate of the other EKF tests accepts, and the real cluster kernel body (host
emulator) lies within the bound at the scales of a live filter."""
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import ekf_common as C
import ekf_ops_ref as E
import ekf_script
import predict_ref as PR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(C.GOLD)
def _params(trail, ms):
    from oracle import ekf_oracle
    o = ekf_oracle.OracleEKF()
    p = o.default_params()
    o.close()
    return C.params_with(lambda: p, trail, ms)


LAYOUTS = ((5, 2), (6, 0), (20, 0))
STATES = ("fresh", "filled", "dense")


@pytest.mark.parametrize("state", STATES)
@pytest.mark.parametrize("trail,ms", LAYOUTS)
def test_c_oracle_within_bound(oracle_lk, trail, ms, state):
    """The C oracle (fp64, literal Joseph form with dense N^3 products, plain loops) lies within the bound for every operation: the
    augmentation at drop indices -1, 0, 1, trail - 1 and after the symmetrisation of an asymmetric P, every fixed-H update, the
    transform at pose -1, 0, trail - 1, the conditioning (no map) and the normalisation."""
    from oracle import ekf_oracle
    p = _params(trail, ms)
    base = ekf_oracle.OracleEKF(p)
    m, P, time = E.start_state(base, state)
    ops = E.Ops(p)
    worst = []

    def run(name, call, ref):
        o = base.clone()
        o.upload(m, P)
        call(o)
        r = ref()
        gm, gP = o.download()
        o.close()
        rat = r.ratios(gm, gP)
        worst.append((max(rat.values()), name))
        assert max(rat.values()) <= 1.0, (name, rat)

    for drop in sorted({-1, 0, 1, trail - 1}):
        run(f"augment[{drop}]", lambda o, d=drop: o.augment(d), lambda d=drop: ops.augment(m, P, d))
    rng = np.random.RandomState(trail)
    Pa = P * (1 + 1e-9 * np.triu(rng.uniform(-1, 1, P.shape), 1))
    o = base.clone()
    o.upload(m, Pa)
    o.symmetrize()
    o.augment(-1)
    r = ops.augment(m, Pa, -1, sym_first=True)
    rat = r.ratios(*o.download())
    o.close()
    assert max(rat.values()) <= 1.0, ("symmetrize + augment", rat)
    for name, call, ref in E.fixed_h_ops(ops, m, P, time):
        run(name, call, ref)
    base.close()
    print(f"\nN={ops.N} {state}: worst error / bound " + ", ".join(f"{n} {w:.3g}" for w, n in sorted(worst)[-4:]))


@pytest.mark.parametrize("state", STATES)
@pytest.mark.parametrize("trail,ms", ((5, 2), (6, 0)))
def test_joseph_and_closed_forms_agree(oracle_lk, trail, ms, state):
    """The literal Joseph form T1 P+ T1' + K R K' (dense, longdouble) and the cancellation-free closed form agree far inside the bound,
    at every drop index."""
    from oracle import ekf_oracle
    p = _params(trail, ms)
    o = ekf_oracle.OracleEKF(p)
    m, P, _ = E.start_state(o, state)
    o.close()
    ops = E.Ops(p)
    for drop in range(trail):
        a, b = ops.augment(m, P, drop, form="joseph"), ops.augment(m, P, drop)
        assert E.bound_ratio(a.P, b.P, b.BP) < 1e-2 and E.bound_ratio(a.m, b.m, b.Bm) < 1e-2, drop


def test_golden_snapshots_chain_within_bound():
    """The compiled reference's snapshots of tests/ekf_script.run_misc_ops (N = 62): each of ops 1-9 applied by the reference to its
    predecessor reproduces the next snapshot within the bound (translate_to exactly), lock_biases (11) from snapshot 9 exactly and
    condition_on_last_pose (12) from snapshot 11 within the bound."""
    p = _params(6, 0)
    ops = E.Ops(p)
    g = ekf_script.imu_sample(np.random.RandomState(5), 1)[0]
    snap = lambda i: (GOLD[f"n62_misc_m_{i}"], GOLD[f"n62_misc_P_{i}"])
    steps = {1: lambda m, P: ops.zupt(m, P, 1e-2), 2: lambda m, P: ops.zrupt(m, P, g), 3: lambda m, P: ops.pseudo_velocity(m, P, 0.7, 1.0),
             4: lambda m, P: ops.position(m, P, [0.1, -0.2, 0.05], 1e-3), 5: lambda m, P: ops.zero_height(m, P, 1e-3),
             6: lambda m, P: ops.orientation(m, P, E.Q_ORI, 1e-2), 8: lambda m, P: ops.transform_to(m, P, [0.5, -0.5, 0.25], E.Q_XF, -1),
             9: lambda m, P: ops.transform_to(m, P, [0.0, 1.0, 0.0], [1.0, 0.0, 0.0, 0.0], 2)}
    for i in range(1, 10):
        m0, P0 = snap(i - 1)
        m1, P1 = snap(i)
        if i == 7:
            assert np.array_equal(ops.translate_to_fp64(m0, [1.0, 2.0, 3.0]), m1) and np.array_equal(P0, P1)
            continue
        r = steps[i](m0, P0).ratios(m1, P1)
        print(f"\ngolden op {i}: error / bound m {r['m']:.3g} P {r['P']:.3g}")
        assert max(r.values()) <= 1.0, (i, r)
    lm, lP = ops.lock_biases_fp64(*snap(9))
    assert np.array_equal(lm, snap(11)[0]) and np.array_equal(lP, snap(11)[1])
    r = ops.condition_on_last_pose(*snap(11)).ratios(*snap(12))
    assert max(r.values()) <= 1.0, r


@pytest.mark.parametrize("trail,ms", ((5, 2), (6, 0)))
def test_bit_exact_ops_match_c_oracle(oracle_lk, trail, ms):
    """unaugment, lock_biases, insert_map_point (every index), translate_to and symmetrize: the fp64 restatements equal the C oracle
    bit for bit."""
    from oracle import ekf_oracle
    p = _params(trail, ms)
    base = ekf_oracle.OracleEKF(p)
    m, P, _ = E.start_state(base, "filled")
    P = P * (1 + 1e-9 * np.triu(np.random.RandomState(1).uniform(-1, 1, P.shape), 1))
    ops = E.Ops(p)
    cases = [("unaugment", lambda o: o.unaugment(), lambda: ops.unaugment_fp64(m, P)),
             ("lock_biases", lambda o: o.lock_biases(), lambda: ops.lock_biases_fp64(m, P)),
             ("translate_to", lambda o: o.translate_to([1.0, 2.0, 3.0]), lambda: (ops.translate_to_fp64(m, [1.0, 2.0, 3.0]), P)),
             ("symmetrize", lambda o: o.symmetrize(), lambda: (m, E.symmetrize_fp64(P)))]
    cases += [(f"insert_map_point[{k}]", lambda o, k=k: o.insert_map_point(k, [3.0, -2.0, 8.0]),
               lambda k=k: ops.insert_map_point_fp64(m, P, k, [3.0, -2.0, 8.0])) for k in range(ms)]
    for name, call, ref in cases:
        o = base.clone()
        o.upload(m, P)
        call(o)
        gm, gP = o.download()
        o.close()
        rm, rP = ref()
        assert np.array_equal(gm, rm) and np.array_equal(gP, rP), name
    base.close()


def _fault_cases(ops, m, P, time):
    """(fault, correct Result, faulty fp64 (m, P)) for every fault the comparator must reject."""
    f64 = lambda r: (np.asarray(r.m, np.float64), np.asarray(r.P, np.float64))
    good = ops.augment(m, P, 1)
    out = [("plain P - K HP augmentation", good, ops.augment_plain_fp64(m, P, 1))]
    for fault in ("drop_off_by_one", "noise_wrong_slot", "noise_position_only"):
        out.append((fault, good, f64(ops.augment(m, P, 1, form="joseph", fault=fault))))
    Pa = P * (1 + 1e-6 * np.triu(np.random.RandomState(2).uniform(-1, 1, P.shape), 1))
    out.append(("symFirst skipped", ops.augment(m, Pa, 1, sym_first=True),
                f64(ops.augment(m, Pa, 1, sym_first=True, form="joseph", fault="sym_first_skipped"))))
    xf = lambda **k: ops.transform_to(m, P, [0.5, -0.5, 0.25], E.Q_XF, -1, **k)
    out.append(("transposed rotation in transform_to", xf(), f64(xf(fault="transposed_rotation"))))
    out.append(("diagonal-only B^-1", ops.condition_on_last_pose(m, P), f64(ops.condition_on_last_pose(m, P, fault="diag_binv"))))
    out.append(("exp(0.5 t) dropped", ops.zupt_initialization(m, P, time), f64(ops.zupt_initialization(m, P, time, fault="no_exp"))))
    out.append(("3-D speed in pseudo-velocity", ops.pseudo_velocity(m, P, 0.7, 1.0), f64(ops.pseudo_velocity(m, P, 0.7, 1.0, fault="speed_3d"))))
    return out


@pytest.mark.parametrize("state", ("fresh", "filled"))
def test_comparator_rejects_faults(oracle_lk, state):
    """Each fault, applied to an otherwise correct result, exceeds the bound by at least 10x. On the fresh filter (trail 6, max|P| =
    1e8 from the trail priors) the plain-downdate augmentation passes the max|dP| / max|P| < 1e-9 gate of the other EKF tests while
    its new slot is wrong relative to its own scale: the gap the per-entry bound closes."""
    from oracle import ekf_oracle
    p = _params(6, 0)
    o = ekf_oracle.OracleEKF(p)
    m, P, time = E.start_state(o, state)
    o.close()
    m[E.VEL:E.VEL + 3] = [0.3, -0.2, 0.5]            # a moving filter: the vertical speed separates 2-D from 3-D speed
    ops = E.Ops(p)
    for name, good, (bm, bP) in _fault_cases(ops, m, P, time):
        if state == "fresh" and name in ("drop_off_by_one", "diagonal-only B^-1"):
            continue        # a fresh filter's trail slots hold the same diagonal prior: another drop index or a diagonal B^-1 change nothing
        r = max(good.ratios(bm, bP).values())
        rel = ekf_script.rel_err(bP, np.asarray(good.P, np.float64))
        print(f"\n{state} {name}: error / bound {r:.3g}, max|dP| / max|P| {rel:.3g}, scaled {PR.scaled_error(bP, good.P):.3g}")
        assert r >= 10.0, name
        if name.startswith("plain") and state == "fresh":
            assert np.abs(P).max() == 1e8 and rel < C.TOL_P_REL
            assert PR.scaled_error(bP, good.P) > 1e-9          # the new slot, on its own scale, wrong far above fp64 rounding


# ------------------------------------------------------------------------------------------------ the cluster kernel body on the emulator
def _emu_exe(tmp_path):
    exe = str(tmp_path / "emu_update")
    obj = str(tmp_path / "orc_ekf.o")
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-c", os.path.join(ROOT, "oracle", "hv_oracle_ekf.c"), "-o", obj])
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-pthread", "-I" + os.path.join(ROOT, "tests", "emu", "stubs"),
                           "-I" + os.path.join(ROOT, "tests", "emu"), "-I" + os.path.join(ROOT, "hybvio_b200", "csrc"),
                           os.path.join(ROOT, "tests", "emu", "emu_update.cpp"), obj, "-lm", "-o", exe])
    return exe


OP_CODES = {"zupt": 1, "zrupt": 2, "pseudo_velocity": 3, "position": 4, "zero_height": 5, "orientation": 6, "augment": 7}


def emu_run(exe, tmp_path, ops, m, P, op, R, ysmall=(0, 0, 0, 0), speed=0.0, drop=0, sym_first=0, normalize_all=0, symmetrize=0):
    """Runs ek2_body once through the emulator's file mode: header (op, N, trail, mapDim, drop, symFirst, normalizeAll, symmetrize as
    doubles; Rdiag, noiseScale, augNoisePos, augNoiseOri, defaultSpeed, ysmall[4]), then m and P (column-major) in, m and P out."""
    q = ops.augment_noise()
    head = [OP_CODES[op], ops.N, ops.trail, 3 * ops.map_size, drop, sym_first, normalize_all, symmetrize,
            R, ops.ns, q[0], q[3], speed, *ysmall]
    src, dst = tmp_path / "in.bin", tmp_path / "out.bin"
    np.concatenate([np.asarray(head, np.float64), np.asarray(m, np.float64), np.asarray(P, np.float64).ravel(order="F")]).tofile(src)
    out = subprocess.run([exe, "file", str(src), str(dst)], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    res = np.fromfile(dst, np.float64)
    return res[:ops.N], res[ops.N:].reshape((ops.N, ops.N), order="F")


def test_cluster_body_within_bound_on_emulator(oracle_lk, tmp_path):
    """The real cluster kernel body (ekf_cluster2.cuh, host emulator) for the augmentation on a fresh filter (1e8 trail priors: the
    new slot's cancellation), with the deferred symmetrisation, on a filled and a dense state, and for every fixed-H update, against
    the reference's bound."""
    from oracle import ekf_oracle
    exe = _emu_exe(tmp_path)
    p = _params(6, 0)
    ops = E.Ops(p)
    ns = ops.ns
    for state in ("fresh", "filled", "dense"):
        o = ekf_oracle.OracleEKF(p)
        m, P, time = E.start_state(o, state)
        o.close()
        m[E.VEL:E.VEL + 3] = [0.3, -0.2, 0.5]
        R_aug = np.float64(p.augment_r) * ns
        cases = [("augment[-1]", dict(op="augment", R=R_aug, drop=5, normalize_all=1, symmetrize=1), ops.augment(m, P, -1)),
                 ("augment[0]", dict(op="augment", R=R_aug, drop=0, normalize_all=1, symmetrize=1), ops.augment(m, P, 0)),
                 ("zupt", dict(op="zupt", R=np.float64(1e-2) * ns), ops.zupt(m, P, 1e-2)),
                 ("zrupt", dict(op="zrupt", R=np.float64(p.rotation_zupt_r) * ns, ysmall=(0.01, -0.02, 0.2, 0)),
                  ops.zrupt(m, P, [0.01, -0.02, 0.2])),
                 ("pseudo_velocity", dict(op="pseudo_velocity", R=np.float64(1.0) * ns, speed=0.7), ops.pseudo_velocity(m, P, 0.7, 1.0)),
                 ("position", dict(op="position", R=np.float64(1e-3) * ns, ysmall=(0.1, -0.2, 0.05, 0), symmetrize=1),
                  ops.position(m, P, [0.1, -0.2, 0.05], 1e-3)),
                 ("zero_height", dict(op="zero_height", R=np.float64(1e-3) * ns, symmetrize=1), ops.zero_height(m, P, 1e-3)),
                 ("orientation", dict(op="orientation", R=np.float64(1e-2) * ns, ysmall=tuple(E.Q_ORI), normalize_all=1, symmetrize=1),
                  ops.orientation(m, P, E.Q_ORI, 1e-2))]
        Pa = P * (1 + 1e-9 * np.triu(np.random.RandomState(3).uniform(-1, 1, P.shape), 1))
        cases.append(("symmetrize + augment[-1]", dict(op="augment", R=R_aug, drop=5, sym_first=1, normalize_all=1, symmetrize=1, P=Pa),
                      ops.augment(m, Pa, -1, sym_first=True)))
        for name, kw, ref in cases:
            Pin = kw.pop("P", P)
            gm, gP = emu_run(exe, tmp_path, ops, m, Pin, **kw)
            r = ref.ratios(gm, gP)
            w, i, j = ref.worst_entry(gP)
            print(f"\nEMU {state} {name}: error / bound m {r['m']:.3g} P {r['P']:.3g} (worst at {E.block_of(i, 6, 0)} / {E.block_of(j, 6, 0)})")
            assert max(r.values()) <= 1.0, (state, name, r)
