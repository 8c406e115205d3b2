"""GPU: the compiled five-point solver through hv_find_essential at m == 5 (where the call returns every solution) against the
extended-precision reference (tests/essential_ref.py), with the gates of tests/test_essential_ref.py (count on fp64-determined sets,
each E within its bound; not the true E, which rounding q to float32 moves by about kappa 6e-8, and which the CPU test checks on
the exact doubles): 1 000 sets of the cv2 comparison's generator (pixel points, EuRoC-like K),
250 noise-free sets per family (normalised points rounded to float32 and passed with identity intrinsics, so that the solver sees
exactly the q the reference gets), and the named regressions (noise-free ones rounded to float32 as above)."""
import ctypes
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import essential_common as ec  # noqa: E402
from test_essential_ref import judge, references  # noqa: E402

pytestmark = pytest.mark.gpu
GENERATOR_SETS = 1000
FAMILY_SETS = 250


def _device(hv, p1, p2, k):
    """every solution (nsol, 3, 3) row-major of the device's m == 5 call"""
    from hybvio_b200.capi import _ptr, check
    p1, p2 = np.ascontiguousarray(p1, np.float32), np.ascontiguousarray(p2, np.float32)
    E = np.full(90, np.nan)
    mask = np.zeros(5, np.uint8)
    nsol, inl = ctypes.c_int(-1), ctypes.c_int(-1)
    check(hv.lib.hv_find_essential(hv.h, _ptr(p1), _ptr(p2), None, 5, *k, 0.999, 1.0, 1000, _ptr(E), ctypes.byref(nsol), _ptr(mask),
                                   ctypes.byref(inl)), "hv_find_essential")
    return np.ascontiguousarray(E.reshape(10, 3, 3)[:nsol.value].transpose(0, 2, 1))


def _sets():
    """(label, p1, p2, intrinsics, q the solver receives, true E or None)"""
    out = []
    rng = np.random.default_rng(2024)
    for k in range(GENERATOR_SETS):
        p1, p2 = ec.scene(rng, 5, 0.0, 0.5, "side" if k % 2 else "forward", rot=0.1)
        out.append((f"generator {k}", p1, p2, (ec.FX, ec.FY, ec.CX, ec.CY), ec.normalise(p1, p2), None))
    unit = (1.0, 1.0, 0.0, 0.0)
    for family in sorted(ec.FAMILIES):
        for i, (q, E) in enumerate(ec.noise_free_sets(family, 100, FAMILY_SETS)):
            q = q.astype(np.float32).astype(np.float64)
            out.append((f"{family} {i}", q[:, :2], q[:, 2:], unit, q, None))
    for name, (family, seed, k, _) in sorted(ec.REGRESSIONS.items()):
        if family == "generator":
            rng = np.random.default_rng(seed)
            for j in range(k + 1):
                p1, p2 = ec.scene(rng, 5, 0.0, 0.5, "side" if j % 2 else "forward", rot=0.1)
            out.append((name, p1, p2, (ec.FX, ec.FY, ec.CX, ec.CY), ec.normalise(p1, p2), None))
        else:
            # the exact doubles cannot pass through float32 points: the float32-rounded set is the one the call can receive
            q, _ = ec.regression_set(name, as_float32=True)
            out.append((f"{name} (float32)", q[:, :2], q[:, 2:], unit, q, None))
    return out


def test_device_solutions_match_the_reference(hv):
    sets = _sets()
    for label, p1, p2, k, q, _ in sets:
        assert np.array_equal(ec.normalise(p1, p2, *k), q), label
    refs = references([s[4] for s in sets])
    bad = {}
    for (label, p1, p2, k, q, E), ref in zip(sets, refs):
        f = [x for x in judge(q, ref, _device(hv, p1, p2, k), E) if x != "exempt"]
        if f:
            bad[label] = f
    print(f"device against the reference: {len(sets)} sets, failing {len(bad)}")
    assert not bad, dict(list(bad.items())[:10])
