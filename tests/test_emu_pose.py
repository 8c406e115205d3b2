"""CPU test: the REAL relative-pose kernel (hybvio_b200/csrc/pose.cu) compiled for the host thread emulator (tests/emu) and compared bit
for bit with the oracle (oracle/hv_oracle_pose.c) -- R, t, mask and good -- per call and as one batch, at m = 0, 4, 5, 6, 150 and 4096
points, with and without an input mask, in place, at nsol NULL / 0 / 1 / above 1, for three distance thresholds; plus the ctypes mirror
of hv_pose_job against the C layout. The GPU tests (test_gpu_pose.py) remain the authority on the compiled sm_90a code."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
import essential_common as ec  # noqa: E402

EMU = ["-I" + os.path.join(ROOT, "tests", "emu", "stubs"), "-I" + os.path.join(ROOT, "tests", "emu"), "-I" + os.path.join(ROOT, "hybvio_b200", "csrc")]


@pytest.fixture(scope="module")
def emu_exe(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("emu_pose")
    src = open(os.path.join(ROOT, "hybvio_b200", "csrc", "pose.cu")).read()
    (tmp / "pose_device.inc").write_text(src[:src.index("\ncudaError_t hv_launch_pose")] + "\n")
    obj, exe = str(tmp / "orc_pose.o"), str(tmp / "emu_pose")
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-c", os.path.join(ROOT, "oracle", "hv_oracle_pose.c"), "-o", obj])
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-ffp-contract=off", "-pthread", "-w", "-I" + str(tmp)] + EMU +
                          [os.path.join(ROOT, "tests", "emu", "emu_pose.cpp"), obj, "-o", exe, "-lm"])
    return exe, tmp


def _write_jobs(path, jobs, dist):
    with open(path, "wb") as f:
        f.write(np.int32(len(jobs)).tobytes())
        for Ecm, nsol, p1, p2, mask, in_place, k in jobs:
            f.write(np.int32(p1.shape[0]).tobytes() + np.array(k, np.float64).tobytes())
            f.write(np.array([nsol, mask is not None, in_place], np.int32).tobytes() + np.ascontiguousarray(Ecm, np.float64).ravel()[:9].tobytes())
            f.write(np.ascontiguousarray(p1, np.float32).tobytes() + np.ascontiguousarray(p2, np.float32).tobytes())
            if mask is not None:
                f.write(np.ascontiguousarray(mask, np.uint8).tobytes())
        f.write(np.float64(dist).tobytes())


def pose_jobs():
    """(E column-major, nsol (-1: NULL), p1, p2, mask or None, in place, intrinsics) over m = 0, 4, 5, 6, 150, 4096, E from the essential
    oracle where it finds one; plus E = 0 and a rank-1 E."""
    from oracle.essential_oracle import OracleEssential
    oe = OracleEssential()
    rng = np.random.default_rng(23)
    jobs = []
    for j, (m, outl) in enumerate(((0, 0.0), (4, 0.0), (5, 0.0), (6, 0.0), (150, 0.3), (4096, 0.2), (150, 0.0), (5, 0.0))):
        p1, p2 = ec.scene(rng, m, outl, 0.5, "side" if j % 2 else "forward")
        k = (ec.FX * (1 + 0.02 * j), ec.FY, ec.CX + j, ec.CY)
        if m >= 5:
            E, nsol, mask, _ = oe.find_essential(p1, p2, *k)
        else:
            E, nsol, mask = np.eye(3)[None] * np.array([1.0, 1.0, 0.0]), 1, np.ones(m, np.uint8)
        Ecm = E.reshape(-1)[:9]
        mask = mask * rng.integers(1, 256, m).astype(np.uint8) if j % 3 == 1 else mask
        jobs.append((Ecm, [-1, nsol][j % 2], p1, p2, [mask, None][j % 2 if j != 4 else 0], j == 4, k))
    p1, p2 = ec.scene(rng, 150, 0.1, 0.5)
    jobs.append((jobs[4][0], 0, p1, p2, None, False, jobs[4][6]))                        # nsol 0
    jobs.append((np.zeros(9), -1, p1, p2, None, False, jobs[4][6]))                      # E = 0
    u, v = np.array([0.3, -0.5, 0.8]), np.array([0.6, 0.64, 0.48])
    jobs.append((np.outer(u, v).T.ravel(), -1, p1, p2, None, False, jobs[4][6]))         # rank 1
    jobs.append((jobs[4][0], -1, p1, p2, np.ones(150, np.uint8), True, jobs[4][6]))      # in place, every point used
    return jobs


@pytest.mark.parametrize("dist", [50.0, 5.0, 1e9])
def test_pose_kernel_on_host_emulator(emu_exe, dist):
    exe, tmp = emu_exe
    jobs = pose_jobs()
    path = str(tmp / f"jobs_{dist:g}.bin")
    _write_jobs(path, jobs, dist)
    out = subprocess.run([exe, path], capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.count("  ok") == 2 * len(jobs) and "FAIL" not in out.stdout and "all ok" in out.stdout, out.stdout


def test_ctypes_pose_job_matches_the_header(tmp_path):
    from hybvio_b200 import capi
    py = capi.PoseJob
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "hybvio_b200.h"', 'int main(void) {',
             'printf("size %zu\\n", sizeof(hv_pose_job));']
    lines += [f'printf("{f} %zu\\n", offsetof(hv_pose_job, {f}));' for f, _ in py._fields_]
    lines.append("return 0; }")
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines))
    subprocess.check_call(["gcc", "-std=c99", "-I" + os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = dict(ln.split() for ln in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["size"]) == ctypes.sizeof(py)
    for f, _ in py._fields_:
        assert int(got[f]) == getattr(py, f).offset, f
