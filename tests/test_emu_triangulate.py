"""CPU test: the REAL triangulation kernel (hybvio_b200/csrc/triangulate.cu) compiled for the host thread emulator (tests/emu) and
compared bit for bit with the oracle (oracle/hv_oracle_triangulate.c) -- X4, xyz and used -- per call and as one batch of mixed jobs
(every scene of tests/triangulate_common.py, n = 0 and 1, both / one / no status, used aliasing either status, each output alone). The
GPU tests (test_gpu_triangulate.py) remain the authority on the compiled sm_90a code."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import triangulate_common as tc  # noqa: E402

EMU = ["-I" + os.path.join(ROOT, "tests", "emu", "stubs"), "-I" + os.path.join(ROOT, "tests", "emu"), "-I" + os.path.join(ROOT, "hybvio_b200", "csrc")]


@pytest.fixture(scope="module")
def emu_exe(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("emu_triangulate")
    src = open(os.path.join(ROOT, "hybvio_b200", "csrc", "triangulate.cu")).read()
    (tmp / "triangulate_device.inc").write_text(src[:src.index("\ncudaError_t hv_launch_triangulate")] + "\n")
    obj, exe = str(tmp / "orc_triangulate.o"), str(tmp / "emu_triangulate")
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-c", os.path.join(ROOT, "oracle", "hv_oracle_triangulate.c"), "-o", obj])
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-ffp-contract=off", "-pthread", "-w", "-I" + str(tmp)] + EMU +
                          [os.path.join(ROOT, "tests", "emu", "emu_triangulate.cpp"), obj, "-o", exe, "-lm"])
    return exe, tmp


def _write_jobs(path, jobs):
    with open(path, "wb") as f:
        f.write(np.int32(len(jobs)).tobytes())
        for P1, P2, a, b, s1, s2, alias, outs in jobs:
            n = a.shape[0]
            f.write(np.array([n, s1 is not None, s2 is not None, alias] + list(outs), np.int32).tobytes())
            f.write(np.ascontiguousarray(P1, np.float64).tobytes() + np.ascontiguousarray(P2, np.float64).tobytes())
            f.write(np.ascontiguousarray(a, np.float32).tobytes() + np.ascontiguousarray(b, np.float32).tobytes())
            for s in (s1, s2):
                if s is not None:
                    f.write(np.ascontiguousarray(s, np.uint8).tobytes())


def triangulate_jobs():
    """(P1, P2, xy1, xy2, status, status2, alias, (X4, xyz, used wanted)) over every scene, with statuses, aliasing and outputs varied"""
    rng = np.random.default_rng(31)
    jobs = []
    for j, (name, fam, P1, P2, a, b) in enumerate(tc.scenes()):
        n = min(a.shape[0], 130 + 37 * j)
        a, b = a[:n], b[:n]
        s1 = (rng.random(n) > 0.2).astype(np.uint8) * rng.integers(1, 256, n).astype(np.uint8) if j % 3 != 2 else None
        s2 = (rng.random(n) > 0.1).astype(np.uint8) if j % 2 else None
        alias = 1 if (j % 5 == 1 and s1 is not None) else (2 if (j % 5 == 3 and s2 is not None) else 0)
        outs = [(1, 1, 1), (1, 0, 1), (0, 1, 0), (1, 1, 0)][j % 4]
        jobs.append((P1, P2, a, b, s1, s2, alias, outs))
    P1, P2, a, b = tc.rectified(7, 1)
    jobs.append((P1, P2, a, b, None, None, 0, (1, 1, 1)))                                              # n = 1
    jobs.append((P1, P2, a[:0], b[:0], None, None, 0, (0, 0, 0)))                                      # n = 0, no outputs
    P1, P2, a, b = tc.rectified(8, 300)
    cap = 384
    jobs.append((P1, P2, tc.padded(a, cap), tc.padded(b, cap), np.r_[np.ones(300), np.zeros(cap - 300)].astype(np.uint8), None, 1,
                 (1, 1, 1)))                                                                            # padded capacity
    return jobs


def test_triangulate_kernel_on_host_emulator(emu_exe):
    exe, tmp = emu_exe
    jobs = triangulate_jobs()
    path = str(tmp / "jobs.bin")
    _write_jobs(path, jobs)
    out = subprocess.run([exe, path], capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.count("  ok") == 2 * len(jobs) and "FAIL" not in out.stdout and "all ok" in out.stdout, out.stdout
