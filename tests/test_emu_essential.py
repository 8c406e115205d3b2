"""CPU test: the REAL essential-matrix RANSAC kernel (hybvio_b200/csrc/essential.cu) compiled for the host thread emulator (tests/emu)
and compared bit for bit with the oracle (oracle/hv_oracle_essential.c) -- E, nsol, mask and inliers -- per call and as one batch, on
scenes with m = 0, 4, 5, 6, 20, 150 and 300 used points, with and without a status, at different intrinsics and two parameter sets;
plus the ctypes mirror of hv_essential_job against the C layout. The GPU tests (test_gpu_essential.py) remain the authority on the
compiled sm_90a code."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import essential_common as ec  # noqa: E402

EMU = ["-I" + os.path.join(ROOT, "tests", "emu", "stubs"), "-I" + os.path.join(ROOT, "tests", "emu"), "-I" + os.path.join(ROOT, "hybvio_b200", "csrc")]


@pytest.fixture(scope="module")
def emu_exe(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("emu_essential")
    src = open(os.path.join(ROOT, "hybvio_b200", "csrc", "essential.cu")).read()
    dev = src[:src.index("\ncudaError_t hv_launch_essential")]
    decl = "extern __shared__ __align__(16) unsigned char ess_smem[];"
    assert decl in dev
    (tmp / "essential_device.inc").write_text(dev.replace(decl, "unsigned char* ess_smem = emu_dynamic_smem;") + "\n")
    obj, exe = str(tmp / "orc_essential.o"), str(tmp / "emu_essential")
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-c", os.path.join(ROOT, "oracle", "hv_oracle_essential.c"), "-o", obj])
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-ffp-contract=off", "-pthread", "-w", "-I" + str(tmp)] + EMU +
                          [os.path.join(ROOT, "tests", "emu", "emu_essential.cpp"), obj, "-o", exe])
    return exe, tmp


def _write_jobs(path, jobs, prob, thr, mi):
    with open(path, "wb") as f:
        f.write(np.int32(len(jobs)).tobytes())
        for p1, p2, st, k in jobs:
            f.write(np.int32(p1.shape[0]).tobytes() + np.array(k, np.float64).tobytes() + np.int32(st is not None).tobytes())
            f.write(np.ascontiguousarray(p1, np.float32).tobytes() + np.ascontiguousarray(p2, np.float32).tobytes())
            if st is not None:
                f.write(np.ascontiguousarray(st, np.uint8).tobytes())
        f.write(np.float64(prob).tobytes() + np.float64(thr).tobytes() + np.int32(mi).tobytes())


@pytest.mark.parametrize("params", [(0.999, 1.0, 1000), (0.99, 2.0, 3)])
def test_essential_kernel_on_host_emulator(emu_exe, params):
    exe, tmp = emu_exe
    rng = np.random.default_rng(17)
    jobs = []
    for j, (m, outl) in enumerate(((0, 0.0), (4, 0.0), (5, 0.0), (6, 0.0), (20, 0.2), (150, 0.3), (300, 0.5))):
        p1, p2 = ec.scene(rng, m, outl, 0.5, "side" if j % 2 else "forward")
        st = None if j % 3 else (rng.random(m) > 0.2).astype(np.uint8) * 5
        k = (ec.FX * (1 + 0.02 * j), ec.FY, ec.CX + j, ec.CY)
        jobs.append((p1, p2, st, k))
    path = str(tmp / f"jobs_{params[2]}.bin")
    _write_jobs(path, jobs, *params)
    out = subprocess.run([exe, path], capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.count("  ok") == 2 * len(jobs) and "FAIL" not in out.stdout and "all ok" in out.stdout, out.stdout


def test_ctypes_essential_job_matches_the_header(tmp_path):
    sys.path.insert(0, ROOT)
    from hybvio_b200 import capi
    py = capi.EssentialJob
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "hybvio_b200.h"', 'int main(void) {',
             'printf("size %zu\\n", sizeof(hv_essential_job));']
    lines += [f'printf("{f} %zu\\n", offsetof(hv_essential_job, {f}));' for f, _ in py._fields_]
    lines.append("return 0; }")
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines))
    subprocess.check_call(["gcc", "-std=c99", "-I" + os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = dict(ln.split() for ln in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["size"]) == ctypes.sizeof(py)
    for f, _ in py._fields_:
        assert int(got[f]) == getattr(py, f).offset, f
