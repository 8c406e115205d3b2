"""CPU test: the REAL absolute-pose RANSAC kernel (hybvio_b200/csrc/pnp.cu) compiled for the host thread emulator (tests/emu) and
compared bit for bit with the oracle (oracle/hv_oracle_pnp.c) -- rvec, tvec, mask, inliers and ok -- per call and as one batch, on scenes
with m = 0, 3, 4, 5, 150 and 4096 used points, with and without a status, at different intrinsics and two parameter sets; plus the
ctypes mirror of hv_pnp_job against the C layout. The GPU tests (test_gpu_pnp.py) remain the authority on the compiled sm_90a code."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import pnp_common as pc  # noqa: E402

EMU = ["-I" + os.path.join(ROOT, "tests", "emu", "stubs"), "-I" + os.path.join(ROOT, "tests", "emu"), "-I" + os.path.join(ROOT, "hybvio_b200", "csrc")]


@pytest.fixture(scope="module")
def emu_exe(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("emu_pnp")
    src = open(os.path.join(ROOT, "hybvio_b200", "csrc", "pnp.cu")).read()
    dev = src[:src.index("\ncudaError_t hv_launch_pnp")]
    decl = "extern __shared__ __align__(16) unsigned char pnp_smem[];"
    assert decl in dev
    (tmp / "pnp_device.inc").write_text(dev.replace(decl, "unsigned char* pnp_smem = emu_dynamic_smem;") + "\n")
    obj, exe = str(tmp / "orc_pnp.o"), str(tmp / "emu_pnp")
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-c", os.path.join(ROOT, "oracle", "hv_oracle_pnp.c"), "-o", obj])
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-ffp-contract=off", "-pthread", "-w", "-I" + str(tmp)] + EMU +
                          [os.path.join(ROOT, "tests", "emu", "emu_pnp.cpp"), obj, "-o", exe, "-lm"])
    return exe, tmp


def write_jobs(path, jobs, iterations, reproj, conf):
    with open(path, "wb") as f:
        f.write(np.int32(len(jobs)).tobytes())
        for X, x, st, k in jobs:
            f.write(np.int32(X.shape[0]).tobytes() + np.array(k, np.float64).tobytes() + np.int32(st is not None).tobytes())
            f.write(np.ascontiguousarray(X, np.float32).tobytes() + np.ascontiguousarray(x, np.float32).tobytes())
            if st is not None:
                f.write(np.ascontiguousarray(st, np.uint8).tobytes())
        f.write(np.int32(iterations).tobytes() + np.float32(reproj).tobytes() + np.float64(conf).tobytes())


@pytest.mark.parametrize("params", [(100, 8.0, 0.99), (3, 2.0, 0.999)])
def test_pnp_kernel_on_host_emulator(emu_exe, params):
    exe, tmp = emu_exe
    rng = np.random.default_rng(29)
    jobs = []
    for j, (m, outl) in enumerate(((0, 0.0), (3, 0.0), (4, 0.0), (5, 0.0), (150, 0.3), (4096, 0.5))):
        X, x, _, _ = pc.scene(rng, m, outl, 0.5, pc.MOTIONS[j % 3], pc.DEPTHS[j % 2])
        st = None if j % 2 else (rng.random(m) > 0.1).astype(np.uint8) * 3
        if st is not None and m <= 5:
            st[:] = 1
        k = (pc.FX * (1 + 0.02 * j), pc.FY, pc.CX + j, pc.CY)
        jobs.append((X, x, st, k))
    path = str(tmp / f"jobs_{params[0]}.bin")
    write_jobs(path, jobs, *params)
    out = subprocess.run([exe, path], capture_output=True, text=True, timeout=3000)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.count("  ok") == 2 * len(jobs) and "FAIL" not in out.stdout and "all ok" in out.stdout, out.stdout
    assert "ok 1/1" in out.stdout


def test_ctypes_pnp_job_matches_the_header(tmp_path):
    sys.path.insert(0, ROOT)
    from hybvio_b200 import capi
    py = capi.PnpJob
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "hybvio_b200.h"', 'int main(void) {',
             'printf("size %zu\\n", sizeof(hv_pnp_job));']
    lines += [f'printf("{f} %zu\\n", offsetof(hv_pnp_job, {f}));' for f, _ in py._fields_]
    lines.append("return 0; }")
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines))
    subprocess.check_call(["gcc", "-std=c99", "-I" + os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = dict(ln.split() for ln in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["size"]) == ctypes.sizeof(py)
    for f, _ in py._fields_:
        assert int(got[f]) == getattr(py, f).offset, f
