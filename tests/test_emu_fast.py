"""CPU test: the REAL FAST kernels (hybvio_b200/csrc/fast.cu: the per-frame mark + scatter kernels and their batch forms) compiled for
the host thread emulator (tests/emu) and compared bit for bit with the cv::FAST oracle (oracle/hv_oracle_fast.c) -- count, order, (x, y),
response and padding -- over images of different sizes and pitches, images smaller than 7 x 7, thresholds 0 / 10 / 20 / 300 with and
without suppression, and capacities above, below and at 0 of the count; plus the ctypes mirror of hv_fast_job against the C layout.
The GPU tests (test_gpu_fast.py) remain the authority on the compiled sm_90a code."""
import ctypes
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = ["-I" + os.path.join(ROOT, "tests", "emu", "stubs"), "-I" + os.path.join(ROOT, "tests", "emu"), "-I" + os.path.join(ROOT, "hybvio_b200", "csrc")]
NJOBS, RUNS = 9, 4


def test_fast_kernels_on_host_emulator(tmp_path):
    src = open(os.path.join(ROOT, "hybvio_b200", "csrc", "fast.cu")).read()
    (tmp_path / "fast_device.inc").write_text(src[:src.index("\ncudaError_t hv_launch_fast")] + "\n")
    obj, exe = str(tmp_path / "orc_fast.o"), str(tmp_path / "emu_fast")
    subprocess.check_call(["gcc", "-O2", "-c", os.path.join(ROOT, "oracle", "hv_oracle_fast.c"), "-o", obj])
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-pthread", "-w", "-I" + str(tmp_path)] + EMU +
                          [os.path.join(ROOT, "tests", "emu", "emu_fast.cpp"), obj, "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.count("  ok") == 2 * NJOBS * RUNS and "FAIL" not in out.stdout and "all ok" in out.stdout, out.stdout


def test_ctypes_fast_job_matches_the_header(tmp_path):
    import sys
    sys.path.insert(0, ROOT)
    from hybvio_b200 import capi
    py = capi.FastJob
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "hybvio_b200.h"', 'int main(void) {',
             'printf("size %zu\\n", sizeof(hv_fast_job));']
    lines += [f'printf("{f} %zu\\n", offsetof(hv_fast_job, {f}));' for f, _ in py._fields_]
    lines.append("return 0; }")
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines))
    subprocess.check_call(["gcc", "-std=c99", "-I" + os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = dict(ln.split() for ln in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["size"]) == ctypes.sizeof(py)
    for f, _ in py._fields_:
        assert int(got[f]) == getattr(py, f).offset, f
