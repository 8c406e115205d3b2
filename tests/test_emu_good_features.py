"""CPU test: the REAL Shi-Tomasi kernels (hybvio_b200/csrc/good_features.cu: the per-frame response, candidate and select kernels and
their batch forms) compiled for the host thread emulator (tests/emu) and compared bit for bit with the cv::goodFeaturesToTrack oracle
(oracle/hv_oracle_good_features.c) -- response map, count, order, (x, y), response and padding -- over noise, a periodic pattern, a ramp
and a flat image, three masks, min_distance 0 to 30 and max_corners 1 to above the candidate count. The select is built with 256-key
rounds, so that its radix select runs several rounds on these small images. Plus the ctypes mirror of hv_good_features_job against the
C layout. The GPU tests (test_gpu_good_features.py) remain the authority on the compiled sm_90a code."""
import ctypes
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = ["-I" + os.path.join(ROOT, "tests", "emu", "stubs"), "-I" + os.path.join(ROOT, "tests", "emu"), "-I" + os.path.join(ROOT, "hybvio_b200", "csrc")]


def test_good_features_kernels_on_host_emulator(tmp_path):
    src = open(os.path.join(ROOT, "hybvio_b200", "csrc", "good_features.cu")).read()
    dev = src[:src.index('\n#include "hv_device_once.cuh"')]
    decl = "extern __shared__ __align__(16) unsigned char gf_smem[];"
    assert decl in dev
    (tmp_path / "good_features_device.inc").write_text(dev.replace(decl, "unsigned char* gf_smem = emu_dynamic_smem;") + "\n")
    obj, exe = str(tmp_path / "orc_gf.o"), str(tmp_path / "emu_good_features")
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-c", os.path.join(ROOT, "oracle", "hv_oracle_good_features.c"), "-o", obj])
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-ffp-contract=off", "-pthread", "-w", "-DHV_GF_CHUNK=256", "-I" + str(tmp_path)] + EMU +
                          [os.path.join(ROOT, "tests", "emu", "emu_good_features.cpp"), obj, "-o", exe, "-lm"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0, out.stdout + out.stderr
    ncases = len(re.findall(r"^frame ", out.stdout, re.M))
    assert ncases >= 10 and out.stdout.count("  ok") == 2 * ncases and "FAIL" not in out.stdout and "all ok" in out.stdout, out.stdout
    rounds = int(re.search(r"more candidates than one round holds: (\d+)", out.stdout).group(1))
    assert rounds >= 2, out.stdout


def test_ctypes_good_features_job_matches_the_header(tmp_path):
    import sys
    sys.path.insert(0, ROOT)
    from hybvio_b200 import capi
    py = capi.GoodFeaturesJob
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "hybvio_b200.h"', 'int main(void) {',
             'printf("size %zu\\n", sizeof(hv_good_features_job));']
    lines += [f'printf("{f} %zu\\n", offsetof(hv_good_features_job, {f}));' for f, _ in py._fields_]
    lines.append("return 0; }")
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines))
    subprocess.check_call(["gcc", "-std=c99", "-I" + os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = dict(ln.split() for ln in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["size"]) == ctypes.sizeof(py)
    for f, _ in py._fields_:
        assert int(got[f]) == getattr(py, f).offset, f
