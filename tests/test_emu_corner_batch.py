"""CPU tests of the batched new-corner step (hybvio_b200/csrc/gftt_select.cu, subpix.cu): the REAL batch kernels compiled for the host
thread emulator (tests/emu) against the oracles, bit for bit --
  * hv_gftt_select_batch_kernel: every crafted list of gftt_select_common as one job of ONE launch (different nkp, sort widths, radii,
    max_tracks and spare capacity) against orc_gftt_corners (oracle/hv_oracle_gftt.c);
  * hv_subpix_batch_kernel: the flattened (job, point) grid over images of different sizes and pitches, empty jobs included, against
    orc_subpix_refine (oracle/hv_oracle_subpix.c);
and the ctypes mirrors of hv_corner_job / hv_subpix_job against the C layout. The GPU tests (test_gpu_corner_batch.py) remain the
authority on the compiled sm_90a code."""
import ctypes
import os
import subprocess

import gftt_select_common as gc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = ["-I" + os.path.join(ROOT, "tests", "emu", "stubs"), "-I" + os.path.join(ROOT, "tests", "emu"), "-I" + os.path.join(ROOT, "hybvio_b200", "csrc")]


def _cut(name, end, decl, tmp_path, inc):
    src = open(os.path.join(ROOT, "hybvio_b200", "csrc", name)).read()
    dev = src[:src.index(end)]
    assert decl in dev
    (tmp_path / inc).write_text(dev.replace(decl, f"unsigned char* {decl.split()[-1][:-3]} = emu_dynamic_smem;") + "\n")


def _build(tmp_path, cpp, oracle_c):
    obj, exe = str(tmp_path / "orc.o"), str(tmp_path / cpp[:-4])
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-c", os.path.join(ROOT, "oracle", oracle_c), "-o", obj])
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-ffp-contract=off", "-pthread", "-w", "-I" + str(tmp_path)] + EMU +
                          [os.path.join(ROOT, "tests", "emu", cpp), obj, "-lm", "-o", exe])
    return exe


def test_select_batch_kernel_on_host_emulator(tmp_path):
    _cut("gftt_select.cu", '\n#include "hv_device_once.cuh"', "extern __shared__ __align__(16) unsigned char select_smem[];", tmp_path,
         "gftt_select_device.inc")
    cases = gc.crafted_cases()
    assert 8 <= len(cases) <= 64
    gc.write_cases(str(tmp_path / "cases.bin"), cases)
    exe = _build(tmp_path, "emu_gftt_select_batch.cpp", "hv_oracle_gftt.c")
    out = subprocess.run([exe, str(tmp_path / "cases.bin")], capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.count("  ok") == len(cases) and "FAIL" not in out.stdout and "all ok" in out.stdout, out.stdout


def test_subpix_batch_kernel_on_host_emulator(tmp_path):
    _cut("subpix.cu", "\ncudaError_t hv_launch_subpix", "extern __shared__ __align__(16) unsigned char subpix_smem[];", tmp_path,
         "subpix_device.inc")
    exe = _build(tmp_path, "emu_subpix_batch.cpp", "hv_oracle_subpix.c")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.count("  ok") == 16 and "FAIL" not in out.stdout and "all ok" in out.stdout, out.stdout


def test_ctypes_job_structs_match_the_header(tmp_path):
    import sys
    sys.path.insert(0, ROOT)
    from hybvio_b200 import capi
    pairs = {"hv_corner_job": capi.CornerJob, "hv_subpix_job": capi.SubpixJob}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "hybvio_b200.h"', 'int main(void) {',
             'printf("max %d\\n", HV_CORNER_BATCH_MAX);']
    for cname, py in pairs.items():
        lines.append(f'printf("{cname} size %zu\\n", sizeof({cname}));')
        lines += [f'printf("{cname} {f} %zu\\n", offsetof({cname}, {f}));' for f, _ in py._fields_]
    lines.append("return 0; }")
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines))
    subprocess.check_call(["gcc", "-std=c99", "-I" + os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = {}
    for ln in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines():
        k = ln.split()
        got[tuple(k[:-1])] = int(k[-1])
    assert got[("max",)] == capi.CORNER_BATCH_MAX
    for cname, py in pairs.items():
        assert got[(cname, "size")] == ctypes.sizeof(py), cname
        for f, _ in py._fields_:
            assert got[(cname, f)] == getattr(py, f).offset, (cname, f)

