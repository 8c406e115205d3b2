"""CPU tests of the batched frame ingest (hybvio_b200/csrc/ingest.cu): the REAL hv_ingest_batch_kernel compiled for the host thread
emulator (tests/emu) against the frame-ingest oracle (orc_gray / orc_remap, oracle/hv_oracle_gftt.c), bit for bit, in one launch over jobs
of every mode (colour, remap, colour + remap fused), widths below / at / across 256 with every w % 4, padded strides and 1 .. 4 channels;
and the ctypes mirror of hv_ingest_job against the C layout. The GPU tests (test_gpu_ingest_batch.py) remain the authority on the
compiled sm_90a code."""
import ctypes
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = ["-I" + os.path.join(ROOT, "tests", "emu", "stubs"), "-I" + os.path.join(ROOT, "tests", "emu"), "-I" + os.path.join(ROOT, "hybvio_b200", "csrc")]


def test_ingest_batch_kernel_on_host_emulator(tmp_path):
    src = open(os.path.join(ROOT, "hybvio_b200", "csrc", "ingest.cu")).read()
    dev = src[:src.index("\ncudaError_t hv_launch_gray")]        # the device code: everything ahead of the launch helpers
    assert "hv_ingest_batch_kernel" in dev
    (tmp_path / "ingest_device.inc").write_text(dev + "\n")
    obj, exe = str(tmp_path / "orc.o"), str(tmp_path / "emu_ingest_batch")
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-c", os.path.join(ROOT, "oracle", "hv_oracle_gftt.c"), "-o", obj])
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-ffp-contract=off", "-pthread", "-w", "-I" + str(tmp_path)] + EMU +
                          [os.path.join(ROOT, "tests", "emu", "emu_ingest_batch.cpp"), obj, "-lm", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.count("  ok") == 64 and "FAIL" not in out.stdout and "all ok" in out.stdout, out.stdout
    for mode in ("colour,", "remap,", "colour + remap,"):
        assert out.stdout.count(mode) >= 4, mode


def test_ctypes_ingest_job_matches_the_header(tmp_path):
    import sys
    sys.path.insert(0, ROOT)
    from hybvio_b200 import capi
    py = capi.IngestJob
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "hybvio_b200.h"', 'int main(void) {',
             'printf("max %d\\n", HV_INGEST_BATCH_MAX);', 'printf("size %zu\\n", sizeof(hv_ingest_job));']
    lines += [f'printf("{f} %zu\\n", offsetof(hv_ingest_job, {f}));' for f, _ in py._fields_]
    lines.append("return 0; }")
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines))
    subprocess.check_call(["gcc", "-std=c99", "-I" + os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = dict(ln.split() for ln in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["max"]) == capi.INGEST_BATCH_MAX
    assert int(got["size"]) == ctypes.sizeof(py)
    for f, _ in py._fields_:
        assert int(got[f]) == getattr(py, f).offset, f
