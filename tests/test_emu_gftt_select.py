"""CPU tests of the corner selection (hybvio_b200/csrc/gftt_select.cu):
  * the REAL body of hv_gftt_select_kernel compiled for the host thread emulator (tests/emu) against orc_gftt_corners
    (oracle/hv_oracle_gftt.c) on the crafted lists of gftt_select_common: list, count and padding bit for bit;
  * the numpy restatement of the selection equals the oracle on the same lists, and each injected fault (unstable sort, `<=` for `<`,
    a fused multiply-add in the distance, the quirk dropped, the cap applied without a radius) changes the result on them -- so these
    inputs can tell those mistakes apart. The GPU tests (test_gpu_gftt_select.py) remain the authority on the compiled sm_90a code."""
import os
import subprocess

import numpy as np
import pytest

import gftt_select_common as gc
from oracle import gftt_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def orc(oracle_lk):
    return gftt_oracle.OracleGftt()


def test_select_kernel_body_on_host_emulator(tmp_path, oracle_lk):
    src = open(os.path.join(ROOT, "hybvio_b200", "csrc", "gftt_select.cu")).read()
    dev = src[:src.index('\n#include "hv_device_once.cuh"')]
    decl = "extern __shared__ __align__(16) unsigned char select_smem[];"
    assert decl in dev
    (tmp_path / "gftt_select_device.inc").write_text(dev.replace(decl, "unsigned char* select_smem = emu_dynamic_smem;") + "\n")
    cases = gc.crafted_cases()
    gc.write_cases(str(tmp_path / "cases.bin"), cases)
    exe = str(tmp_path / "emu_gftt_select")
    obj = str(tmp_path / "orc_gftt.o")
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-c", os.path.join(ROOT, "oracle", "hv_oracle_gftt.c"), "-o", obj])
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-ffp-contract=off", "-pthread", "-w", "-I" + str(tmp_path),
                           "-I" + os.path.join(ROOT, "tests", "emu", "stubs"), "-I" + os.path.join(ROOT, "tests", "emu"),
                           "-I" + os.path.join(ROOT, "hybvio_b200", "csrc"), os.path.join(ROOT, "tests", "emu", "emu_gftt_select.cpp"), obj,
                           "-lm", "-o", exe])
    out = subprocess.run([exe, str(tmp_path / "cases.bin")], capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.count("  ok") == len(cases) and "FAIL" not in out.stdout and "all ok" in out.stdout, out.stdout


def test_restatement_matches_the_oracle(orc):
    for name, kp, prev, r, m in gc.crafted_cases():
        want = orc.corners(kp, prev, r, m)
        got = gc.select(kp, prev, r, m)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), name


@pytest.mark.parametrize("fault", gc.FAULTS)
def test_each_fault_changes_the_list_on_these_inputs(orc, fault):
    changed = []
    for name, kp, prev, r, m in gc.crafted_cases():
        want = orc.corners(kp, prev, r, m)
        got = gc.select(kp, prev, r, m, fault)
        if got.shape != want.shape or not np.array_equal(got.view(np.uint32), want.view(np.uint32)):
            changed.append(name)
    assert changed, f"no crafted list detects the fault {fault}"
