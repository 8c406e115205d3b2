"""CPU test: the REAL body of hv_subpix_kernel (hybvio_b200/csrc/subpix.cu) compiled for the host thread emulator (tests/emu) and
compared bit for bit with the cv::cornerSubPix oracle (oracle/hv_oracle_subpix.c) -- indexing, border-patch and warp-protocol
mistakes surface without a GPU. The GPU tests (test_gpu_subpix.py) remain the authority on the compiled sm_90a code."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_subpix_kernel_body_on_host_emulator(tmp_path):
    src = open(os.path.join(ROOT, "hybvio_b200", "csrc", "subpix.cu")).read()
    dev = src[:src.index("\ncudaError_t hv_launch_subpix")]
    decl = "extern __shared__ __align__(16) unsigned char subpix_smem[];"
    assert decl in dev
    (tmp_path / "subpix_device.inc").write_text(dev.replace(decl, "unsigned char* subpix_smem = emu_dynamic_smem;") + "\n")
    exe = str(tmp_path / "emu_subpix")
    obj = str(tmp_path / "orc_subpix.o")
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-c", os.path.join(ROOT, "oracle", "hv_oracle_subpix.c"), "-o", obj])
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-ffp-contract=off", "-pthread", "-w", "-I" + str(tmp_path),
                           "-I" + os.path.join(ROOT, "tests", "emu", "stubs"), "-I" + os.path.join(ROOT, "tests", "emu"),
                           "-I" + os.path.join(ROOT, "hybvio_b200", "csrc"), os.path.join(ROOT, "tests", "emu", "emu_subpix.cpp"), obj, "-lm", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.count("  ok") == 8 and "FAIL" not in out.stdout and "all ok" in out.stdout, out.stdout
