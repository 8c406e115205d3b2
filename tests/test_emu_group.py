"""CPU test: the body of the group cluster kernel (ek2_group_body: cluster i of a launch runs its own argument block) on the host
emulator, three clusters from two filters at N = 62 against the C oracle -- each cluster works on its own filter buffers, exchange
area, result words and second buffers."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_group_cluster_body_on_host_emulator(tmp_path):
    exe = str(tmp_path / "emu_group")
    obj = str(tmp_path / "orc_ekf.o")
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-c", os.path.join(ROOT, "oracle", "hv_oracle_ekf.c"), "-o", obj])
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-pthread", "-I" + os.path.join(ROOT, "tests", "emu", "stubs"),
                           "-I" + os.path.join(ROOT, "tests", "emu"), "-I" + os.path.join(ROOT, "hybvio_b200", "csrc"),
                           os.path.join(ROOT, "tests", "emu", "emu_group.cpp"), obj, "-lm", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.count("  ok") == 3 and "FAIL" not in out.stdout, out.stdout
