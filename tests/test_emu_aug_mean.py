"""CPU test: the one-CTA mean of the pose augmentation (ek2_aug_mean_cta, ekf_cluster2.cuh) on the host emulator
(tests/emu/emu_aug_mean.cpp) against the cluster body on the same inputs, bit for bit, and the same body under ThreadSanitizer."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INC = ["-I" + os.path.join(ROOT, "tests", "emu", "stubs"), "-I" + os.path.join(ROOT, "tests", "emu"), "-I" + os.path.join(ROOT, "hybvio_b200", "csrc")]
SRC = os.path.join(ROOT, "tests", "emu", "emu_aug_mean.cpp")
CASES = 25


def test_aug_mean_matches_cluster_body_on_host_emulator(tmp_path):
    """N = 62 / 160 / 202, pose trail not yet full / full, discarded pose last / in the middle, deferred symmetrisation on / off, and a
    non-positive pivot: the mean in the second buffer and the result words bitwise equal; (m, P) untouched."""
    exe = str(tmp_path / "emu_aug_mean")
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-pthread", *INC, SRC, "-lm", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=1500)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.count("  ok") == CASES and "FAIL" not in out.stdout


def test_aug_mean_is_race_free_under_thread_sanitizer(tmp_path):
    """Every CUDA thread an OS thread in one process: a missing barrier between the staging of the shifted P, HP, the block partials of S,
    the elimination and the in-place update of the mean is a race."""
    probe = tmp_path / "probe.cpp"
    probe.write_text("int main() { return 0; }\n")
    if subprocess.run(["g++", "-fsanitize=thread", str(probe), "-o", str(tmp_path / "probe")], capture_output=True).returncode != 0:
        pytest.skip("g++ -fsanitize=thread is not available")
    if subprocess.run([str(tmp_path / "probe")], capture_output=True).returncode != 0:
        pytest.skip("ThreadSanitizer binaries do not start here (address-space layout)")
    flags = ["g++", "-std=c++20", "-O1", "-g", "-fsanitize=thread", "-ffp-contract=off", "-pthread", "-w", *INC, "-DEMU_CLUSTER_THREADS"]
    exe, lib = str(tmp_path / "emu_aug_mean_tsan"), str(tmp_path / "libemu_aug_mean_body.so")
    subprocess.check_call(flags + [SRC, "-lm", "-ldl", "-o", exe])
    subprocess.check_call(flags + ["-DEMU_AS_LIB", "-shared", "-fPIC", "-fvisibility=hidden", SRC, "-o", lib])
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0", EMU_BODY_LIB=lib)
    # N = 62 trail not full; N = 202 full with the deferred symmetrisation; a non-positive pivot
    for case in ("0", "23", "24"):
        out = subprocess.run([exe, case], capture_output=True, text=True, timeout=1500, env=env)
        text = out.stdout + out.stderr
        assert "WARNING: ThreadSanitizer" not in text, (case, text[text.index("WARNING: ThreadSanitizer"):][:1500])
        assert out.returncode == 0 and "FAIL" not in out.stdout and " ok" in out.stdout, (case, out.stdout[-800:] + out.stderr[-400:])
