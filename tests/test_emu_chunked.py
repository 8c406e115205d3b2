"""CPU test: the row-chunked form of the cluster update (ekf_cluster2.cuh, EkfUpdateArgs::rowChunk) on the host emulator
(tests/emu/emu_update_chunked.cpp) against the C oracle, and the same body under ThreadSanitizer (the barriers between chunks and
between the check and update passes are the new synchronisation)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INC = ["-I" + os.path.join(ROOT, "tests", "emu", "stubs"), "-I" + os.path.join(ROOT, "tests", "emu"), "-I" + os.path.join(ROOT, "hybvio_b200", "csrc")]
SRC = os.path.join(ROOT, "tests", "emu", "emu_update_chunked.cpp")
CASES = 15


def _oracle(tmp_path, flags=()):
    obj = str(tmp_path / "orc_ekf.o")
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", *flags, "-c", os.path.join(ROOT, "oracle", "hv_oracle_ekf.c"), "-o", obj])
    return obj


def test_row_chunked_update_on_host_emulator(tmp_path):
    """Chunk heights 8 / 16 / n - 8 / 40 (84 = 40 + 40 + 4) / 41 (60 = 41 + 19), N = 202 .. 400: check, update, check+update with one
    and with two noise levels, gated chain links; statuses identical, chi2 within 1e-8 relative, m within 1e-9, max|dP| / max|P| <= 1e-9;
    S positive definite on the first chunk only: the numeric flag and (m, P) bit-identical."""
    exe = str(tmp_path / "emu_update_chunked")
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-pthread", *INC, SRC, _oracle(tmp_path), "-lm", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=1500)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.count("  ok") == CASES and "FAIL" not in out.stdout


def test_row_chunked_update_is_race_free_under_thread_sanitizer(tmp_path):
    """All CTAs in one process (emu_cluster.h), every CUDA thread an OS thread: a missing barrier between chunks or passes is a race."""
    probe = tmp_path / "probe.cpp"
    probe.write_text("int main() { return 0; }\n")
    if subprocess.run(["g++", "-fsanitize=thread", str(probe), "-o", str(tmp_path / "probe")], capture_output=True).returncode != 0:
        pytest.skip("g++ -fsanitize=thread is not available")
    if subprocess.run([str(tmp_path / "probe")], capture_output=True).returncode != 0:
        pytest.skip("ThreadSanitizer binaries do not start here (address-space layout)")
    flags = ["g++", "-std=c++20", "-O1", "-g", "-fsanitize=thread", "-ffp-contract=off", "-pthread", "-w", *INC, "-DEMU_CLUSTER_THREADS"]
    exe, lib = str(tmp_path / "emu_chunked_tsan"), str(tmp_path / "libemu_chunked_body.so")
    subprocess.check_call(flags + [SRC, _oracle(tmp_path), "-lm", "-ldl", "-o", exe])
    subprocess.check_call(flags + ["-DEMU_AS_LIB", "-shared", "-fPIC", "-fvisibility=hidden", SRC, "-o", lib])
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0", EMU_BODY_LIB=lib)
    # three chunks with a short last one; the check pass then the update pass; 8-row chunks with one-stage S, gated; failure in chunk 2
    for case in ("3", "8", "10", "14"):
        out = subprocess.run([exe, case], capture_output=True, text=True, timeout=1500, env=env)
        text = out.stdout + out.stderr
        assert "WARNING: ThreadSanitizer" not in text, (case, text[text.index("WARNING: ThreadSanitizer"):][:1500])
        assert out.returncode == 0 and "FAIL" not in out.stdout and " ok" in out.stdout, (case, out.stdout[-800:] + out.stderr[-400:])
