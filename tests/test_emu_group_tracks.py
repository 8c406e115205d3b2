"""CPU test: the body of the group model kernel (tm_group_body: CTA i of a launch runs the chain step of its own argument block) on the
host emulator, three filters -- different means, one mono and two stereo rigs, different tracks, one gated off by its success counter --
bit for bit against the per-filter body at the same track; also under ThreadSanitizer."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "emu", "emu_group_tracks.cpp")
INC = ["-I" + os.path.join(ROOT, "tests", "emu", "stubs"), "-I" + os.path.join(ROOT, "tests", "emu"), "-I" + os.path.join(ROOT, "hybvio_b200", "csrc")]


def _check(out):
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.count("  ok") == 3 and "FAIL" not in out.stdout, out.stdout


def test_group_model_body_on_host_emulator(tmp_path):
    exe = str(tmp_path / "emu_group_tracks")
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-pthread", *INC, SRC, "-lm", "-o", exe])
    _check(subprocess.run([exe], capture_output=True, text=True, timeout=600))


def test_group_model_body_is_race_free_under_thread_sanitizer(tmp_path):
    probe = tmp_path / "probe.cpp"
    probe.write_text("int main() { return 0; }\n")
    if subprocess.run(["g++", "-fsanitize=thread", str(probe), "-o", str(tmp_path / "probe")], capture_output=True).returncode != 0:
        pytest.skip("g++ -fsanitize=thread is not available")
    if subprocess.run([str(tmp_path / "probe")], capture_output=True).returncode != 0:
        pytest.skip("ThreadSanitizer binaries do not start here (address-space layout)")
    exe = str(tmp_path / "emu_group_tracks_tsan")
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-g", "-fsanitize=thread", "-ffp-contract=off", "-pthread", "-w", *INC, SRC, "-lm", "-o", exe])
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=1500, env=env)
    text = out.stdout + out.stderr
    assert "WARNING: ThreadSanitizer" not in text, text[text.index("WARNING: ThreadSanitizer"):][:1500]
    _check(out)
