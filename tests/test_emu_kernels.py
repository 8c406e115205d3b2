"""CPU test: the REAL body of the fused predict kernel (hybvio_b200/csrc/ekf_predict.cuh) compiled for the host thread
emulator (tests/emu) and compared with the C oracle -- catches indexing / staging / protocol mistakes without a GPU.
The GPU parity tests (test_gpu_ekf.py) remain the authority on the compiled sm_90a code."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_predict_kernel_body_on_host_emulator(tmp_path):
    exe = str(tmp_path / "emu_predict")
    obj = str(tmp_path / "orc_ekf.o")
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-c", os.path.join(ROOT, "oracle", "hv_oracle_ekf.c"), "-o", obj])
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-pthread", "-I" + os.path.join(ROOT, "tests", "emu", "stubs"),
                           "-I" + os.path.join(ROOT, "tests", "emu"), "-I" + os.path.join(ROOT, "hybvio_b200", "csrc"),
                           os.path.join(ROOT, "tests", "emu", "emu_predict.cpp"), obj, "-lm", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.count(" ok") == 12 and "FAIL" not in out.stdout


def test_cluster_update_kernel_body_on_host_emulator(tmp_path):
    """ekf_cluster2.cuh (8 CTAs as forked processes, distributed shared memory as a shared mapping): dense check /
    update / check+update at n = 8..84, augmentation incl. the deferred symmetrisation, selector updates, and the device-side
    gates of a chain issued without host round trips (open; closed by the model flag / the success counter / the check result),
    check + update with two noise levels in one kernel, results into the second buffers (speculative update; augmentation
    sharing a launch with outlier checks); vs the C oracle."""
    exe = str(tmp_path / "emu_update")
    obj = str(tmp_path / "orc_ekf.o")
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-c", os.path.join(ROOT, "oracle", "hv_oracle_ekf.c"), "-o", obj])
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-pthread", "-I" + os.path.join(ROOT, "tests", "emu", "stubs"),
                           "-I" + os.path.join(ROOT, "tests", "emu"), "-I" + os.path.join(ROOT, "hybvio_b200", "csrc"),
                           os.path.join(ROOT, "tests", "emu", "emu_update.cpp"), obj, "-lm", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.count(" ok") == 24 and "FAIL" not in out.stdout


def test_track_model_kernel_body_on_host_emulator(tmp_path):
    """track_model.cuh (triangulation + prepareVisualUpdate of one track per CTA) vs oracle/hv_oracle_tri.c: mono / stereo,
    2..10 poses, time shift on / off, clean and spoiled tracks (OK, BEHIND, BAD_COND, NO_CONVERGENCE)."""
    exe = str(tmp_path / "emu_track_model")
    obj = str(tmp_path / "orc_tri.o")
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-c", os.path.join(ROOT, "oracle", "hv_oracle_tri.c"), "-o", obj])
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-pthread", "-I" + os.path.join(ROOT, "tests", "emu", "stubs"),
                           "-I" + os.path.join(ROOT, "tests", "emu"), "-I" + os.path.join(ROOT, "hybvio_b200", "csrc"),
                           os.path.join(ROOT, "tests", "emu", "emu_track_model.cpp"), obj, "-lm", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.count("  ok") == 45 and "FAIL" not in out.stdout          # 40 compared with the oracle (incl. 21-pose tracks, the reference's KAT) + 5 skipped by the success counter
    assert "OK 30 BEHIND 6 BAD_COND 3 NO_CONVERGENCE 1" in out.stdout and 'reference KAT "visual"' in out.stdout


def test_track_model_ldlt_matches_oracle(tmp_path):
    """The register-resident 3x3 pivoted LDL^T of the track-model kernel vs the oracle's (Eigen's algorithm) on 200k random
    symmetric matrices: same pivots, backward error at rounding level."""
    exe = str(tmp_path / "emu_ldlt3")
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-fpermissive", "-w", "-I" + os.path.join(ROOT, "tests", "emu", "stubs"),
                           "-I" + os.path.join(ROOT, "tests", "emu"), "-I" + os.path.join(ROOT, "hybvio_b200", "csrc"),
                           os.path.join(ROOT, "tests", "emu", "emu_ldlt3.cpp"), "-lm", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "pivot mismatches 0;" in out.stdout, out.stdout + out.stderr


def test_device_gated_chain_on_host_emulator(tmp_path):
    """The device side of hv_ekf_visual_tracks: per track tm_body -> ek2_body check -> ek2_body update, talking through the gate /
    slot / counter words only (inlier, chi2 outlier, point behind the cameras, skipped after the last allowed update), against
    the same loop driven through the C oracles; final filter state within 1e-9."""
    exe = str(tmp_path / "emu_chain")
    objs = []
    for name in ("hv_oracle_ekf", "hv_oracle_tri"):
        obj = str(tmp_path / (name + ".o"))
        subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-c", os.path.join(ROOT, "oracle", name + ".c"), "-o", obj])
        objs.append(obj)
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-pthread", "-I" + os.path.join(ROOT, "tests", "emu", "stubs"),
                           "-I" + os.path.join(ROOT, "tests", "emu"), "-I" + os.path.join(ROOT, "hybvio_b200", "csrc"),
                           os.path.join(ROOT, "tests", "emu", "emu_chain.cpp"), *objs, "-lm", "-o", exe])
    for args, tag in (([], "chain: 3 updates (oracle 3)"), (["fused"], "chain (fused check+update): 3 updates (oracle 3)")):
        out = subprocess.run([exe, *args], capture_output=True, text=True, timeout=900)
        assert out.returncode == 0, out.stdout + out.stderr
        assert out.stdout.count("  ok") == 10 and "FAIL" not in out.stdout and tag in out.stdout


def _lk_device_part(tmp_path):
    """The device part of hybvio_b200/csrc/lk.cu (everything before the host launcher, which uses <<< >>>) as an includable file."""
    src = open(os.path.join(ROOT, "hybvio_b200", "csrc", "lk.cu")).read()
    cut = src.index("\ncudaError_t hv_launch_lk")
    inc = tmp_path / "lk_device.inc"
    inc.write_text(src[:cut] + "\n")
    return str(tmp_path)


def test_lk_kernel_bodies_on_host_emulator(tmp_path):
    """hv_lk_cta_kernel<WIN> (CTA per feature; 4 warps, and 8 at WIN = 31) and hv_lk_kernel<WIN> (warp per feature) for every window size
    the launcher dispatches (11, 15, 21, 31) on the emulator: end points and statuses bit-identical to the C oracle in the kernels'
    accumulation order, with and without initial flow, incl. points outside the image and on a flat patch."""
    exe = str(tmp_path / "emu_lk")
    obj = str(tmp_path / "orc_lk.o")
    incdir = _lk_device_part(tmp_path)
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-c", os.path.join(ROOT, "oracle", "hv_oracle_lk.c"), "-o", obj])
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-ffp-contract=off", "-pthread", "-w", "-I" + incdir, "-I" + os.path.join(ROOT, "tests", "emu", "stubs"),
                           "-I" + os.path.join(ROOT, "tests", "emu"), "-I" + os.path.join(ROOT, "hybvio_b200", "csrc"),
                           os.path.join(ROOT, "tests", "emu", "emu_lk.cpp"), obj, "-lm", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.count("  ok") == 18 and "FAIL" not in out.stdout and "hv_lk_cta_kernel<31, 8>" in out.stdout
    for win, tracked in ((31, 35), (21, 34), (15, 33), (11, 30)):
        assert out.stdout.count(f"<{win}") == (6 if win == 31 else 4) and f"<{win}>, useInitial=1: 40 features, {tracked} tracked" in out.stdout


def _pyr_device_part(tmp_path):
    """The device part of hybvio_b200/csrc/pyramid.cu; its `extern __shared__` array becomes a pointer the harness sets."""
    src = open(os.path.join(ROOT, "hybvio_b200", "csrc", "pyramid.cu")).read()
    dev = src[:src.index("\n// ---- TMA descriptors (host)")]
    decl = "extern __shared__ __align__(128) uint8_t smem[];"
    assert decl in dev
    (tmp_path / "pyr_device.inc").write_text(dev.replace(decl, "uint8_t* smem = emu_dynamic_smem;") + "\n")
    return str(tmp_path)


def test_pyramid_kernel_body_on_host_emulator(tmp_path):
    """hv_pyr_fused2_kernel (strips, two 16-bit lanes per register) on the emulator: gray and Scharr gradient
    images of every level bit-identical to the oracle (OpenCV's pyrDown + Scharr arithmetic), 752 x 480 and 512 x 512 with 4 levels,
    ragged sizes, widths that are not multiples of 4, 6-level pyramids down to 5 pixels, images of only 0 / 255 (lane limits), frame
    copied into level 0 or read from a separate buffer; every vector access of the second generation checked for alignment."""
    exe = str(tmp_path / "emu_pyramid")
    obj = str(tmp_path / "orc_lk.o")
    incdir = _pyr_device_part(tmp_path)
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-c", os.path.join(ROOT, "oracle", "hv_oracle_lk.c"), "-o", obj])
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-pthread", "-w", "-I" + incdir, "-I" + os.path.join(ROOT, "tests", "emu", "stubs"),
                           "-I" + os.path.join(ROOT, "tests", "emu"), "-I" + os.path.join(ROOT, "hybvio_b200", "csrc"),
                           os.path.join(ROOT, "tests", "emu", "emu_pyramid.cpp"), obj, "-lm", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.count("  ok") == 18 and "FAIL" not in out.stdout
    assert "gen2 752x480, 4 levels" in out.stdout and "gen2 130x70, 5 levels" in out.stdout and "gen2 512x512, 4 levels" in out.stdout


def test_kernel_bodies_are_race_free_under_thread_sanitizer(tmp_path):
    """The emulator runs every CUDA thread as an OS thread and every barrier as a real barrier, so ThreadSanitizer sees a missing
    __syncthreads / __syncwarp / cluster.sync as a data race. Single-CTA kernels run as they are; the cluster kernels run in the
    all-CTAs-in-one-process mode of emu_cluster.h (every CTA out of its own copy of the harness's shared library), so that accesses
    between CTAs -- distributed shared memory, exchanges through global memory -- are covered as well. No report allowed."""
    import pytest
    probe = tmp_path / "probe.cpp"
    probe.write_text("int main() { return 0; }\n")
    if subprocess.run(["g++", "-fsanitize=thread", str(probe), "-o", str(tmp_path / "probe")], capture_output=True).returncode != 0:
        pytest.skip("g++ -fsanitize=thread is not available")
    if subprocess.run([str(tmp_path / "probe")], capture_output=True).returncode != 0:
        pytest.skip("ThreadSanitizer binaries do not start here (address-space layout)")
    incdir = _lk_device_part(tmp_path)
    _pyr_device_part(tmp_path)
    objs = {}
    for name in ("hv_oracle_ekf", "hv_oracle_tri", "hv_oracle_lk"):
        objs[name] = str(tmp_path / (name + ".o"))
        subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-c", os.path.join(ROOT, "oracle", name + ".c"), "-o", objs[name]])
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0")
    flags = ["g++", "-std=c++20", "-O1", "-g", "-fsanitize=thread", "-ffp-contract=off", "-pthread", "-w", "-I" + incdir,
             "-I" + os.path.join(ROOT, "tests", "emu", "stubs"), "-I" + os.path.join(ROOT, "tests", "emu"), "-I" + os.path.join(ROOT, "hybvio_b200", "csrc")]
    # (harness, oracle objects, argument lists, extra environment, cluster kernel?)
    runs = [("emu_track_model", ["hv_oracle_tri"], [[]], {}, False), ("emu_track_model", ["hv_oracle_tri"], [[]], {"EMU_NT": "512"}, False),
            ("emu_predict", ["hv_oracle_ekf"], [[]], {}, False), ("emu_lk", ["hv_oracle_lk"], [[]], {}, False), ("emu_pyramid", ["hv_oracle_lk"], [[]], {}, False),
            ("emu_update", ["hv_oracle_ekf"], [["0"], ["3"], ["5"], ["12"], ["18"], ["21"]], {}, True),
            ("emu_chain", ["hv_oracle_ekf", "hv_oracle_tri"], [[], ["fused"]], {}, True)]
    built = {}
    for src, deps, arglists, extra, cluster in runs:
        if src not in built:
            exe = str(tmp_path / (src + "_tsan"))
            cpp = os.path.join(ROOT, "tests", "emu", src + ".cpp")
            mode = ["-DEMU_CLUSTER_THREADS"] if cluster else []
            subprocess.check_call(flags + mode + [cpp, *[objs[d] for d in deps], "-lm", "-ldl", "-o", exe])
            lib = None
            if cluster:
                lib = str(tmp_path / ("lib" + src + "_body.so"))
                subprocess.check_call(flags + mode + ["-DEMU_AS_LIB", "-shared", "-fPIC", "-fvisibility=hidden", cpp, "-o", lib])
            built[src] = (exe, lib)
        exe, lib = built[src]
        for args in arglists:
            e = dict(env, **extra)
            if lib:
                e["EMU_BODY_LIB"] = lib
            out = subprocess.run([exe, *args], capture_output=True, text=True, timeout=1500, env=e)
            text = out.stdout + out.stderr
            assert "WARNING: ThreadSanitizer" not in text, (src, args, text[text.index("WARNING: ThreadSanitizer"):][:1500])
            assert out.returncode == 0 and "FAIL" not in out.stdout and " ok" in out.stdout, (src, args, out.stdout[-800:] + out.stderr[-400:])
