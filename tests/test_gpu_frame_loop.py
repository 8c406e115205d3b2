"""The benchmarked frame loop against the serial replay of tests/frame_loop_replay.py, under every schedule the benchmark uses.

Four drivers run the loop of bench.Session: step_device (Python, two streams with events, programmatic dependent launch, the
covariance launch and the outlier checks on the library's side streams), hv_dev_run (native; LK on the filter stream, its own
evLk / evPyr events for the pyramid rebuild), step_e2e (Python, host buffers, results polled from mapped pinned memory) and
hv_e2e_run (native, host buffers). Each runs 200 frames of BASELINE config 2 with a frame pool of 8 stereo pairs (it turns round
every 14 frames; the EKF input pool wraps at 64 frames, the pose trail at 20), in chunks of 1, 2, 3, 7, 16 and 64 frames. After
every chunk: the last frame's pyramids and LK outputs bit for bit, its check decisions identical and chi2 within 1e-8, m and P
within the replay's rounding envelope. hv_e2e_run keeps its LK outputs and check results inside the driver: for it, the
pyramids, the state and the returned pose are compared.

The same 200 frames must leave the same bits whatever the schedule: one uninterrupted call, the chunks, HV_EKF_NO_PDL=1 and
HV_BENCH_NO_OVERLAP=1 (step_device). Those switches are read once per process, so every configuration runs in a child process, once.

Host-buffer and device families run the same kernels for the benchmark's list (see ekf_capi.cu: run_ops_host_async and run_ops
both issue the IMU burst as one predict launch, every check + update through launch_update, and the 15 outlier checks as one
ekf_check_batch_cluster2_kernel launch; the symmetrise + augmentation runs the same cluster body either as one more cluster of
that launch or, on the device path in latency mode, as its own ekf_update_cluster2_kernel launch), so the two families must
agree bit for bit as well.

In the benchmark the EKF measurements come from a synthetic pool that does not depend on LK, and the LK initial guesses are
precomputed: the flow predictor and the measurement model are not part of what this checks.
"""
import hashlib
import json
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import frame_loop_replay as R  # noqa: E402
import bench  # noqa: E402

pytestmark = pytest.mark.gpu

FRAMES = 200
POOL = 8
CHUNKS = R.chunk_schedule(FRAMES)
SESSION_CHUNKS = [1, 7, 64, 128]
DEVICE_DRIVERS = ("step_device", "dev_native")
HOST_DRIVERS = ("step_e2e", "e2e_native")
DRIVERS = DEVICE_DRIVERS + HOST_DRIVERS
# child process jobs: environment, and the (driver, schedule) runs made under it
JOBS = {
    "default": ({}, [(d, "chunked") for d in DRIVERS + ("step_device_copy",)] + [(d, "one_call") for d in DRIVERS]),
    "no_pdl": ({"HV_EKF_NO_PDL": "1"}, [(d, "chunked") for d in DRIVERS]),
    "no_overlap": ({"HV_BENCH_NO_OVERLAP": "1"}, [("step_device", "chunked")]),
}
LAUNCHES_PER_FRAME = {"default": 12, "no_pdl": 11}       # hv_dev_run: latency mode, throughput mode (HV_EKF_NO_PDL=1)


# ------------------------------------------------------------------------------------------------ child side
def step_device_copy(self):
    """bench.Session.step_device line for line, so that its event waits can be changed in an experiment without touching bench.py.
    Taking out A.wait_event(self.ev_ekf) changes no output: in the benchmark LK reads nothing the filter writes (its initial guesses
    are precomputed), so that wait orders work without carrying data. Likewise hv_dev_run's evLk only protects the LK of frames
    whose outputs the next frame overwrites, and the pyramid build that its evPyr wait orders before LK finishes well within the
    filter work queued ahead of that LK. Taking out either wait changed no output in a run of this file on an H100."""
    self.k += 1
    j = bench.frame_index(self.k)
    ctx, inp, A, B = self.ctx, self.inp, self.stream, self.stream_b
    cur = self.pyr[2:4]
    ctx.build_pyramids(cur[:bench.NCAM], [self.d_frames[j, c] for c in range(bench.NCAM)], device=True)
    fr = self._ekf_inputs(self.k)
    ops = self.ops_dev[fr]
    for s in range(bench.PREDICTS):
        self.t += 0.005
        ops[2 * s].t = self.t
    if not self.overlap:
        A.wait_stream(B); B.wait_stream(A)
    self.ekf.run_device(ops, bench.IMU_OPS)
    self.ekf.predicted_mean_device(self.d_mean.data_ptr())
    self.ev_ekf.record(B)
    self.ekf.flush()
    A.wait_event(self.ev_ekf)
    init = self.d_init[0, j - 1] if j > self.prev_j else self.d_init[1, j]
    with self.torch.cuda.stream(A):
        self.d_next.copy_(init)
    ctx.lk_track_device(self.pyr[0], cur[0], self.d_points, self.d_next, self.d_status, self.d_ts, bench.NFEAT, True)
    if bench.STEREO:
        ctx.lk_track_device(cur[0], cur[1], self.d_next, self.d_next2, self.d_status, self.d_ts, bench.NFEAT, False)
    self.ev_lk.record(A)
    B.wait_event(self.ev_lk)
    self.ekf.run_device(bench.ctypes_slice(ops, bench.IMU_OPS, self.nops - bench.IMU_OPS), self.nops - bench.IMU_OPS)
    self.pyr = self.pyr[2:4] + self.pyr[0:2]
    self.prev_j = j


def _digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def pyramid_digests(levels):
    """[camera][level] -> (gray digest, deriv digest) of unpadded (uint8, int16) levels."""
    return [[(_digest(np.asarray(g, np.uint8)), _digest(np.asarray(d, np.int16))) for g, d in cam] for cam in levels]


class Driver:
    """One session driven by one of the four drivers; observe() reads what the last frame left."""

    def __init__(self, kind, inputs):
        import torch
        self.kind, self.torch = kind, torch
        self.sess = bench.Session(0, inputs)
        self.cap = {}
        if kind == "step_e2e":
            s, cap = self.sess, self.cap
            run_host, lk_track = s.ekf.run_host, s.ctx.lk_track

            def run_host_(*a, **kw):
                r = run_host(*a, **kw)
                cap["status"], cap["chi2"] = r[0][bench.IMU_OPS:], r[1][bench.IMU_OPS:]
                return r

            def lk_track_(*a, **kw):
                r = lk_track(*a, **kw)
                cap["lk"] = (cap.get("lk", []) + [r])[-bench.NCAM:]
                return r
            s.ekf.run_host, s.ctx.lk_track = run_host_, lk_track_

    def run(self, n):
        s = self.sess
        if self.kind == "step_device":
            for _ in range(n):
                s.step_device()
        elif self.kind == "step_device_copy":
            for _ in range(n):
                step_device_copy(s)
        elif self.kind == "dev_native":
            s.run_dev_native(n)
        elif self.kind == "step_e2e":
            for _ in range(n):
                self.cap["m"] = s.step_e2e()
        elif self.kind == "e2e_native":
            self.cap["pose"] = s.run_e2e_native(n)[1]
        else:
            raise ValueError(self.kind)

    def observe(self):
        s = self.sess
        s.ctx.sync(); s.ctx_b.sync()
        self.torch.cuda.synchronize()
        o = {"k": s.k}
        if self.kind in ("step_device", "step_device_copy", "dev_native"):
            vu, chi2 = s.ekf.run_device_results(s.nops - bench.IMU_OPS)
            o["status"], o["chi2"] = vu[:bench.CHECKS], chi2[:bench.CHECKS]
            o["lk_next_temporal"] = s.d_next.cpu().numpy()
            if bench.STEREO:
                o["lk_next_stereo"] = s.d_next2.cpu().numpy()
            o["lk_status"], o["lk_track_status"] = s.d_status.cpu().numpy(), s.d_ts.cpu().numpy()
        elif self.kind == "step_e2e":
            o["status"], o["chi2"] = self.cap["status"][:bench.CHECKS], self.cap["chi2"][:bench.CHECKS]
            lk = self.cap["lk"]
            o["lk_next_temporal"] = lk[0][0]
            if bench.STEREO:
                o["lk_next_stereo"] = lk[1][0]
            o["lk_status"], o["lk_track_status"] = lk[-1][1], lk[-1][2]
        o["m"], o["P"] = s.ekf.download()
        if "m" in self.cap:
            o["m_returned"] = self.cap["m"]
        if "pose" in self.cap:
            o["pose_returned"] = self.cap["pose"]
        o["pyr"] = pyramid_digests([[p.download(lv) for lv in range(p.levels)] for p in s.pyr[:bench.NCAM]])
        return o


def save_run(path, observations):
    arrays, meta = {}, []
    for i, o in enumerate(observations):
        meta.append({"k": o["k"], "pyr": o["pyr"]})
        for key, v in o.items():
            if key not in ("k", "pyr"):
                arrays[f"{i}:{key}"] = np.asarray(v)
    np.savez(path + ".npz", **arrays)
    with open(path + ".json", "w") as f:
        json.dump(meta, f)


def load_run(path):
    meta = json.load(open(path + ".json"))
    z = np.load(path + ".npz")
    obs = [{"k": m["k"], "pyr": [[tuple(x) for x in cam] for cam in m["pyr"]]} for m in meta]
    for key in z.files:
        i, name = key.split(":", 1)
        obs[int(i)][name] = z[key]
    return obs


def launches_per_frame(inputs):
    d = Driver("dev_native", inputs)
    d.run(4)
    d.observe()
    c = d.sess.ctx.launches + d.sess.ctx_b.launches
    d.run(16)
    d.observe()
    return (d.sess.ctx.launches + d.sess.ctx_b.launches - c) / 16.0


def child_main(job, out_dir):
    import torch
    assert bench.POOL_FRAMES == POOL, "run with HV_BENCH_POOL_FRAMES"
    os.makedirs(out_dir, exist_ok=True)
    inputs = bench.Inputs(torch.device("cuda", 0))
    info = {}
    if job == "sessions":
        # one session alone, then four on one shared Inputs driven concurrently from threads (bench.py's run_parallel)
        alone = Driver("dev_native", inputs)
        for n in SESSION_CHUNKS:
            alone.run(n)
        save_run(os.path.join(out_dir, "alone"), [alone.observe()])
        group = [Driver("dev_native", inputs) for _ in range(4)]
        for n in SESSION_CHUNKS:
            gate = threading.Barrier(len(group))

            def work(d, n=n):
                torch.cuda.set_device(0)
                gate.wait()
                d.run(n)
            th = [threading.Thread(target=work, args=(d,)) for d in group]
            for t in th:
                t.start()
            for t in th:
                t.join()
        for i, d in enumerate(group):
            save_run(os.path.join(out_dir, f"session{i}"), [d.observe()])
    else:
        for kind, sched in JOBS[job][1]:
            d = Driver(kind, inputs)
            obs = []
            for n in (CHUNKS if sched == "chunked" else [FRAMES]):
                d.run(n)
                obs.append(d.observe())
            save_run(os.path.join(out_dir, f"{kind}.{sched}"), obs)
        info["launches_per_frame"] = launches_per_frame(inputs)
    with open(os.path.join(out_dir, "info.json"), "w") as f:
        json.dump(info, f)


# ------------------------------------------------------------------------------------------------ parent side
def run_child(job, out_dir, extra_env):
    env = dict(os.environ, HV_BENCH_POOL_FRAMES=str(POOL), **extra_env)
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "child", job, out_dir], capture_output=True, text=True,
                       timeout=1200, env=env, cwd=ROOT)
    assert r.returncode == 0, f"child {job} failed:\n{r.stdout[-2000:]}\n{r.stderr[-3000:]}"


@pytest.fixture(scope="module")
def loop_runs(tmp_path_factory):
    base = str(tmp_path_factory.mktemp("frame_loop"))
    for job, (env, _) in JOBS.items():
        run_child(job, os.path.join(base, job), env)
    run_child("sessions", os.path.join(base, "sessions"), {"HV_EKF_NO_PDL": "1", "CUDA_DEVICE_MAX_CONNECTIONS": "32"})
    return base


@pytest.fixture(scope="module")
def replay():
    """The serial replay of the same 200 frames, with the tracker outputs of every chunk end (Inputs built as the sessions
    built theirs: same config, same pool size, on the GPU)."""
    import torch
    with R.configured(2, POOL):
        inputs = bench.Inputs(torch.device("cuda", 0))
        marks = sorted(set(R.chunk_ends(CHUNKS)) | set(R.chunk_ends(SESSION_CHUNKS)))
        rep = R.Replay(inputs, FRAMES, marks)
        rep.tracker = {}
        for k in marks:
            t = R.tracker_replay(inputs, k)
            t["pyr"] = pyramid_digests(t["pyr"])
            rep.tracker[k] = t
    return rep


def compare_with_replay(rep, obs, label):
    """Every observation of a run against the replay; prints frames compared and the worst ratio to D(k). Returns failures."""
    bad, worst = [], (0.0, 0.0)
    for o in obs:
        k = int(o["k"])
        ok, rm, rP, dm, dP = rep.gate(k, o["m"], o["P"])
        worst = (max(worst[0], rm), max(worst[1], rP))
        if not ok:
            bad.append(f"frame {k}: m {dm:.3g} ({rm:.2f} D), P {dP:.3g} ({rP:.2f} D)")
        if "status" in o:
            bad += R.check_mismatches(rep, k, o["status"], o["chi2"])
        ref = rep.tracker[k]
        got = {key: o[key] for key in ("lk_next_temporal", "lk_next_stereo", "lk_status", "lk_track_status") if key in o}
        bad += [f"frame {k}: {x}" for x in R.tracker_mismatches(dict(ref, pyr=[]), got)]
        if [list(map(tuple, c)) for c in o["pyr"]] != [list(map(tuple, c)) for c in ref["pyr"]]:
            bad.append(f"frame {k}: pyramids differ from the oracle")
        if "pose_returned" in o and not np.array_equal(o["pose_returned"], o["m"][:20]):
            bad.append(f"frame {k}: pose returned by hv_e2e_run differs from the downloaded state")
        if "m_returned" in o and not np.array_equal(o["m_returned"], o["m"]):
            bad.append(f"frame {k}: m returned by step_e2e differs from the downloaded state")
    print(f"\n{label}: {len(obs)} chunk ends, last frame {int(obs[-1]['k'])}, worst |GPU - replay| / D(k): m {worst[0]:.2f}, P {worst[1]:.2f}")
    return bad


def same_bits(a, b, keys=("m", "P", "lk_next_temporal", "lk_next_stereo", "lk_status", "lk_track_status")):
    """Names of what differs between two final observations (pyramids by digest)."""
    out = [k for k in keys if k in a and k in b and not np.array_equal(a[k], b[k])]
    if a["pyr"] != b["pyr"]:
        out.append("pyramids")
    return out


RUNS = [(job, kind, sched) for job, (_, runs) in JOBS.items() for kind, sched in runs]


@pytest.mark.parametrize("job,kind,sched", RUNS, ids=[f"{k}-{s}-{j}" for j, k, s in RUNS])
def test_driver_matches_serial_replay(loop_runs, replay, job, kind, sched):
    obs = load_run(os.path.join(loop_runs, job, f"{kind}.{sched}"))
    assert int(obs[-1]["k"]) == FRAMES
    bad = compare_with_replay(replay, obs, f"{kind} {sched} ({job})")
    assert not bad, bad[:10]


@pytest.mark.parametrize("kind", DRIVERS)
def test_schedules_do_not_change_bits(loop_runs, kind):
    ref = load_run(os.path.join(loop_runs, "default", f"{kind}.chunked"))[-1]
    others = [(job, sched) for job, kind_, sched in RUNS if kind_ == kind and (job, sched) != ("default", "chunked")]
    assert len(others) >= 2
    for job, sched in others:
        o = load_run(os.path.join(loop_runs, job, f"{kind}.{sched}"))[-1]
        assert not same_bits(ref, o), f"{kind}: {sched} under {job} differs from the chunked default run in {same_bits(ref, o)}"


def test_drivers_agree_bit_for_bit(loop_runs):
    """step_device and hv_dev_run issue the same kernels; so does the copy of step_device; and the host-buffer family runs the same
    kernels as the device family for this list (module docstring): every driver ends on the same bits."""
    final = {k: load_run(os.path.join(loop_runs, "default", f"{k}.chunked"))[-1] for k in DRIVERS + ("step_device_copy",)}
    ref = final["step_device"]
    for k, o in final.items():
        keys = ("m", "P") if k == "e2e_native" else ("m", "P", "lk_next_temporal", "lk_next_stereo", "lk_status", "lk_track_status")
        assert not same_bits(ref, o, keys), f"{k} differs from step_device in {same_bits(ref, o, keys)}"
        if "status" in o:
            assert np.array_equal(o["status"], ref["status"]) and np.array_equal(o["chi2"], ref["chi2"]), k


def test_several_sessions_on_one_gpu_match_one_session(loop_runs, replay):
    alone = load_run(os.path.join(loop_runs, "sessions", "alone"))
    assert not compare_with_replay(replay, alone, "dev_native alone (HV_EKF_NO_PDL=1, 32 connections)")
    for i in range(4):
        o = load_run(os.path.join(loop_runs, "sessions", f"session{i}"))[-1]
        assert int(o["k"]) == FRAMES
        assert not same_bits(alone[-1], o), f"session {i} of 4 differs from the session run alone in {same_bits(alone[-1], o)}"
        assert np.array_equal(o["status"], alone[-1]["status"]) and np.array_equal(o["chi2"], alone[-1]["chi2"])


@pytest.mark.parametrize("job", sorted(LAUNCHES_PER_FRAME))
def test_launches_per_device_resident_frame(loop_runs, job):
    """DESIGN.md / README: a device-resident frame is 12 launches (pyramids, predicted mean, predict, 2 LK, 5 check + update,
    outlier checks, symmetrise + augmentation). In throughput mode (HV_EKF_NO_PDL=1) the augmentation is one more cluster of the
    outlier checks' launch: 11."""
    got = json.load(open(os.path.join(loop_runs, job, "info.json")))["launches_per_frame"]
    print(f"\nhv_dev_run launches per frame ({job}): {got}")
    assert got == LAUNCHES_PER_FRAME[job]


# ------------------------------------------------------------------------------------------------ the headline command's own outputs
DUMP_CASES = {
    "config2_readme": (2, ["--steps", "400", "--warmup", "20"]),
    "config4": (4, ["--steps", "60", "--warmup", "10"]),
    "config1_mono": (1, ["--steps", "60", "--warmup", "10"]),
}


def bench_dump(out_dir, cid, args):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--step-only", "--config", str(cid), *args, "--dump-outputs", out_dir],
                       capture_output=True, text=True, timeout=1200, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    return {f[:-4]: np.load(os.path.join(out_dir, f)) for f in os.listdir(out_dir)}


def frames_seen(args):
    """The filter of session 0 sees 2 W + min(S, 100) + S frames: timed_loop(step_device) (W warm-up + min(S, 100)), then
    run_dev_native for W warm-up and S steps."""
    s, w = int(args[args.index("--steps") + 1]), max(3, int(args[args.index("--warmup") + 1]))
    return 2 * w + min(s, 100) + s


@pytest.fixture(scope="module")
def dumps(tmp_path_factory):
    base = tmp_path_factory.mktemp("dumps")
    return {name: bench_dump(str(base / name), cid, args) for name, (cid, args) in DUMP_CASES.items()}


@pytest.mark.parametrize("case", sorted(DUMP_CASES))
def test_bench_dump_matches_serial_replay(dumps, case):
    import torch
    cid, args = DUMP_CASES[case]
    d = dumps[case]
    k = frames_seen(args)
    with R.configured(cid):
        inputs = bench.Inputs(torch.device("cuda", 0))
        rep = R.Replay(inputs, k, [k])
        t = R.tracker_replay(inputs, k)
        assert ("lk_next_stereo" in d) == bench.STEREO
        cams = ("left", "right")[:bench.NCAM]
        got = {key: d[key] for key in ("lk_next_temporal", "lk_next_stereo", "lk_status", "lk_track_status") if key in d}
        got["pyr"] = [[(d[f"pyr_{c}_l{lv}_gray"], d[f"pyr_{c}_l{lv}_deriv"]) for lv in range(bench.MAXLEVEL + 1)] for c in cams]
        bad = R.tracker_mismatches(t, got)
        bad += R.check_mismatches(rep, k, d["ekf_check_status"], d["ekf_check_chi2"])
        ok, rm, rP, dm, dP = rep.gate(k, d["ekf_mean"], d["ekf_cov"])
    print(f"\nbench.py {' '.join(args)} --config {cid}: frame {k}, |GPU - replay| / D(k): m {rm:.2f}, P {rP:.2f}")
    assert ok, f"frame {k}: m {dm:.3g} ({rm:.2f} D), P {dP:.3g} ({rP:.2f} D)"
    assert not bad, bad


def test_bench_dump_of_four_sessions_matches_one_session(dumps, tmp_path):
    """--sessions 4 (HV_EKF_NO_PDL=1, 32 hardware queues, four sessions on threads): session 0 ends on the bits of the single session."""
    cid, args = DUMP_CASES["config2_readme"]
    four = bench_dump(str(tmp_path / "four"), cid, args + ["--sessions", "4"])
    one = dumps["config2_readme"]
    assert set(four) == set(one)
    assert [k for k in sorted(one) if not np.array_equal(one[k], four[k])] == []


if __name__ == "__main__" and len(sys.argv) == 4 and sys.argv[1] == "child":
    child_main(sys.argv[2], sys.argv[3])
