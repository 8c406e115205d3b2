"""Serial CPU replay of the benchmarked frame loop (bench.Session and the drivers of hybvio_b200/host/e2e_driver.cu).

What the loop computes for frame k (the first frame is k = 1), replayed one operation after the other with the C oracle:

  EKF (oracle.ekf_oracle.OracleEKF, camera_trail_length = bench.TRAIL, initialize_orientation(imu[0, 3:])), fr = k % POOL_EKF:
    1. 10 x (predict(t += 0.005, imu[10 fr + s, :3], imu[10 fr + s, 3:]), normalize_quaternions(True));
    2. the CHECKS visual checks of pool row fr in order, r = VISUAL_R, no RMSE gate; slots c < UPDATES are check + update
       (the update is applied when the check passes), the others are checks only;
    3. symmetrize(); 4. augment(-1).
  Tracker, for the last frame of a chunk: the pyramids of frame_index(k) (OracleLK.pyramid(img, 31, MAXLEVEL)), the temporal LK
  from the previous frame's left image to this frame's left image (start inputs.points, initial guess inputs.init_guess(prev_j, j))
  and the stereo LK from this frame's left to its right image (start: the temporal result, no initial guess), accum_mode=1, 20
  iterations, eps 0.03, min_eig 1e-3: the kernel's own arithmetic, so pyramids and LK must match bit for bit.

What this does NOT check: in the benchmark the EKF measurements are a synthetic pool that does not depend on LK, and the LK
initial guesses are precomputed, so the flow predictor and the measurement model are not part of the loop. The replay checks
the loop's schedule (stream order, events, programmatic dependent launch, side streams, second buffers, polled results, ring
and pool wrap-around) and the arithmetic of what it runs, not the coupling between tracker and filter.

Tolerance of the filter state: a rounding envelope derived from the oracle itself. ekf_common.TOL_M (1e-9 absolute) does not
hold over hundreds of frames even between two correct implementations: positions reach hundreds of metres and the first
frames amplify a one-ulp difference by about 1e5. D(k) is the larger of two distances from the plain replay,
  - to a replay with m <- nextafter(m, +inf) before frame 1, and
  - to a replay with that push plus m <- nextafter(m, +inf), P <- P (1 + 2^-52) after every frame,
each measured as (max over entries of |dm| / max(1, |m|), max |dP| / max |P|). A device state passes at frame k when its
distance to the plain replay is at most C_ENVELOPE * D(k), and never needs to be below FLOOR.

C_ENVELOPE = 32. Worst device distance / D(k) measured on an H100 SXM (tests/test_gpu_frame_loop.py, every driver and schedule):
  config 2, 200 frames, every chunk end: m 0.84, P 1.06;  bench.py config 2, frame 540: m 0.11, P 0.47;
  config 4, frame 140: m 4.2, P 2.3;  config 1 (mono), frame 140: m 12.5, P 18.7.
c = 8 was not enough for config 1, and the reason is the envelope, not the order of the work: in config 2 D(k) is set by the push
before frame 1 (the first frames amplify it by about 1e5); in config 1 they amplify it far less, and D(k) is set by the one ulp
per frame (m 1.2e-12, P 3.8e-14 of max |P| at frame 140). The device's own rounding is more than one ulp per frame (about 50
operations per frame, each some ulps from the oracle's summation order): a replay pushed by 16 ulps after every frame lands at
m 3.9e-11, P 3.4e-13 at frame 140 of config 1; the device is at m 1.5e-11, P 7.1e-13. Every misordering of the loop that
tests/test_frame_loop_replay.py injects is at least 700 D(k) away at the first chunk end after it.

What the envelope cannot see: a skipped symmetrize() moves P by 3e-16 to 2e-13 of max |P| -- inside D(k). The op's own tests
(tests/test_gpu_ekf_ops_ref.py) cover it.
"""
import contextlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402
from oracle import ekf_oracle, lk_oracle  # noqa: E402

C_ENVELOPE = 32.0
FLOOR = 1e-12
CHI2_RTOL = 1e-8

FAULTS = ("update_twice", "stale_check", "imu_after_visual", "timestamp")


@contextlib.contextmanager
def configured(cid, pool_frames=None):
    """bench.set_config(cid) and, optionally, the frame pool size (what HV_BENCH_POOL_FRAMES sets at import), restored after."""
    old_cid, old_pool = bench.CONFIG_ID, bench.POOL_FRAMES
    bench.set_config(cid)
    if pool_frames is not None:
        bench.POOL_FRAMES = pool_frames
    try:
        yield
    finally:
        bench.POOL_FRAMES = old_pool
        bench.set_config(old_cid)


def new_filter(inputs):
    if not os.path.exists(ekf_oracle.ORACLE_SO):
        import subprocess
        subprocess.check_call(["make", "-C", ROOT, "oracle"])
    o = ekf_oracle.OracleEKF()
    p = o.default_params()
    o.close()
    p.camera_trail_length = bench.TRAIL
    o = ekf_oracle.OracleEKF(p)
    o.initialize_orientation(inputs.imu[0, 3:])
    return o


def measurement(inputs, fr, c):
    off, n, l = inputs.ekf_off[c]
    row = inputs.ekf_pool[fr]
    return row[off:off + n * l].reshape((n, l), order="F"), row[off + n * l:off + n * l + n], row[off + n * l + n:off + n * l + 2 * n]


class FilterReplay:
    """The filter part of the loop, frame by frame. push: None, "first" (one ulp on m before frame 1) or "every" (that, and one
    ulp on m and P after every frame). fault / fault_frame: one deliberate misordering (FAULTS) at one frame."""

    def __init__(self, inputs, push=None, fault=None, fault_frame=None):
        assert fault is None or fault in FAULTS
        self.inp, self.push, self.fault, self.fault_frame = inputs, push, fault, fault_frame
        self.o = new_filter(inputs)
        self.t, self.k = 0.0, 0
        if push:
            m, _ = self.o.download()
            self.o.upload(m=np.nextafter(m, np.inf))

    def close(self):
        self.o.close()

    def _imu(self, fr, faulty):
        for s in range(bench.PREDICTS):
            self.t += 0.005
            u = self.inp.imu[fr * bench.PREDICTS + s]
            dt = 1e-7 if faulty and self.fault == "timestamp" and s == 3 else 0.0
            self.o.predict(self.t + dt, u[:3], u[3:])
            self.o.normalize_quaternions(True)

    def step(self):
        """One frame; returns (status int32[CHECKS], chi2 float64[CHECKS])."""
        self.k += 1
        k, fr = self.k, self.k % bench.POOL_EKF
        faulty = self.fault is not None and k == self.fault_frame
        if not (faulty and self.fault == "imu_after_visual"):
            self._imu(fr, faulty)
        st, chi2 = np.zeros(bench.CHECKS, np.int32), np.zeros(bench.CHECKS)
        snap = None
        for c in range(bench.CHECKS):
            H, f, y = measurement(self.inp, fr, c)
            if faulty and self.fault == "stale_check" and c == 0:
                snap = self.o.clone()                  # the state a check of slot 1 that read P too early would see
            if faulty and self.fault == "stale_check" and c == 1:
                self.o.close()
                self.o = snap
            st[c], chi2[c] = self.o.visual_check(H, f, y, bench.VISUAL_R)
            if c < bench.UPDATES and st[c] == 0:
                self.o.visual_update(H, f, y, bench.VISUAL_R)
                if faulty and self.fault == "update_twice" and c == 3:
                    self.o.visual_update(H, f, y, bench.VISUAL_R)
        if faulty and self.fault == "imu_after_visual":
            self._imu(fr, False)
        self.o.symmetrize()
        self.o.augment(-1)
        if self.push == "every":
            m, P = self.o.download()
            self.o.upload(m=np.nextafter(m, np.inf), P=P * (1.0 + 2.0 ** -52))
        return st, chi2


def distance(m_ref, P_ref, m, P):
    """(max |dm| / max(1, |m_ref|), max |dP| / max |P_ref|)."""
    dm = float(np.max(np.abs(m - m_ref) / np.maximum(1.0, np.abs(m_ref))))
    dP = float(np.max(np.abs(P - P_ref)) / np.max(np.abs(P_ref)))
    return dm, dP


class Replay:
    """Plain replay of frames 1..nframes with the envelope D(k) and the state at the frames in `marks` (chunk ends).
    status / chi2: (nframes + 1, CHECKS), row k = frame k."""

    def __init__(self, inputs, nframes, marks, fault=None, fault_frame=None, envelope=True):
        marks = sorted(set(int(k) for k in marks if 1 <= k <= nframes))
        runs = {"plain": FilterReplay(inputs, fault=fault, fault_frame=fault_frame)}
        if envelope:
            runs["first"] = FilterReplay(inputs, push="first")
            runs["every"] = FilterReplay(inputs, push="every")
        self.nframes, self.marks = nframes, marks
        self.status = np.full((nframes + 1, bench.CHECKS), -1, np.int32)
        self.chi2 = np.full((nframes + 1, bench.CHECKS), np.nan)
        self.m, self.P, self.D = {}, {}, {}
        for k in range(1, nframes + 1):
            self.status[k], self.chi2[k] = runs["plain"].step()
            for name in ("first", "every"):
                if name in runs:
                    runs[name].step()
            if k in marks:
                self.m[k], self.P[k] = runs["plain"].o.download()
                if envelope:
                    d = [distance(self.m[k], self.P[k], *runs[name].o.download()) for name in ("first", "every")]
                    self.D[k] = (max(d[0][0], d[1][0]), max(d[0][1], d[1][1]))
        for r in runs.values():
            r.close()

    def gate(self, k, m, P, c=C_ENVELOPE):
        """(ok, ratio_m, ratio_P, dist_m, dist_P) of a device state at frame k against the plain replay and c D(k)."""
        dm, dP = distance(self.m[k], self.P[k], m, P)
        Dm, DP = self.D[k]
        rm, rP = dm / max(Dm, FLOOR / c), dP / max(DP, FLOOR / c)
        return bool(rm <= c and rP <= c and np.isfinite(m).all() and np.isfinite(P).all()), rm, rP, dm, dP


def tracker_replay(inputs, k, lk=None, stale_pyramid=False):
    """Pyramids and LK of frame k (the last frame of a chunk). Returns a dict with "pyr" ([camera][level] -> (gray, deriv),
    unpadded), "lk_next_temporal", "lk_next_stereo" (stereo configs), "lk_status", "lk_track_status" (those of the last LK
    call of the frame, as the device buffers hold them). stale_pyramid: the LK calls read the pyramids of the frame before."""
    lk = lk or lk_oracle.OracleLK()
    j, prev_j = bench.frame_index(k), bench.frame_index(k - 1)
    frames = inputs.frames
    img = lambda jj, c: np.ascontiguousarray(frames[jj, c].cpu().numpy() if hasattr(frames, "cpu") else frames[jj, c])
    cur = [lk.pyramid(img(j, c), bench.WIN, bench.MAXLEVEL) for c in range(bench.NCAM)]
    prev = lk.pyramid(img(prev_j, 0), bench.WIN, bench.MAXLEVEL)
    src = [lk.pyramid(img(prev_j, c), bench.WIN, bench.MAXLEVEL) for c in range(bench.NCAM)] if stale_pyramid else cur
    out = {"pyr": [[p.download(lv, padded=False) for lv in range(p.levels)] for p in cur]}
    kw = dict(max_level=bench.MAXLEVEL, max_iter=20, eps=0.03, min_eig=1e-3, accum_mode=1)
    nxt, st, ts = lk.lk(prev, src[0], inputs.points, inputs.init_guess(prev_j, j), **kw)
    out["lk_next_temporal"] = nxt
    if bench.STEREO:
        nxt2, st, ts = lk.lk(src[0], src[1], nxt, None, **kw)
        out["lk_next_stereo"] = nxt2
    out["lk_status"], out["lk_track_status"] = st, ts
    for p in set(cur + [prev] + src):
        p.free()
    return out


def tracker_mismatches(ref, got):
    """Names of the tracker outputs in `got` that are not bit-identical to `ref` (keys missing from `got` are not compared)."""
    bad = []
    if "pyr" in got:
        for c, levels in enumerate(ref["pyr"]):
            for lv, (g, d) in enumerate(levels):
                gg, gd = got["pyr"][c][lv]
                if not np.array_equal(g, gg):
                    bad.append(f"pyr[{c}][{lv}].gray")
                if not np.array_equal(d, gd):
                    bad.append(f"pyr[{c}][{lv}].deriv")
    for key in ("lk_next_temporal", "lk_next_stereo"):
        if key in got and key in ref and not np.array_equal(np.asarray(ref[key], np.float32).view(np.uint32),
                                                            np.ascontiguousarray(got[key], np.float32).view(np.uint32)):
            bad.append(key)
    for key in ("lk_status", "lk_track_status"):
        if key in got and not np.array_equal(np.asarray(ref[key]).astype(np.int64), np.asarray(got[key]).astype(np.int64)):
            bad.append(key)
    return bad


def check_mismatches(replay, k, status, chi2):
    """The frame-k check decisions must be identical and chi2 within CHI2_RTOL."""
    bad = []
    status = np.asarray(status)[:bench.CHECKS].astype(np.int64)
    chi2 = np.asarray(chi2, np.float64)[:bench.CHECKS]
    if not np.array_equal(status, replay.status[k].astype(np.int64)):
        bad.append(f"check status at frame {k}: {status.tolist()} != {replay.status[k].tolist()}")
    rel = np.abs(chi2 - replay.chi2[k]) / np.abs(replay.chi2[k])
    if not (np.isfinite(rel).all() and rel.max() <= CHI2_RTOL):
        bad.append(f"chi2 at frame {k}: relative difference {np.nanmax(rel):.3g}")
    return bad


def chunk_ends(chunks):
    return list(np.cumsum(chunks))


def chunk_schedule(total, lengths=(1, 2, 3, 7, 16, 64)):
    """Chunk lengths cycling through `lengths` that add up to `total` (the last one cut short)."""
    out, i = [], 0
    while sum(out) < total:
        out.append(min(lengths[i % len(lengths)], total - sum(out)))
        i += 1
    return out
