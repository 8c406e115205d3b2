"""Time of the two-view triangulation (csrc/triangulate.cu, cv::triangulatePoints + convertPointsFromHomogeneous) on seeded rectified
stereo points (tests/triangulate_common.py: f = 450, B = 0.11 m, 0.5 px noise), with cv2.triangulatePoints' host time as a rough guide.

  * per call, n in {150, 300, 600, 4096, 65536}: hv_triangulate_points_device writing X4, xyz and used, after warm-up.
      - queued: CUDA events around 200 back-to-back calls issued behind a sleep kernel longer than their issue from Python, so the
        queue never runs dry and the events time the device, launch gaps included (median of 5 windows; the host's issue time per call
        is reported beside it, and the window is flagged if the issue outlasted the sleep);
      - alone: CUDA events around one call behind a sleep kernel (median of 200 launches);
      - host call: hv_triangulate_points end to end (host clock; it copies both ways and synchronises; median of 50);
  * 64 sessions of 300 points: one hv_triangulate_points_batch_device against 64 hv_triangulate_points_device calls, alternating, each
    behind a sleep kernel longer than their issue (median of 200 repetitions). The outputs of the two ways are compared byte for byte;
  * cv2.triangulatePoints on the host CPU (median of up to 20): a rough guide only, on whatever CPU runs the script.
Prints a header line with the GPU's name and power limit, then one JSON line per measurement.

    python tools/triangulate_time.py [--out results.jsonl]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402

import triangulate_common as tc  # noqa: E402
from essential_time import gpu_info  # noqa: E402

SLEEP_CYCLES = 2_000_000          # ~1 ms at 1.98 GHz: longer than issuing one call
LONG_SLEEP_CYCLES = 60_000_000    # ~30 ms: longer than issuing 200 calls (or 64) from Python


def buffers(a, b):
    import torch
    n = a.shape[0]
    return {"xy1": torch.from_numpy(a).cuda(), "xy2": torch.from_numpy(b).cuda(), "X4": torch.zeros(4 * n, dtype=torch.float32, device="cuda"),
            "xyz": torch.zeros((n, 3), dtype=torch.float32, device="cuda"), "used": torch.zeros(n, dtype=torch.uint8, device="cuda")}


def timed(fn, reps=1, cycles=SLEEP_CYCLES):
    """(device time (us) of `reps` calls of fn, host issue time (us) of them, whether the issue ended before the sleep did): the calls
    are issued behind a sleep kernel so that the events time the device and not the host's issue rate"""
    import torch
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s0.record()
    torch.cuda._sleep(cycles)
    s1.record()
    a.record()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    issue = (time.perf_counter() - t0) * 1e6
    e.record()
    e.synchronize()
    return a.elapsed_time(e) * 1e3, issue, issue < s0.elapsed_time(s1) * 1e3


def main():
    import torch
    from hybvio_b200 import capi
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    out = open(args.out, "w") if args.out else None

    def emit(d):
        line = json.dumps(d)
        print(line, flush=True)
        if out:
            out.write(line + "\n")

    emit({"gpu": gpu_info()})
    hv = capi.Context(0, stream=torch.cuda.current_stream().cuda_stream)
    try:
        import cv2
    except ImportError:
        cv2 = None

    for n in (150, 300, 600, 4096, 65536):
        P1, P2, a, b = tc.rectified(n, n)
        d = buffers(a, b)
        call = lambda: hv.triangulate_points_device(P1, P2, d["xy1"], d["xy2"], d["X4"], d["xyz"], d["used"])   # noqa: E731
        for _ in range(20):
            call()
        torch.cuda.synchronize()
        q = [timed(call, 200, LONG_SLEEP_CYCLES) for _ in range(5)]
        queued = float(np.median([x[0] / 200 for x in q]))
        alone = float(np.median([timed(call)[0] for _ in range(200)]))
        hs = []
        for _ in range(50):
            t0 = time.perf_counter()
            hv.triangulate_points(P1, P2, a, b)
            hs.append((time.perf_counter() - t0) * 1e6)
        r = {"n": n, "device_us_per_call_queued": round(queued, 2), "host_issue_us_per_call": round(float(np.median([x[1] / 200 for x in q])), 2),
             "queue_stayed_full": all(x[2] for x in q), "device_us_one_call": round(alone, 2), "host_call_us": round(float(np.median(hs)), 1)}
        if cv2 is not None:
            cs = []
            at, bt = np.ascontiguousarray(a.T), np.ascontiguousarray(b.T)
            for _ in range(20 if n <= 4096 else 5):
                t0 = time.perf_counter()
                cv2.triangulatePoints(P1, P2, at, bt)
                cs.append((time.perf_counter() - t0) * 1e6)
            r["cv2_host_us_rough_guide"] = round(float(np.median(cs)), 1)
        emit(r)

    # 64 sessions: one batch against 64 per-session calls
    S, n = 64, 300
    scenes = []
    for j in range(S):
        k = np.array([[tc.F * (1 + 0.002 * j), 0, tc.CX], [0, tc.F, tc.CY], [0, 0, 1]])
        P1, P2 = tc.stereo_pair(tc.B, k)
        rng = np.random.default_rng(2000 + j)
        X = tc.cloud(rng, n)
        scenes.append((P1, P2, tc.project(P1, X, rng, 0.5), tc.project(P2, X, rng, 0.5)))
    bb = [buffers(s[2], s[3]) for s in scenes]
    bs = [buffers(s[2], s[3]) for s in scenes]
    jobs = [capi.triangulate_job(s[0], s[1], x["xy1"], x["xy2"], x["X4"], x["xyz"], x["used"]) for s, x in zip(scenes, bb)]

    def batch():
        hv.triangulate_points_batch_device(jobs)

    def singles():
        for s, x in zip(scenes, bs):
            hv.triangulate_points_device(s[0], s[1], x["xy1"], x["xy2"], x["X4"], x["xyz"], x["used"])

    for _ in range(5):
        batch(); singles()
    torch.cuda.synchronize()
    tb, tsg = [], []
    for _ in range(200):
        tb.append(timed(batch))
        tsg.append(timed(singles, 1, LONG_SLEEP_CYCLES))
    same = all(torch.equal(x[k], y[k]) for x, y in zip(bb, bs) for k in ("X4", "xyz", "used"))
    emit({"sessions": S, "n": n, "batch_us": round(float(np.median([x[0] for x in tb])), 2),
          "per_session_calls_us": round(float(np.median([x[0] for x in tsg])), 2),
          "per_session_calls_host_issue_us": round(float(np.median([x[1] for x in tsg])), 1),
          "queue_stayed_full": all(x[2] for x in tb + tsg), "outputs_identical": bool(same)})
    hv.close()


if __name__ == "__main__":
    main()
