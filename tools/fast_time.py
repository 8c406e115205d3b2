"""Device time of FAST corner detection (csrc/fast.cu) on 752 x 480 frames, and cv2.FAST's host time as a rough guide.

  * per frame: hv_fast_detect_device (its two launches: mark + count, then scan + scatter) from CUDA events around 400 back-to-back
    calls on the context's stream, for thresholds 10 / 20 with suppression and 10 without; the keypoint count of the frame beside it;
  * the host call hv_fast_detect end to end (host clock, it synchronises), median of 200;
  * S sessions: S per-session hv_fast_detect_device calls against one hv_fast_detect_batch_device, alternating in one process, each
    behind a short sleep kernel so that the events time the device and not the host's issue rate; medians over the repetitions after
    warm-up. The outputs of the two ways are compared byte for byte after the last repetition;
  * cv2.FastFeatureDetector on the host with IPP off and on (median of 50): a rough guide only, on whatever CPU runs the script.
Prints a header line with the GPU's name and power limit, then one JSON line per measurement.

    python tools/fast_time.py [--reps 30] [--sizes 1,2,4,8,16,32,64] [--out results.jsonl]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

W, H, WARMUP, CAP = 752, 480, 5, 8192


def gpu_info():
    import torch
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
        out["power_limit_and_max_sm_clock"] = q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unavailable"
    except (OSError, subprocess.TimeoutExpired):
        out["power_limit_and_max_sm_clock"] = "unavailable"
    return out


def _buffers(S):
    import torch
    return [(torch.zeros((CAP, 2), dtype=torch.float32, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda"),
             torch.zeros(CAP, dtype=torch.float32, device="cuda")) for _ in range(S)]


def per_frame(hv, stream, pyr, threshold, nonmax, n=400):
    import torch
    (xy, cnt, resp), = _buffers(1)
    call = lambda: hv.lib.hv_fast_detect_device(hv.h, pyr.h, threshold, int(nonmax), xy.data_ptr(), resp.data_ptr(), CAP, cnt.data_ptr())
    for _ in range(20):
        call()
    hv.sync()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(n):
        call()
    e1.record(stream)
    e1.synchronize()
    dev_us = e0.elapsed_time(e1) * 1e3 / n
    xs = np.zeros((CAP, 2), np.float32)
    c = ctypes.c_int()
    host = []
    for i in range(200 + WARMUP):
        t0 = time.perf_counter()
        hv.lib.hv_fast_detect(hv.h, pyr.h, threshold, int(nonmax), xs.ctypes.data, None, CAP, ctypes.byref(c))
        if i >= WARMUP:
            host.append((time.perf_counter() - t0) * 1e6)
    return {"what": "per_frame", "threshold": threshold, "nonmax": nonmax, "keypoints": c.value, "device_us_per_call": round(dev_us, 2),
            "host_call_us_median": round(float(np.median(host)), 1)}


def batch_vs_sessions(hv, stream, frames, S, reps, threshold=10, nonmax=True):
    import torch
    from hybvio_b200 import capi
    pyrs = []
    for j in range(S):
        p = hv.pyramid(W, H, 31, 0)
        p.build(frames[j % len(frames)])
        pyrs.append(p)
    single, batch = _buffers(S), _buffers(S)
    jobs = [capi.fast_job(pyrs[j], *batch[j][:2], batch[j][2]) for j in range(S)]
    lib = hv.lib
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    t_single, t_batch = [], []
    for r in range(reps + WARMUP):
        torch.cuda._sleep(2_000_000)
        ev[0].record(stream)
        for p, (xy, cnt, resp) in zip(pyrs, single):
            lib.hv_fast_detect_device(hv.h, p.h, threshold, int(nonmax), xy.data_ptr(), resp.data_ptr(), CAP, cnt.data_ptr())
        ev[1].record(stream)
        torch.cuda._sleep(2_000_000)
        ev[2].record(stream)
        hv.fast_detect_batch_device(jobs, threshold, nonmax)
        ev[3].record(stream)
        ev[3].synchronize()
        if r >= WARMUP:
            t_single.append(ev[0].elapsed_time(ev[1]) * 1e3)
            t_batch.append(ev[2].elapsed_time(ev[3]) * 1e3)
    same = all(a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes() for s, b_ in zip(single, batch) for a, b in zip(s, b_))
    for p in pyrs:
        p.release()
    ms, mb = float(np.median(t_single)), float(np.median(t_batch))
    return {"what": "sessions", "S": S, "threshold": threshold, "nonmax": nonmax, "per_session_us": round(ms, 1), "batch_us": round(mb, 1),
            "speedup": round(ms / mb, 2), "launches_per_session_way": 2 * S, "launches_batch": 2, "outputs_identical": same}


def cv2_host(frame):
    try:
        import cv2
    except ImportError:
        return [{"what": "cv2_host", "note": "cv2 not installed"}]
    out = []
    old = cv2.ipp.useIPP()
    for ipp in (False, True):
        cv2.ipp.setUseIPP(ipp)
        det = cv2.FastFeatureDetector_create(10, True, cv2.FAST_FEATURE_DETECTOR_TYPE_9_16)
        ts = []
        for i in range(50 + WARMUP):
            t0 = time.perf_counter()
            kp = det.detect(frame)
            if i >= WARMUP:
                ts.append((time.perf_counter() - t0) * 1e6)
        out.append({"what": "cv2_host", "ipp": ipp, "threshold": 10, "nonmax": True, "keypoints": len(kp), "host_us_median": round(float(np.median(ts)), 1),
                    "cpu_count": os.cpu_count()})
    cv2.ipp.setUseIPP(old)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--sizes", default="1,2,4,8,16,32,64")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from hybvio_b200 import capi, synth
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: this tool measures device time only")
    info = gpu_info()
    print("# " + json.dumps(info), flush=True)
    hv = capi.Context(0)
    stream = torch.cuda.ExternalStream(hv.stream)
    frames = [np.ascontiguousarray(synth.stereo_frame(k, W, H)[0]) for k in range(8)]
    rows = []
    pyr = hv.pyramid(W, H, 31, 0)
    pyr.build(frames[0])
    for t, nms in ((10, True), (20, True), (10, False)):
        rows.append(per_frame(hv, stream, pyr, t, nms))
        print(json.dumps(rows[-1]), flush=True)
    pyr.release()
    for S in [int(s) for s in args.sizes.split(",")]:
        rows.append(batch_vs_sessions(hv, stream, frames, S, args.reps))
        print(json.dumps(rows[-1]), flush=True)
    for r in cv2_host(frames[0]):
        rows.append(r)
        print(json.dumps(r), flush=True)
    hv.close()
    if args.out:
        with open(args.out, "w") as f:
            f.write(json.dumps({"gpu": info}) + "\n")
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
