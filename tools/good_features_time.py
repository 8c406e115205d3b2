"""Device time of Shi-Tomasi corner detection (csrc/good_features.cu) on 752 x 480 frames, and cv2.goodFeaturesToTrack's host time as a
rough guide.

  * per frame: hv_good_features_device (its three launches: response + max, candidates, select) from CUDA events around 200
    back-to-back calls on the context's stream, for the typical parameters (quality 0.01, max_corners 150, min_distance 10 and 20) and
    the worst cases (raw noise at quality 1e-4, a periodic pattern of equal responses; budgets above the candidate count); the candidate
    count and the list length beside each. Also the host call hv_good_features end to end (host clock, it synchronises), median of 100;
  * S sessions: S per-session hv_good_features_device calls against one hv_good_features_batch_device, alternating in one process, each
    behind a short sleep kernel so that the events time the device and not the host's issue rate; medians over the repetitions after
    warm-up. The outputs of the two ways are compared byte for byte after the last repetition;
  * the split of the typical call's device time between its three kernels (torch.profiler, 50 calls, in a run of its own);
  * cv2.goodFeaturesToTrack on the host with its defaults (median of 30): a rough guide only, on whatever CPU runs the script.
Prints a header line with the GPU's name and power limit, then one JSON line per measurement.

    python tools/good_features_time.py [--reps 30] [--sizes 1,2,4,8,16,32,64] [--out results.jsonl]
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

W, H, WARMUP = 752, 480, 5


def gpu_info():
    import torch
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
        out["power_limit_and_max_sm_clock"] = q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unavailable"
    except (OSError, subprocess.TimeoutExpired):
        out["power_limit_and_max_sm_clock"] = "unavailable"
    return out


def _buffers(S, cap):
    import torch
    return [(torch.zeros((cap, 2), dtype=torch.float32, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda"),
             torch.zeros(cap, dtype=torch.float32, device="cuda")) for _ in range(S)]


def candidates(orc, img, q):
    """the candidate count: the list without a distance filter or budget"""
    return len(orc.detect(img, 1 << 30, q, 0.0))


def per_frame(hv, stream, orc, name, img, mc, q, md, n=200):
    import torch
    pyr = hv.pyramid(W, H, 31, 0)
    pyr.build(img)
    (xy, cnt, resp), = _buffers(1, mc)
    call = lambda: hv.lib.hv_good_features_device(hv.h, pyr.h, 3, mc, q, md, None, 0, xy.data_ptr(), resp.data_ptr(), mc, cnt.data_ptr())
    for _ in range(10):
        call()
    hv.sync()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(n):
        call()
    e1.record(stream)
    e1.synchronize()
    dev_us = e0.elapsed_time(e1) * 1e3 / n
    count = int(cnt.cpu().numpy()[0])
    xs = np.zeros((mc, 2), np.float32)
    c = ctypes.c_int()
    host = []
    for i in range(100 + WARMUP):
        t0 = time.perf_counter()
        hv.lib.hv_good_features(hv.h, pyr.h, 3, mc, q, md, None, 0, xs.ctypes.data, None, mc, ctypes.byref(c))
        if i >= WARMUP:
            host.append((time.perf_counter() - t0) * 1e6)
    pyr.release()
    return {"what": "per_frame", "image": name, "quality": q, "min_distance": md, "max_corners": mc, "candidates": candidates(orc, img, q),
            "corners": count, "device_us_per_call": round(dev_us, 1), "host_call_us_median": round(float(np.median(host)), 1)}


def batch_vs_sessions(hv, stream, frames, S, reps, q=0.01, md=10.0, mc=150):
    import torch
    from hybvio_b200 import capi
    pyrs = []
    for j in range(S):
        p = hv.pyramid(W, H, 31, 0)
        p.build(frames[j % len(frames)])
        pyrs.append(p)
    single, batch = _buffers(S, mc), _buffers(S, mc)
    jobs = [capi.good_features_job(pyrs[j], batch[j][0], batch[j][1], mc, batch[j][2]) for j in range(S)]
    lib = hv.lib
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    t_single, t_batch = [], []
    for r in range(reps + WARMUP):
        torch.cuda._sleep(2_000_000)
        ev[0].record(stream)
        for p, (xy, cnt, resp) in zip(pyrs, single):
            lib.hv_good_features_device(hv.h, p.h, 3, mc, q, md, None, 0, xy.data_ptr(), resp.data_ptr(), mc, cnt.data_ptr())
        ev[1].record(stream)
        torch.cuda._sleep(2_000_000)
        ev[2].record(stream)
        hv.good_features_batch_device(jobs, q, md)
        ev[3].record(stream)
        ev[3].synchronize()
        if r >= WARMUP:
            t_single.append(ev[0].elapsed_time(ev[1]) * 1e3)
            t_batch.append(ev[2].elapsed_time(ev[3]) * 1e3)
    same = all(a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes() for s, b_ in zip(single, batch) for a, b in zip(s, b_))
    for p in pyrs:
        p.release()
    ms, mb = float(np.median(t_single)), float(np.median(t_batch))
    return {"what": "sessions", "S": S, "quality": q, "min_distance": md, "max_corners": mc, "per_session_us": round(ms, 1),
            "batch_us": round(mb, 1), "speedup": round(ms / mb, 2), "launches_per_session_way": 3 * S, "launches_batch": 3,
            "outputs_identical": same}


def kernel_split(hv, frame, n=50, mc=150, q=0.01, md=10.0):
    """Mean device time per call of each kernel of hv_good_features_device (torch.profiler with CUDA activities)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    pyr = hv.pyramid(W, H, 31, 0)
    pyr.build(frame)
    (xy, cnt, resp), = _buffers(1, mc)
    call = lambda: hv.lib.hv_good_features_device(hv.h, pyr.h, 3, mc, q, md, None, 0, xy.data_ptr(), resp.data_ptr(), mc, cnt.data_ptr())
    for _ in range(10):
        call()
    hv.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            call()
        hv.sync()
    out = {}
    for e in prof.key_averages():
        if "hv_gf_" in e.key:
            name = e.key.split("(")[0].replace("void ", "")
            t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            out[name] = round(t / n, 1)
    pyr.release()
    return {"what": "kernel_split", "quality": q, "min_distance": md, "max_corners": mc, "device_us_per_call": out}


def cv2_host(frame):
    try:
        import cv2
    except ImportError:
        return [{"what": "cv2_host", "note": "cv2 not installed"}]
    out = []
    for md in (10.0, 20.0):
        ts = []
        for i in range(30 + WARMUP):
            t0 = time.perf_counter()
            c = cv2.goodFeaturesToTrack(frame, 150, 0.01, md, blockSize=3)
            if i >= WARMUP:
                ts.append((time.perf_counter() - t0) * 1e6)
        out.append({"what": "cv2_host", "cv2": cv2.__version__, "quality": 0.01, "min_distance": md, "max_corners": 150,
                    "corners": 0 if c is None else len(c), "host_us_median": round(float(np.median(ts)), 1), "cpu_count": os.cpu_count()})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--sizes", default="1,2,4,8,16,32,64")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from hybvio_b200 import capi, synth
    from oracle import good_features_oracle
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: this tool measures device time only")
    info = gpu_info()
    print("# " + json.dumps(info), flush=True)
    orc = good_features_oracle.OracleGoodFeatures()
    hv = capi.Context(0)
    stream = torch.cuda.ExternalStream(hv.stream)
    frames = [np.ascontiguousarray(synth.stereo_frame(k, W, H)[0]) for k in range(8)]
    noise = np.random.RandomState(21).randint(0, 256, (H, W)).astype(np.uint8)
    y, x = np.mgrid[0:H, 0:W]
    periodic = np.where(((x // 4) + (y // 4)) % 2 == 1, 200, 50).astype(np.uint8)
    rows = []
    cases = [("frame", frames[0], 150, 0.01, 10.0), ("frame", frames[0], 150, 0.01, 20.0),
             ("frame", frames[0], 100000, 0.01, 10.0), ("noise", noise, 150, 1e-4, 10.0), ("noise", noise, 100000, 1e-4, 30.0),
             ("noise", noise, 100000, 1e-4, 0.0), ("periodic", periodic, 100000, 0.01, 2.5), ("periodic", periodic, 150, 0.01, 10.0)]
    for name, img, mc, q, md in cases:
        rows.append(per_frame(hv, stream, orc, name, img, mc, q, md))
        print(json.dumps(rows[-1]), flush=True)
    for S in [int(s) for s in args.sizes.split(",")]:
        rows.append(batch_vs_sessions(hv, stream, frames, S, args.reps))
        print(json.dumps(rows[-1]), flush=True)
    rows.append(kernel_split(hv, frames[0]))
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
