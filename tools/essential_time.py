"""Time of the essential-matrix RANSAC (csrc/essential.cu) on seeded two-view scenes (tests/essential_common.py: EuRoC-like K, sideways
motion, 0.5 px noise, outliers uniform in the image), and cv2.findEssentialMat's host time as a rough guide.

  * per call: hv_find_essential_device from CUDA events around back-to-back calls on the context's stream (median of 9 windows of 20
    calls), for m in {150, 300, 600} at outlier ratios 0.1, 0.3 and 0.5, prob 0.999, threshold 1 px, max_iters 1000; the number of
    RANSAC iterations the call ran beside it (the oracle's replay). Also the host call hv_find_essential end to end (host clock, it
    synchronises; median of 50);
  * 64 sessions: one hv_find_essential_batch_device against 64 hv_find_essential_device calls, alternating, each behind a short sleep
    kernel so that the events time the device and not the host's issue rate; medians over the repetitions. The outputs of the two ways
    are compared byte for byte;
  * cv2.findEssentialMat(..., cv2.RANSAC, 0.999, 1.0) on the host with its defaults (median of 10): a rough guide only, on whatever CPU
    runs the script.
Prints a header line with the GPU's name and power limit, then one JSON line per measurement.

    python tools/essential_time.py [--out results.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import essential_common as ec  # noqa: E402


def gpu_info():
    import torch
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
        out["power_limit_and_max_sm_clock"] = q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unavailable"
    except (OSError, subprocess.TimeoutExpired):
        out["power_limit_and_max_sm_clock"] = "unavailable"
    return out


def buffers(p1, p2):
    import torch
    n = p1.shape[0]
    return {"xy1": torch.from_numpy(p1).cuda(), "xy2": torch.from_numpy(p2).cuda(), "E": torch.zeros(90, dtype=torch.float64, device="cuda"),
            "nsol": torch.zeros(1, dtype=torch.int32, device="cuda"), "mask": torch.zeros(n, dtype=torch.uint8, device="cuda"),
            "inl": torch.zeros(1, dtype=torch.int32, device="cuda")}


def iterations(orc, p1, p2, prob, thr, mi):
    """the number of iterations the loop runs (the oracle's subsets replayed through the acceptance rule)"""
    q, _ = orc.compact(p1, p2, ec.FX, ec.FY, ec.CX, ec.CY)
    sub = orc.subsets(len(q), mi)
    ns, _, err = orc.hypotheses(q, sub)
    niters, good, it, m = mi, 0, 0, len(q)
    t = thr / ((ec.FX + ec.FY) / 2.0)
    t2 = np.float32(t * t)
    while it < niters:
        for r in range(ns[it]):
            c = int((err[it, r].astype(np.float32) <= t2).sum())
            if c > max(good, 4):
                good, niters = c, orc.update_niters(prob, (m - c) / m, niters)
        it += 1
    return it


def event_time(fn, calls=20, windows=9):
    import torch
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(windows):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(calls):
            fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) * 1e3 / calls)
    return float(np.median(ts))


def main():
    import torch
    from hybvio_b200 import capi
    from oracle.essential_oracle import OracleEssential
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
    orc = OracleEssential()
    try:
        import cv2
    except ImportError:
        cv2 = None
    prob, thr, mi = 0.999, 1.0, 1000
    for m in (150, 300, 600):
        for outl in (0.1, 0.3, 0.5):
            p1, p2 = ec.scene(np.random.default_rng(m + int(100 * outl)), m, outl, 0.5, "side")
            b = buffers(p1, p2)
            call = lambda: hv.find_essential_device(b["xy1"], b["xy2"], b["E"], b["nsol"], b["mask"], b["inl"], ec.FX, ec.FY, ec.CX, ec.CY,
                                                    prob, thr, mi)
            dev_us = event_time(call)
            hs = []
            for _ in range(50):
                t0 = time.perf_counter()
                hv.find_essential(p1, p2, ec.FX, ec.FY, ec.CX, ec.CY, prob, thr, mi)
                hs.append((time.perf_counter() - t0) * 1e6)
            d = {"m": m, "outliers": outl, "iterations": iterations(orc, p1, p2, prob, thr, mi), "inliers": int(b["inl"].item()),
                 "device_us_per_call": round(dev_us, 1), "host_call_us": round(float(np.median(hs)), 1)}
            if cv2 is not None:
                cs = []
                for _ in range(10):
                    t0 = time.perf_counter()
                    cv2.findEssentialMat(p1, p2, ec.K, cv2.RANSAC, prob, thr, mi)
                    cs.append((time.perf_counter() - t0) * 1e6)
                d["cv2_host_us_rough_guide"] = round(float(np.median(cs)), 1)
            emit(d)

    # 64 sessions: one batch against 64 per-session calls
    S = 64
    rng = np.random.default_rng(7)
    scenes = [ec.scene(rng, 300, [0.1, 0.3, 0.5][j % 3], 0.5, "side") for j in range(S)]
    bb = [buffers(*s) for s in scenes]
    bs = [buffers(*s) for s in scenes]
    jobs = [capi.essential_job(x["xy1"], x["xy2"], x["E"], x["nsol"], x["mask"], x["inl"], ec.FX, ec.FY, ec.CX, ec.CY) for x in bb]

    def batch():
        hv.find_essential_batch_device(jobs, prob, thr, mi)

    def singles():
        for x in bs:
            hv.find_essential_device(x["xy1"], x["xy2"], x["E"], x["nsol"], x["mask"], x["inl"], ec.FX, ec.FY, ec.CX, ec.CY, prob, thr, mi)

    tb, tsg = [], []
    for _ in range(3):
        batch(); singles()
    torch.cuda.synchronize()
    for _ in range(15):
        for fn, acc in ((batch, tb), (singles, tsg)):
            a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda._sleep(2_000_000)
            a.record()
            fn()
            e.record()
            e.synchronize()
            acc.append(a.elapsed_time(e) * 1e3)
    same = all(torch.equal(x[k], y[k]) for x, y in zip(bb, bs) for k in ("E", "nsol", "mask", "inl"))
    emit({"sessions": S, "m": 300, "outliers": "0.1/0.3/0.5", "batch_us": round(float(np.median(tb)), 1),
          "per_session_calls_us": round(float(np.median(tsg)), 1), "outputs_identical": bool(same)})
    hv.close()


if __name__ == "__main__":
    main()
