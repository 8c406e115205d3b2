"""Time of the absolute-pose RANSAC (csrc/pnp.cu, cv::solvePnPRansac with SOLVEPNP_P3P) on seeded scenes (tests/pnp_common.py:
EuRoC-like K, sideways motion, near depths, 0.5 px noise), and cv2.solvePnPRansac's host time as a rough guide.

  * per call: hv_solve_pnp_ransac_device from CUDA events around back-to-back calls on the context's stream (median of 9 windows of
    20 calls), for m in {150, 300, 600, 4096} at 10 / 30 / 50 % outliers, 100 iterations, reprojection error 8, confidence 0.99; also
    the host call hv_solve_pnp_ransac end to end (host clock, it synchronises; median of 30);
  * 64 sessions (m = 300, 30 % outliers): one hv_solve_pnp_ransac_batch_device against 64 hv_solve_pnp_ransac_device calls,
    alternating, each behind a short sleep kernel; medians over the repetitions; outputs compared byte for byte;
  * cv2.solvePnPRansac on the host (median of 10): a rough guide only, on whatever CPU runs the script.
Prints a header line with the GPU's name and power limit, then one JSON line per measurement.

    python tools/pnp_time.py [--out results.jsonl]
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

import pnp_common as pc  # noqa: E402
from essential_time import event_time, gpu_info  # noqa: E402

KK = (pc.FX, pc.FY, pc.CX, pc.CY)


def buffers(X, x):
    import torch
    n = X.shape[0]
    return {"xyz": torch.from_numpy(X).cuda(), "xy": torch.from_numpy(x).cuda(), "r": torch.zeros(3, dtype=torch.float64, device="cuda"),
            "t": torch.zeros(3, dtype=torch.float64, device="cuda"), "mask": torch.zeros(n, dtype=torch.uint8, device="cuda"),
            "inl": torch.zeros(1, dtype=torch.int32, device="cuda"), "ok": torch.zeros(1, dtype=torch.int32, device="cuda")}


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
    it, thr, conf = 100, 8.0, 0.99
    for m in (150, 300, 600, 4096):
        for outl in (0.1, 0.3, 0.5):
            X, x, _, _ = pc.scene(np.random.default_rng(m + int(100 * outl)), m, outl, 0.5, "side", "near")
            b = buffers(X, x)
            call = lambda: hv.solve_pnp_ransac_device(b["xyz"], b["xy"], b["r"], b["t"], b["mask"], b["inl"], b["ok"], *KK, it, thr, conf)
            dev_us = event_time(call)
            hs = []
            for _ in range(30):
                t0 = time.perf_counter()
                hv.solve_pnp_ransac(X, x, *KK, it, thr, conf)
                hs.append((time.perf_counter() - t0) * 1e6)
            d = {"m": m, "outliers": outl, "inliers": int(b["inl"].item()), "device_us_per_call": round(dev_us, 1),
                 "host_call_us": round(float(np.median(hs)), 1)}
            if cv2 is not None:
                cs = []
                for _ in range(10):
                    t0 = time.perf_counter()
                    cv2.solvePnPRansac(X, x, pc.K, None, iterationsCount=it, reprojectionError=thr, confidence=conf, flags=cv2.SOLVEPNP_P3P)
                    cs.append((time.perf_counter() - t0) * 1e6)
                d["cv2_host_us_rough_guide"] = round(float(np.median(cs)), 1)
            emit(d)

    S = 64
    scenes = [pc.scene(np.random.default_rng(5000 + j), 300, 0.3, 0.5, "side", "near")[:2] for j in range(S)]
    bb = [buffers(*s) for s in scenes]
    bs = [buffers(*s) for s in scenes]
    jobs = [capi.pnp_job(q["xyz"], q["xy"], q["r"], q["t"], q["mask"], q["inl"], q["ok"], *KK) for q in bb]

    def batch():
        hv.solve_pnp_ransac_batch_device(jobs, it, thr, conf)

    def singles():
        for q in bs:
            hv.solve_pnp_ransac_device(q["xyz"], q["xy"], q["r"], q["t"], q["mask"], q["inl"], q["ok"], *KK, it, thr, conf)

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
    same = all(torch.equal(p[k], q[k]) for p, q in zip(bb, bs) for k in ("r", "t", "mask", "inl", "ok"))
    emit({"sessions": S, "m": 300, "batch_us": round(float(np.median(tb)), 1), "per_session_calls_us": round(float(np.median(tsg)), 1),
          "outputs_identical": bool(same)})
    hv.close()


if __name__ == "__main__":
    main()
