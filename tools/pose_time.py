"""Time of the relative pose (csrc/pose.cu, cv::recoverPose) on seeded two-view scenes (tests/essential_common.py: EuRoC-like K,
sideways motion, 0.5 px noise, 10 % outliers), with E and the inlier mask from the essential oracle, and cv2.recoverPose's host time as a
rough guide.

  * per call: hv_recover_pose_device from CUDA events around back-to-back calls on the context's stream (median of 9 windows of 20
    calls), for m in {150, 300, 600, 4096}, distance_thresh 50, with the inlier mask; also the host call hv_recover_pose end to end
    (host clock, it synchronises; median of 50);
  * 64 sessions (m = 300): one hv_recover_pose_batch_device against 64 hv_recover_pose_device calls, alternating, each behind a short
    sleep kernel so that the events time the device and not the host's issue rate; medians over the repetitions. The outputs of the
    two ways are compared byte for byte;
  * cv2.recoverPose(E, p1, p2, K, mask=...) on the host (median of 10): a rough guide only, on whatever CPU runs the script.
Prints a header line with the GPU's name and power limit, then one JSON line per measurement.

    python tools/pose_time.py [--out results.jsonl]
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

import essential_common as ec  # noqa: E402
from essential_time import event_time, gpu_info  # noqa: E402


def buffers(p1, p2, Ecm, mask):
    import torch
    n = p1.shape[0]
    return {"xy1": torch.from_numpy(p1).cuda(), "xy2": torch.from_numpy(p2).cuda(), "E": torch.from_numpy(np.ascontiguousarray(Ecm)).cuda(),
            "mask": torch.from_numpy(np.ascontiguousarray(mask, np.uint8)).cuda(), "R": torch.zeros(9, dtype=torch.float64, device="cuda"),
            "t": torch.zeros(3, dtype=torch.float64, device="cuda"), "out": torch.zeros(n, dtype=torch.uint8, device="cuda"),
            "good": torch.zeros(1, dtype=torch.int32, device="cuda")}


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
    oe = OracleEssential()
    try:
        import cv2
    except ImportError:
        cv2 = None
    dist = 50.0

    def scene(m, seed):
        p1, p2 = ec.scene(np.random.default_rng(seed), m, 0.1, 0.5, "side")
        E, nsol, mask, _ = oe.find_essential(p1, p2, ec.FX, ec.FY, ec.CX, ec.CY)
        assert nsol == 1
        return p1, p2, E.reshape(-1)[:9].copy(), mask

    for m in (150, 300, 600, 4096):
        p1, p2, Ecm, mask = scene(m, m)
        b = buffers(p1, p2, Ecm, mask)
        call = lambda: hv.recover_pose_device(b["E"], b["xy1"], b["xy2"], b["R"], b["t"], b["out"], b["good"], ec.FX, ec.FY, ec.CX, ec.CY,
                                              dist, d_mask_in=b["mask"])
        dev_us = event_time(call)
        Erm = Ecm.reshape(3, 3).T
        hs = []
        for _ in range(50):
            t0 = time.perf_counter()
            hv.recover_pose(Erm, p1, p2, ec.FX, ec.FY, ec.CX, ec.CY, dist, mask)
            hs.append((time.perf_counter() - t0) * 1e6)
        d = {"m": m, "inliers": int(mask.sum()), "good": int(b["good"].item()), "device_us_per_call": round(dev_us, 1),
             "host_call_us": round(float(np.median(hs)), 1)}
        if cv2 is not None:
            cs = []
            for _ in range(10):
                t0 = time.perf_counter()
                cv2.recoverPose(Erm, p1, p2, ec.K, distanceThresh=dist, mask=mask.reshape(-1, 1).copy())
                cs.append((time.perf_counter() - t0) * 1e6)
            d["cv2_host_us_rough_guide"] = round(float(np.median(cs)), 1)
        emit(d)

    # 64 sessions: one batch against 64 per-session calls
    S = 64
    scenes = [scene(300, 1000 + j) for j in range(S)]
    bb = [buffers(*s) for s in scenes]
    bs = [buffers(*s) for s in scenes]
    jobs = [capi.pose_job(x["E"], x["xy1"], x["xy2"], x["R"], x["t"], x["out"], x["good"], ec.FX, ec.FY, ec.CX, ec.CY, d_mask_in=x["mask"])
            for x in bb]

    def batch():
        hv.recover_pose_batch_device(jobs, dist)

    def singles():
        for x in bs:
            hv.recover_pose_device(x["E"], x["xy1"], x["xy2"], x["R"], x["t"], x["out"], x["good"], ec.FX, ec.FY, ec.CX, ec.CY, dist,
                                   d_mask_in=x["mask"])

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
    same = all(torch.equal(x[k], y[k]) for x, y in zip(bb, bs) for k in ("R", "t", "out", "good"))
    emit({"sessions": S, "m": 300, "batch_us": round(float(np.median(tb)), 1), "per_session_calls_us": round(float(np.median(tsg)), 1),
          "outputs_identical": bool(same)})
    hv.close()


if __name__ == "__main__":
    main()
