"""Times sub-pixel corner refinement (cv::cornerSubPix) on a 752 x 480 frame: hv_subpix_refine_device under CUDA events, the host call
hv_subpix_refine end to end, and cv2.cornerSubPix on this machine's CPU with IPP off and on, for the same corners (the best GFTT cell
maxima of the frame) at 150 and 200 corners and half-windows 5 and 10. Prints the card name, its power limit and the host core count
first; with --out, also writes the numbers as JSON."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from hybvio_b200 import capi, synth  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--launches", type=int, default=400, help="timed device launches per configuration")
ap.add_argument("--host-reps", type=int, default=200, help="timed host calls (library and cv2) per configuration")
ap.add_argument("--out", default=None)
args = ap.parse_args()

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(f"card: {card}; host cores: {os.cpu_count()}")
try:
    import cv2
except ImportError:
    cv2 = None

W, H = 752, 480
img = synth.stereo_frame(0, W, H)[0]
hv = capi.Context(0)
pyr = hv.pyramid(W, H, 31, 3)
pyr.build(img)
kp = pyr.gftt_detect(3, 32, 1e-3)
corners = kp[np.argsort(-kp[:, 2], kind="stable"), :2].astype(np.float32)
stream = torch.cuda.ExternalStream(hv.stream)
crit = (3, 30, 0.01)
results = {"card": card, "host_cores": os.cpu_count(), "image": [W, H], "criteria": list(crit), "rows": []}
for n in (150, 200):
    pts = np.ascontiguousarray(corners[:n])
    for half in (5, 10):
        win = (half, half)
        row = {"n": n, "half_window": half}
        # device: every launch refines its own copy of the start points, so each does the full work
        with torch.cuda.stream(stream):
            bufs = torch.from_numpy(pts).cuda().repeat(args.launches + 10, 1, 1).contiguous()
        torch.cuda.synchronize()
        for i in range(10):
            pyr.subpix_refine_device(bufs[args.launches + i], win, (-1, -1), crit)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        for i in range(args.launches):
            pyr.subpix_refine_device(bufs[i], win, (-1, -1), crit)
        b.record(stream)
        b.synchronize()
        row["device_us"] = a.elapsed_time(b) * 1e3 / args.launches
        dev = bufs[0].cpu().numpy()
        # host call end to end (copy in, launch, completion, copy out)
        for _ in range(10):
            pyr.subpix_refine(pts, win, (-1, -1), crit)
        t = []
        for _ in range(args.host_reps):
            t0 = time.perf_counter(); host = pyr.subpix_refine(pts, win, (-1, -1), crit); t.append(time.perf_counter() - t0)
        row["host_call_us_median"] = float(np.median(t) * 1e6)
        row["device_equals_host"] = bool(np.array_equal(dev.view(np.uint32), host.view(np.uint32)))
        if cv2 is not None:
            for ipp in (False, True):
                cv2.ipp.setUseIPP(ipp)
                t = []
                for _ in range(args.host_reps):
                    p = pts.reshape(-1, 1, 2).copy()
                    t0 = time.perf_counter(); ref = cv2.cornerSubPix(img, p, win, (-1, -1), crit); t.append(time.perf_counter() - t0)
                key = "cv2_ipp_on" if ipp else "cv2_ipp_off"
                row[key + "_us_median"] = float(np.median(t) * 1e6)
                row[key + "_bit_equal"] = bool(np.array_equal(ref.reshape(-1, 2).view(np.uint32), host.view(np.uint32)))
            row["cv2_threads"] = cv2.getNumThreads()
        else:
            row["cv2"] = "not measured (cv2 not installed)"
        results["rows"].append(row)
        print(json.dumps(row))
pyr.release()
hv.close()
if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(results, f, indent=1)
