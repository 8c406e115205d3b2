"""Times corner selection (the detector's stable sort, resize quirk and applyMinDistance) on a 752 x 480 frame at cell 32 (345 key points)
and cell 8 (5640 key points):
  * the select kernel alone: CUDA events around --launches launches of hv_gftt_select_device after a warm-up, and the kernel's mean
    device time from torch.profiler in a separate pass;
  * hv_gftt_corners end to end (detect + select, one synchronisation) against hv_gftt_detect followed by the C oracle's
    orc_gftt_corners on the host (a plain-C restatement of the reference's host code, standing in for it; not that code), and that
    host selection alone;
  * the device chain hv_gftt_detect_device -> hv_gftt_select_device -> hv_subpix_refine_device -> hv_lk_track_device (left -> right,
    no initial flow, over the capacity) with one synchronisation, against the host-buffer calls hv_gftt_detect -> orc_gftt_corners ->
    hv_subpix_refine -> hv_lk_track, and against hv_gftt_corners -> hv_subpix_refine -> hv_lk_track; median host wall time.
Prints the card name, power limit and maximum SM clock first (queried in the same run); with --out, also writes the numbers as JSON."""
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
from oracle import gftt_oracle  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--launches", type=int, default=400, help="timed device launches per configuration")
ap.add_argument("--host-reps", type=int, default=300, help="timed host calls per configuration")
ap.add_argument("--out", default=None)
args = ap.parse_args()

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print(f"card: {card}; host cores: {os.cpu_count()}")
if not os.path.exists(gftt_oracle.ORACLE_SO):
    subprocess.check_call(["make", "-C", ROOT, "oracle"])
orc = gftt_oracle.OracleGftt()

W, H = 752, 480
L, R = synth.stereo_frame(0, W, H)
hv = capi.Context(0)
pl, pr = hv.pyramid(W, H, 31, 3), hv.pyramid(W, H, 31, 3)
hv.build_pyramids([pl, pr], [L, R])
hv.sync()
stream = torch.cuda.ExternalStream(hv.stream)
rng = np.random.RandomState(1)
prev = rng.uniform([0, 0], [W, H], (100, 2)).astype(np.float32)
MAX_TRACKS = 150


def median_us(fn, reps):
    for _ in range(10):
        fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter(); fn(); t.append(time.perf_counter() - t0)
    return float(np.median(t) * 1e6)


results = {"card": card, "host_cores": os.cpu_count(), "image": [W, H], "nprev": len(prev), "max_tracks": MAX_TRACKS, "rows": []}
for cell, radius in ((32, 50), (8, 8)):
    cx, cy = pl.gftt_cells(cell)
    nkp = cx * cy
    cap = capi.gftt_select_capacity(nkp, radius, MAX_TRACKS)
    row = {"cell": cell, "nkp": nkp, "mask_radius": radius}
    with torch.cuda.stream(stream):
        d_kp = torch.empty((nkp, 3), dtype=torch.float32, device="cuda")
        d_prev = torch.from_numpy(prev).cuda()
        d_xy = torch.empty((cap, 2), dtype=torch.float32, device="cuda")
        d_cnt = torch.empty((1,), dtype=torch.int32, device="cuda")
        d_next = torch.empty((cap, 2), dtype=torch.float32, device="cuda")
        d_st = torch.empty((cap,), dtype=torch.uint8, device="cuda")
        d_ts = torch.empty((cap,), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    pl.gftt_detect_device(d_kp.data_ptr(), 3, cell, 1e-3)
    hv.sync()

    # ---- the select kernel alone
    for _ in range(20):
        hv.gftt_select_device(d_kp, d_xy, d_cnt, d_prev, radius, MAX_TRACKS)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    for _ in range(args.launches):
        hv.gftt_select_device(d_kp, d_xy, d_cnt, d_prev, radius, MAX_TRACKS)
    b.record(stream)
    b.synchronize()
    row["select_events_us_per_launch"] = a.elapsed_time(b) * 1e3 / args.launches
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(args.launches):
            hv.gftt_select_device(d_kp, d_xy, d_cnt, d_prev, radius, MAX_TRACKS)
        hv.sync()
    ev = [e for e in prof.key_averages() if "hv_gftt_select_kernel" in e.key]
    row["select_kernel_us_profiler"] = (ev[0].device_time_total / ev[0].count) if ev else "not measured (kernel not in the trace)"
    n = int(d_cnt.item())
    kp_host = pl.gftt_detect(3, cell, 1e-3)
    want = orc.corners(kp_host, prev, radius, MAX_TRACKS)
    row["corners"] = n
    row["device_equals_oracle"] = bool(n == len(want) and np.array_equal(d_xy.cpu().numpy()[:n].view(np.uint32), want.view(np.uint32)))

    # ---- host-output selection
    row["host_oracle_select_us_median"] = median_us(lambda: orc.corners(kp_host, prev, radius, MAX_TRACKS), args.host_reps)
    row["detect_plus_host_oracle_us_median"] = median_us(lambda: orc.corners(pl.gftt_detect(3, cell, 1e-3), prev, radius, MAX_TRACKS),
                                                         args.host_reps)
    row["gftt_corners_us_median"] = median_us(lambda: pl.gftt_corners(prev, radius, MAX_TRACKS, 3, cell), args.host_reps)
    row["gftt_corners_equals_oracle"] = bool(np.array_equal(pl.gftt_corners(prev, radius, MAX_TRACKS, 3, cell).view(np.uint32),
                                                            want.view(np.uint32)))

    # ---- the four-call chain
    def device_chain():
        pl.gftt_detect_device(d_kp.data_ptr(), 3, cell, 1e-3)
        hv.gftt_select_device(d_kp, d_xy, d_cnt, d_prev, radius, MAX_TRACKS)
        pl.subpix_refine_device(d_xy)
        hv.lk_track_device(pl, pr, d_xy, d_next, d_st, d_ts, cap, False)
        hv.sync()

    def host_chain_oracle():
        c = orc.corners(pl.gftt_detect(3, cell, 1e-3), prev, radius, MAX_TRACKS)
        return hv.lk_track(pl, pr, pl.subpix_refine(c))

    def host_chain_corners():
        return hv.lk_track(pl, pr, pl.subpix_refine(pl.gftt_corners(prev, radius, MAX_TRACKS, 3, cell)))

    row["device_chain_us_median"] = median_us(device_chain, args.host_reps)
    row["host_chain_detect_oracle_us_median"] = median_us(host_chain_oracle, args.host_reps)
    row["host_chain_gftt_corners_us_median"] = median_us(host_chain_corners, args.host_reps)
    device_chain()
    nxt, _, ts = host_chain_oracle()
    row["device_chain_equals_host_chain"] = bool(int(d_cnt.item()) == len(nxt)
                                                 and np.array_equal(d_next.cpu().numpy()[:len(nxt)].view(np.uint32), nxt.view(np.uint32))
                                                 and np.array_equal(d_ts.cpu().numpy()[:len(nxt)], ts))
    results["rows"].append(row)
    print(json.dumps(row))
pl.release(); pr.release()
hv.close()
if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(results, f, indent=1)
