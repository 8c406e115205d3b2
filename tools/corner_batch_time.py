"""Device time and launches of the new-corner step (detect -> select -> cornerSubPix) for S sessions sharing one context: S per-session
chains (hv_gftt_detect_device, hv_gftt_select_device, hv_subpix_refine_device per session) against the batched calls
(hv_gftt_detect_batch_device, hv_gftt_select_batch_device, hv_subpix_refine_batch_device), alternating in one process.

Every session has its own 752 x 480 frame and 100 previous corners; max_tracks 150, sub-pixel half-window 5 (criteria 3 / 30 / 0.01),
refinement over the whole capacity (the padding included), as a device pipeline runs it. Two settings: cell 32 with mask radius 50, and
cell 8 with mask radius 8. Each repetition issues one chain of each kind behind a short sleep kernel, so that the CUDA events around
each step time the device and not the host's issue rate; the medians over the repetitions after warm-up are reported per step and per
chain. After the last repetition the key points, corner lists, counts and refined points of the two ways are compared byte for byte.
Prints a header line with the GPU's name and power limit, then one JSON line per (setting, S).

    python tools/corner_batch_time.py [--reps 40] [--sizes 1,2,4,8,16,32,64] [--out results.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

W, H, MAX_TRACKS, NPREV, WARMUP = 752, 480, 150, 100, 5
SETTINGS = [(32, 50), (8, 8)]           # (cell, mask radius)
STEPS = ("detect", "select", "refine")


def gpu_info():
    import torch
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
        out["power_limit_and_max_sm_clock"] = q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unavailable"
    except (OSError, subprocess.TimeoutExpired):
        out["power_limit_and_max_sm_clock"] = "unavailable"
    return out


def measure(hv, stream, frames, cell, r, S, reps):
    import torch
    import gftt_select_common as gc
    from hybvio_b200 import capi
    pyrs, bufs, prevs = [], {"s": [], "b": []}, []
    for j in range(S):
        p = hv.pyramid(W, H, 31, 1)
        p.build(frames[j % len(frames)])
        pyrs.append(p)
        prevs.append(torch.from_numpy(gc.prev_points(NPREV, 100 + j, W, H)).cuda())
    nkp = int(np.prod(pyrs[0].gftt_cells(cell)))
    cap = gc.capacity(nkp, r, MAX_TRACKS)
    for k in "sb":
        for j in range(S):
            bufs[k].append((torch.zeros((nkp, 3), dtype=torch.float32, device="cuda"), torch.zeros((cap, 2), dtype=torch.float32, device="cuda"),
                            torch.zeros((1,), dtype=torch.int32, device="cuda")))
    torch.cuda.synchronize()
    lib = hv.lib
    jobs = [capi.corner_job(pyrs[j], *bufs["b"][j], prevs[j], r, MAX_TRACKS) for j in range(S)]
    sjobs = [capi.subpix_job(pyrs[j], bufs["b"][j][1]) for j in range(S)]

    def per_session(step):
        for j in range(S):
            kp, cor, cnt = bufs["s"][j]
            if step == "detect":
                capi.check(lib.hv_gftt_detect_device(hv.h, pyrs[j].h, 3, cell, 1e-3, kp.data_ptr()), "hv_gftt_detect_device")
            elif step == "select":
                capi.check(lib.hv_gftt_select_device(hv.h, kp.data_ptr(), nkp, prevs[j].data_ptr(), NPREV, r, MAX_TRACKS, cor.data_ptr(), cap,
                                                     cnt.data_ptr()), "hv_gftt_select_device")
            else:
                pyrs[j].subpix_refine_device(cor)

    def batch(step):
        if step == "detect":
            hv.gftt_detect_batch_device(jobs, 3, cell, 1e-3)
        elif step == "select":
            hv.gftt_select_batch_device(jobs)
        else:
            hv.subpix_refine_batch_device(sjobs)

    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    times = {"per_session": [], "batch": []}
    launches = {}
    with torch.cuda.stream(stream):
        for rep in range(WARMUP + reps):
            for name, fn in (("per_session", per_session), ("batch", batch)):
                torch.cuda._sleep(int(2e7))          # ~10 ms: the chain is queued before the device reaches it
                c0 = hv.launches
                ev[0].record(stream)
                for i, step in enumerate(STEPS):
                    fn(step)
                    ev[i + 1].record(stream)
                ev[3].synchronize()
                launches[name] = hv.launches - c0
                if rep >= WARMUP:
                    times[name].append([1e3 * ev[i].elapsed_time(ev[i + 1]) for i in range(3)])
    hv.sync()
    equal = all(a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes() for j in range(S) for a, b in zip(bufs["s"][j], bufs["b"][j]))
    counts = [int(bufs["b"][j][2].item()) for j in range(S)]
    for p in pyrs:
        p.release()
    out = {"cell": cell, "mask_radius": r, "S": S, "reps": reps, "bit_equal": bool(equal), "corners_per_session": [min(counts), max(counts)]}
    for name, t in times.items():
        t = np.array(t)
        med = {step: round(float(np.median(t[:, i])), 1) for i, step in enumerate(STEPS)}
        med["chain"] = round(float(np.median(t.sum(axis=1))), 1)
        out[name] = {"device_us_median": med, "launches_per_chain": launches[name]}
    out["chain_speedup"] = round(out["per_session"]["device_us_median"]["chain"] / out["batch"]["device_us_median"]["chain"], 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=40)
    ap.add_argument("--sizes", default="1,2,4,8,16,32,64")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("corner_batch_time: no CUDA device")
    from hybvio_b200 import capi, synth
    stream = torch.cuda.Stream()
    hv = capi.Context(0, stream=stream.cuda_stream)
    frames = [np.ascontiguousarray(synth.stereo_frame(k + 1, W, H)[0]) for k in range(16)]
    sink = open(args.out, "a") if args.out else None

    def emit(d):
        line = json.dumps(d)
        print(line, flush=True)
        if sink:
            sink.write(line + "\n"); sink.flush()

    emit({"gpu": gpu_info(), "frame": [W, H], "max_tracks": MAX_TRACKS, "nprev": NPREV, "subpix_half_window": 5})
    for cell, r in SETTINGS:
        for S in (int(x) for x in args.sizes.split(",")):
            emit(measure(hv, stream, frames, cell, r, S, args.reps))
    hv.close()
    if sink:
        sink.close()


if __name__ == "__main__":
    main()
