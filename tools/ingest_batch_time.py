"""Device and wall time of frame ingest (colour -> gray and rectification into level 0, then the pyramid) for S stereo sessions sharing one
context: 2 S per-frame hv_ingest_frame calls against one hv_ingest_frames call over the same 2 S frames, from host pinned sources, and the
batched call again from device sources, alternating in one process.

Every frame is 752 x 480 with its own random rectification table (the EuRoC case is gray + table; the other setting is RGBA + table) and
a pyramid of win 31, max_level 3. Device time: CUDA events around each way's calls, issued behind a sleep kernel so that the events time
the device and not the host's issue rate. Wall time: host clock from the first call to the end of a stream synchronisation. Medians over
the repetitions after warm-up. After the last repetition every level of every pyramid (gray and gradients) of the three ways is compared
byte for byte. Prints a header line with the GPU's name and power limit, then one JSON line per (setting, S).

    python tools/ingest_batch_time.py [--reps 40] [--sizes 1,2,4,8,16,32,64] [--out results.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

W, H, WIN, MAX_LEVEL, WARMUP = 752, 480, 31, 3, 5
SETTINGS = [("gray+table", 1), ("rgba+table", 4)]
WAYS = ("per_frame", "batch_host", "batch_device")


def gpu_info():
    import torch
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
        out["power_limit_and_max_sm_clock"] = q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unavailable"
    except (OSError, subprocess.TimeoutExpired):
        out["power_limit_and_max_sm_clock"] = "unavailable"
    return out


def random_table(rng):
    from oracle import ingest_oracle as io
    n = W * H
    t = np.zeros(n, io.REMAP_DTYPE)
    t["x0"] = rng.randint(0, W, n); t["y0"] = rng.randint(0, H, n)
    t["xfrac"] = rng.rand(n).astype(np.float32); t["yfrac"] = rng.rand(n).astype(np.float32)
    t["x0"][rng.rand(n) < 0.02] = io.INVALID
    return t


def measure(hv, stream, channels, setting, S, reps):
    import torch
    from hybvio_b200 import capi
    rng = np.random.RandomState(S * 10 + channels)
    n = 2 * S
    shape = (H, W, channels) if channels > 1 else (H, W)
    host = [torch.from_numpy(rng.randint(0, 256, shape).astype(np.uint8)).pin_memory() for _ in range(n)]
    dev = [h.cuda() for h in host]
    tables = [random_table(rng) for _ in range(n)]
    ings = {k: [capi.Ingest(hv, W, H) for _ in range(n)] for k in WAYS}
    pyrs = {k: [hv.pyramid(W, H, WIN, MAX_LEVEL) for _ in range(n)] for k in WAYS}
    for k in WAYS:
        for ing, t in zip(ings[k], tables):
            ing.set_remap(t)
    torch.cuda.synchronize()
    lib = hv.lib
    stride = W * channels
    jobs_host = [capi.ingest_job(ings["batch_host"][j], host[j], pyrs["batch_host"][j]) for j in range(n)]
    jobs_dev = [capi.ingest_job(ings["batch_device"][j], dev[j], pyrs["batch_device"][j]) for j in range(n)]

    def per_frame():
        for j in range(n):
            capi.check(lib.hv_ingest_frame(ings["per_frame"][j].h_, host[j].data_ptr(), stride, channels, None, pyrs["per_frame"][j].h, None),
                       "hv_ingest_frame")

    fns = {"per_frame": per_frame, "batch_host": lambda: hv.ingest_frames(jobs_host), "batch_device": lambda: hv.ingest_frames(jobs_dev, True)}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dev_us = {k: [] for k in WAYS}
    wall_us = {k: [] for k in WAYS}
    launches = {}
    with torch.cuda.stream(stream):
        for rep in range(WARMUP + reps):
            for name in WAYS:
                torch.cuda._sleep(int(2e7 * (1 + S / 4)))       # the calls are queued before the device reaches them
                c0 = hv.launches
                ev0.record(stream)
                fns[name]()
                ev1.record(stream)
                ev1.synchronize()
                launches[name] = hv.launches - c0
                t0 = time.perf_counter()
                fns[name]()
                hv.sync()
                t1 = time.perf_counter()
                if rep >= WARMUP:
                    dev_us[name].append(1e3 * ev0.elapsed_time(ev1))
                    wall_us[name].append(1e6 * (t1 - t0))
    hv.sync()
    equal = True
    for j in range(n):
        for lv in range(pyrs["per_frame"][j].levels):
            ref = [a.tobytes() for a in pyrs["per_frame"][j].download(lv)]
            for k in WAYS[1:]:
                equal &= [a.tobytes() for a in pyrs[k][j].download(lv)] == ref
    for k in WAYS:
        for ing in ings[k]:
            ing.close()
        for p in pyrs[k]:
            p.release()
    out = {"setting": setting, "S": S, "frames": n, "reps": reps, "bit_equal": bool(equal)}
    for k in WAYS:
        out[k] = {"device_us_median": round(float(np.median(dev_us[k])), 1), "wall_us_median": round(float(np.median(wall_us[k])), 1),
                  "launches": launches[k]}
    for k in WAYS[1:]:
        out[k]["device_speedup"] = round(out["per_frame"]["device_us_median"] / out[k]["device_us_median"], 2)
        out[k]["wall_speedup"] = round(out["per_frame"]["wall_us_median"] / out[k]["wall_us_median"], 2)
    assert equal, out
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=40)
    ap.add_argument("--sizes", default="1,2,4,8,16,32,64")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("ingest_batch_time: no CUDA device")
    from hybvio_b200 import capi
    stream = torch.cuda.Stream()
    hv = capi.Context(0, stream=stream.cuda_stream)
    sink = open(args.out, "a") if args.out else None

    def emit(d):
        line = json.dumps(d)
        print(line, flush=True)
        if sink:
            sink.write(line + "\n"); sink.flush()

    emit({"gpu": gpu_info(), "frame": [W, H], "pyramid": {"win": WIN, "max_level": MAX_LEVEL}, "host_sources": "pinned"})
    for setting, channels in SETTINGS:
        for S in (int(x) for x in args.sizes.split(",")):
            emit(measure(hv, stream, channels, setting, S, args.reps))
    hv.close()
    if sink:
        sink.close()


if __name__ == "__main__":
    main()
