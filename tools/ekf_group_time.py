"""Device time and launches per frame of S filters stepped one by one (hv_ekf_run_device, throughput mode) and as one group
(hv_ekf_group_run_device), alternating in one process, at BASELINE config 2 (N = 160) and config 4 (N = 62).

Per-filter frame lists are the bench's (10 predict + normalise, 5 check+update and 15 checks, symmetrise, augment), every filter with
its own IMU stream and measurements. Frames are issued in blocks of 5 behind a short sleep kernel, so that the CUDA events around a
block time the device and not the host's issue rate. The two sets of filters see the same frames; their final states are compared
bit for bit. Prints one JSON line per (config, S) and a header line with the GPU's name and power limit.

    python tools/ekf_group_time.py [--frames 200] [--sizes 1,2,4,8,16]
"""
import argparse
import json
import os
import subprocess
import sys

os.environ["HV_EKF_NO_PDL"] = "1"          # throughput mode (several sessions per GPU), read once by the library
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

BLOCK = 5


def gpu_info():
    import torch
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
        out["power_limit_and_max_sm_clock"] = q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unavailable"
    except (OSError, subprocess.TimeoutExpired):
        out["power_limit_and_max_sm_clock"] = "unavailable"
    return out


def measure(trail, S, frames, stream, hv):
    import torch
    import kalman_ref as K
    import test_gpu_ekf_group as G
    from hybvio_b200 import capi
    N = K.state_dim(trail, 0)
    pool = G.Pool(N, 17 + trail, entries=8)
    A, B = G._twins(hv, trail, S)
    total = frames + 2 * BLOCK                   # the first two blocks of each way are warm-up
    lists = [[G.frame(1.0 + 0.05 * k + 0.0001 * i, 7919 * i + k, pool.entries[(3 * i + k) % len(pool.entries)]) for i in range(S)]
             for k in range(total)]

    def per_filter(k):
        for e, ops in zip(A, lists[k]):
            e.run_device(ops, len(ops))

    def group(k):
        capi.ekf_group_run_device(B, lists[k])

    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    res = {"per_filter": [0.0, 0, 0], "group": [0.0, 0, 0]}       # device ms, frames, launches
    with torch.cuda.stream(stream):
        for b0 in range(0, total, BLOCK):
            for name, fn in (("per_filter", per_filter), ("group", group)):
                torch.cuda._sleep(int(2e7))      # ~10 ms: the block is queued before the device reaches it
                ev0.record(stream)
                c0 = hv.launches
                for k in range(b0, min(total, b0 + BLOCK)):
                    fn(k)
                ev1.record(stream)
                ev1.synchronize()
                if b0 >= 2 * BLOCK:
                    r = res[name]
                    r[0] += ev0.elapsed_time(ev1); r[1] += min(total, b0 + BLOCK) - b0; r[2] += hv.launches - c0
    hv.sync()
    equal = True
    for a, b in zip(A, B):
        ma, Pa = a.download(); mb, Pb = b.download()
        equal = equal and np.array_equal(ma.view(np.uint64), mb.view(np.uint64)) and np.array_equal(Pa.view(np.uint64), Pb.view(np.uint64)) \
            and a.pose_count() == b.pose_count() and a.platform_time() == b.platform_time()
    for e in A + B:
        e.close()
    out = {"N": N, "S": S, "frames": res["group"][1], "bit_equal": bool(equal)}
    for name, (ms, nf, nl) in res.items():
        out[name] = {"device_us_per_frame": round(1e3 * ms / nf, 1), "launches_per_frame": nl / nf}
    out["speedup"] = round(out["per_filter"]["device_us_per_frame"] / out["group"]["device_us_per_frame"], 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--sizes", default="1,2,4,8,16")
    ap.add_argument("--trails", default="20,6", help="camera trail lengths (20: N = 160, config 2; 6: N = 62, config 4)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("ekf_group_time: no CUDA device")
    from hybvio_b200 import capi
    print(json.dumps({"gpu": gpu_info(), "frames": args.frames}), flush=True)
    stream = torch.cuda.Stream()
    hv = capi.Context(0, stream=stream.cuda_stream)
    for trail in (int(x) for x in args.trails.split(",")):
        for S in (int(x) for x in args.sizes.split(",")):
            print(json.dumps(measure(trail, S, args.frames, stream, hv)), flush=True)
    hv.close()


if __name__ == "__main__":
    main()
