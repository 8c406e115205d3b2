"""Device time and launches per frame of the visual-update chains of S filters: per-filter hv_ekf_visual_tracks calls, one after another
on the shared context, against one hv_ekf_group_visual_tracks call; alternating in one process, throughput mode (HV_EKF_NO_PDL=1),
lookahead 0, at BASELINE config 2 (N = 160) and config 4 (N = 62).

Every filter has its own state and, per frame, 20 candidate stereo tracks of mixed length (up to 21 poses at N = 160, 7 at N = 62) with
gross outliers and tracks behind the cameras, max_successful_updates 5 (tests/test_gpu_ekf_group_tracks.py: make_group, make_tracks).
Both calls synchronise before they return, so the CUDA events around a frame span the device work and the host gaps between the
per-filter calls. The two sets of filters see the same tracks; their final states are compared bit for bit. Prints one JSON line per
(config, S) and a header line with the GPU's name, power limit and max SM clock.

    python tools/ekf_group_tracks_time.py [--frames 60] [--sizes 1,2,4,8,16]
"""
import argparse
import json
import os
import sys
import time

os.environ["HV_EKF_NO_PDL"] = "1"          # throughput mode (several sessions per GPU), read once by the library
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402

WARMUP = 5


def measure(trail, S, frames, stream, hv):
    import torch
    import test_gpu_ekf_group_tracks as T
    from hybvio_b200 import capi
    A, B, bases = T.make_group(hv, trail, S, seed=1000 + 10 * trail + S)
    prms = [T.params(5, 0)] * S
    total = frames + WARMUP
    tracks = [[T.make_tracks(bases[i], 20, 7919 * i + k) for i in range(S)] for k in range(total)]

    def per_filter(k):
        for e, t, p in zip(A, tracks[k], prms):
            e.visual_tracks(t, **p)

    def group(k):
        capi.ekf_group_visual_tracks(B, tracks[k], prms)

    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    res = {"per_filter": [0.0, 0.0, 0, 0], "group": [0.0, 0.0, 0, 0]}      # device ms, host s, frames, launches
    with torch.cuda.stream(stream):
        for k in range(total):
            for name, fn in (("per_filter", per_filter), ("group", group)):
                ev0.record(stream)
                c0, t0 = hv.launches, time.perf_counter()
                fn(k)
                ev1.record(stream)
                ev1.synchronize()
                t1 = time.perf_counter()
                if k >= WARMUP:
                    r = res[name]
                    r[0] += ev0.elapsed_time(ev1); r[1] += t1 - t0; r[2] += 1; r[3] += hv.launches - c0
    hv.sync()
    N = A[0].N
    equal = True
    for a, b in zip(A, B):
        ma, Pa = a.download(); mb, Pb = b.download()
        equal = equal and np.array_equal(ma.view(np.uint64), mb.view(np.uint64)) and np.array_equal(Pa.view(np.uint64), Pb.view(np.uint64)) \
            and a.pose_count() == b.pose_count()
    for e in A + B:
        e.close()
    out = {"N": N, "S": S, "frames": res["group"][2], "bit_equal": bool(equal)}
    for name, (ms, hs, nf, nl) in res.items():
        out[name] = {"device_us_per_frame": round(1e3 * ms / nf, 1), "host_us_per_frame": round(1e6 * hs / nf, 1), "launches_per_frame": nl / nf}
    out["speedup"] = round(out["per_filter"]["device_us_per_frame"] / out["group"]["device_us_per_frame"], 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--sizes", default="1,2,4,8,16")
    ap.add_argument("--trails", default="20,6", help="camera trail lengths (20: N = 160, config 2; 6: N = 62, config 4)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("ekf_group_tracks_time: no CUDA device")
    from ekf_group_time import gpu_info
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
