#!/usr/bin/env python
"""tools/check_batch_time.py -- what the outlier-check batch of bench.py's frame costs the frame (H100).

  python tools/check_batch_time.py [--steps 400] [--reps 3]                      frame A/B + the batch alone
  python tools/check_batch_time.py --trace [--out DIR]                            torch.profiler timeline of 100 frames

The default mode times hv_dev_run (bench.py's `value` loop) on the bench session, alternating the frame's full op list with
the same list minus its CHECKS - UPDATES pure checks (the augmentation then runs as a launch of its own): the difference bounds
what any change to the check batch can gain. It also times the check batch alone (CUDA events, as bench.py's kernel rows do)
and asks the runtime how many 8-CTA clusters of 512 threads fit the GPU at once at the batch's shared-memory size.

--trace records the device-resident loop with torch.profiler (a run of its own: tracing slows the host) and reads, per frame:
the gap between the fifth check+update and the augmentation, how long the two LK launches take while a check batch runs and
while none does, and how long the batch itself runs. bench.py is imported, not changed.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

OCC_SRC = r"""
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
__global__ void __launch_bounds__(512) probe(double* p) { extern __shared__ double s[]; if (p) p[threadIdx.x] = s[threadIdx.x]; }
int main(int argc, char** argv)
{
    const int smem = atoi(argv[1]), cl = atoi(argv[2]);
    cudaFuncSetAttribute(probe, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(cl * 16); cfg.blockDim = dim3(512); cfg.dynamicSmemBytes = smem;
    cudaLaunchAttribute at; at.id = cudaLaunchAttributeClusterDimension;
    at.val.clusterDim.x = cl; at.val.clusterDim.y = 1; at.val.clusterDim.z = 1;
    cfg.attrs = &at; cfg.numAttrs = 1;
    int n = -1;
    cudaError_t e = cudaOccupancyMaxActiveClusters(&n, (void*)probe, &cfg);
    printf("%d %s\n", n, cudaGetErrorString(e));
    return e != cudaSuccess;
}
"""


def max_active_clusters(smem, cluster=8):
    """cudaOccupancyMaxActiveClusters for a 512-thread kernel at `smem` bytes of shared memory per CTA (a probe kernel: at more than
    half an SM's shared memory one CTA fills an SM whatever its registers)."""
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "occ.cu"), os.path.join(d, "occ")
        with open(src, "w") as f:
            f.write(OCC_SRC)
        subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe, src])
        out = subprocess.check_output([exe, str(smem), str(cluster)], text=True).split()
    return int(out[0])


def ek2_smem_bytes(n, l, N):
    """ek2_smem_bytes(n, l, N, false) of ekf_cluster2.cuh: the cluster form of a check"""
    C = 8
    B = (N + C - 1) // C
    pad = (20 - (N & 15)) & 15
    LD = N + (pad if pad else 16)
    X = n * max(l, LD)
    w = n + B + 1
    W = w + ((20 - (w & 15)) & 15)
    T = (n * W + 1) & ~1
    mt = (n + 7) >> 3
    RS = n * n if n * n <= 1024 else (64 * (mt * (mt + 1) // 2) + C - 1) // C
    return 8 * (X + T + LD * B + RS)


def strip_checks(sess):
    """The session's op lists without the pure checks (ops IMU_OPS + UPDATES .. IMU_OPS + CHECKS - 1)"""
    capi = sess.capi
    drop = set(range(bench.IMU_OPS + bench.UPDATES, bench.IMU_OPS + bench.CHECKS))
    out = []
    for ops in sess.ops_dev:
        keep = [i for i in range(sess.nops) if i not in drop]
        arr = (capi.EkfOp * len(keep))()
        for j, i in enumerate(keep):
            ctypes.memmove(ctypes.byref(arr[j]), ctypes.byref(ops[i]), ctypes.sizeof(capi.EkfOp))
        out.append(arr)
    return out, sess.nops - len(drop)


def gpu_info(torch):
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,driver_version", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q[0] if q else None}


def batch_alone(sess, reps=200):
    """The CHECKS - UPDATES pure checks of the frame as one launch (no augmentation: the launch stays on the filter stream)"""
    torch = sess.torch
    k0, cnt = bench.IMU_OPS + bench.UPDATES, bench.CHECKS - bench.UPDATES

    def chk(i):
        ops = sess.ops_dev[i % bench.POOL_EKF]
        sess.ekf.run_device(bench.ctypes_slice(ops, k0, cnt), cnt)
    for i in range(5):
        chk(i)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record(sess.stream_b)
    for i in range(reps):
        chk(i)
    e.record(sess.stream_b)
    e.synchronize()
    return s.elapsed_time(e) * 1e3 / reps


def ab(sess, steps, reps):
    full, nfull = sess.ops_dev, sess.nops
    stripped, nstrip = strip_checks(sess)
    res = {"full": [], "no_checks": []}
    sess.run_dev_native(20)
    for r in range(reps):
        for name, ops, n in (("full", full, nfull), ("no_checks", stripped, nstrip)):
            sess.ops_dev, sess.nops = ops, n
            sess.run_dev_native(10)
            ms = sess.run_dev_native(steps)
            res[name].append(round(1e3 * ms / steps, 2))
    sess.ops_dev, sess.nops = full, nfull
    med = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
    return {"us_per_frame": res, "median_us": med, "gain_if_free": round(1.0 - med["no_checks"] / med["full"], 4)}


def trace(sess, out_dir, frames=100):
    torch = sess.torch
    from torch.profiler import ProfilerActivity, profile
    sess.run_dev_native(20)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        sess.run_dev_native(frames)
        torch.cuda.synchronize()
    path = os.path.join(out_dir, "check_batch_frames.pt.trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        ev = [e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel"]
    ev.sort(key=lambda e: e["ts"])
    batches = [e for e in ev if e["name"].startswith("ekf_check_batch_cluster2_kernel")]
    upd = [e for e in ev if e["name"].startswith("ekf_update_cluster2_kernel")]
    lk = [e for e in ev if "lk" in e["name"].lower()]
    gaps, aug_dur = [], []
    for b in batches:
        before = [u for u in upd if u["ts"] + u["dur"] <= b["ts"] + 1.0]
        after = [u for u in upd if u["ts"] >= b["ts"] - 1.0 and u not in before]
        if before and after:
            gaps.append(after[0]["ts"] - (before[-1]["ts"] + before[-1]["dur"]))
            aug_dur.append(after[0]["dur"])
    iv = [(b["ts"], b["ts"] + b["dur"]) for b in batches]
    lk_with, lk_without = [], []
    for e in lk:
        s, t = e["ts"], e["ts"] + e["dur"]
        (lk_with if any(a < t and s < z for a, z in iv) else lk_without).append(e["dur"])
    mean = lambda v: round(sum(v) / len(v), 2) if v else None
    return {"trace": path, "frames": frames, "batches": len(batches),
            "batch_us": mean([b["dur"] for b in batches]),
            "batch_grid": batches[0].get("args", {}).get("grid") if batches else None,
            "aug_start_after_update5_us": mean(gaps), "aug_us": mean(aug_dur),
            "lk_launches_overlapping_a_batch": len(lk_with), "lk_us_overlapping": mean(lk_with),
            "lk_launches_alone": len(lk_without), "lk_us_alone": mean(lk_without)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=400)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--trace", action="store_true")
    ap.add_argument("--out", default=tempfile.gettempdir(), help="directory of the --trace file")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("check_batch_time.py: no CUDA device")
    os.makedirs(args.out, exist_ok=True)
    torch.cuda.set_device(0)
    sess = bench.Session(0, bench.Inputs(torch.device("cuda", 0)))
    out = {"gpu": gpu_info(torch)}
    with torch.cuda.stream(sess.stream):
        if args.trace:
            out["trace"] = trace(sess, args.out)
        else:
            N = sess.ekf.N
            smem = max(ek2_smem_bytes(*bench.ekf_rows(c), N) for c in range(bench.UPDATES, bench.CHECKS))
            out["max_active_clusters_8x512"] = {"dynamic_smem_bytes": smem, "clusters": max_active_clusters(smem)}
            out["batch_alone_us"] = round(batch_alone(sess), 2)
            out["frame_ab"] = ab(sess, args.steps, args.reps)
    sess.ctx.sync(); sess.ctx_b.sync()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
