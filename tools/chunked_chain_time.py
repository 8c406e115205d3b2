"""Device time of one 84-row stereo track (21 poses) on a trail-20 filter with 47 hybrid-map points (N = 301), where the measurement does
not fit the cluster kernel whole:
  chain      hv_ekf_visual_tracks: model kernel + the row-chunked cluster kernel (check with chi_outlier_r, update with visual_r);
  per-track  hv_ekf_track_models + hv_ekf_visual_track(check) + hv_ekf_visual_track(update): the single-CTA kernel, host round trips;
and the config-2 chain (trail 20, N = 160, 20 candidate tracks of 2..21 poses, 5 updates: what bench.py reports as visual_update_loop),
which runs the unchunked cluster kernel. Times between CUDA events on the library's stream (the calls synchronise inside), median of
--reps; the filter state is re-uploaded before every repetition, outside the timed interval. Prints one JSON line with the GPU name,
power limit and clocks next to the numbers.

    python tools/chunked_chain_time.py [--reps 50]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    try:
        q = "name,power.limit,clocks.sm,clocks.mem,clocks.max.sm"
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except Exception as ex:                                    # noqa: BLE001
        return f"unavailable ({ex})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--config2-only", action="store_true", help="only the N = 160 chain (also runs on builds without the chunked form)")
    args = ap.parse_args()
    import torch
    import tri_common
    from hybvio_b200 import capi

    hv = capi.Context(0)
    stream = torch.cuda.ExternalStream(hv.stream)

    def ekf(trail, ms):
        p = capi.EkfParams()
        capi.load().hv_ekf_default_params(ctypes.byref(p))
        p.camera_trail_length = trail
        p.hybrid_map_size = ms
        return capi.Ekf(hv, p)

    def timed(fn, reset):
        ts = []
        for i in range(args.reps + 3):
            reset()
            hv.sync()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            fn()
            b.record(stream)
            b.synchronize()
            if i >= 3:
                ts.append(a.elapsed_time(b) * 1e3)
        return float(np.median(ts))

    def state(trail, ms, seed):
        base = tri_common.make_track(seed, trail=trail, npose=4, stereo=True)
        rng = np.random.RandomState(seed)
        m = np.concatenate([base["m"], rng.normal(0, 1.0, 3 * ms)])
        A = rng.normal(0, 1, (len(m), len(m)))
        P = 1e-4 * (A @ A.T) / len(m) + np.diag(np.full(len(m), 1e-4))
        return base, m, P

    def track(base, npose, rng):
        idx = np.concatenate([[0], np.sort(rng.choice(np.arange(1, 21), npose - 1, replace=False))]).astype(np.int32)
        ip = tri_common.project(base["m"], idx, base["T1"], base["T2"], True, base["pf_true"] + rng.normal(0, 0.4, 3))
        return idx, ip + rng.normal(0, 2e-3, ip.shape), rng.normal(0, 0.05, ip.shape)

    chi_r, vis_r = 0.01, 0.004
    res = {"gpu (name, power limit, SM clock, memory clock, max SM clock)": gpu_info(), "reps": args.reps}
    if not args.config2_only:
        one_track_at_301(res, ekf, timed, state, track, chi_r, vis_r)
    # ---- config 2: trail 20, 20 candidate tracks, 5 updates, one synchronisation
    base, m, P = state(20, 0, 5)
    rng = np.random.RandomState(9)
    tracks = [track(base, 2 + (k * 7) % 20, rng) for k in range(20)]
    e = ekf(20, 0)
    e.set_camera_model(base["T1"], base["T2"], use_stereo=True)
    reset = lambda: e.upload(m=m, P=P)                         # noqa: E731
    res["N160_config2_chain_us"] = timed(lambda: e.visual_tracks(tracks, chi_r, vis_r, max_successful_updates=5), reset)
    e.close()
    hv.close()
    print(json.dumps(res))


def one_track_at_301(res, ekf, timed, state, track, chi_r, vis_r):
    base, m, P = state(20, 47, 7)
    t84 = track(base, 21, np.random.RandomState(3))
    e = ekf(20, 47)
    e.set_camera_model(base["T1"], base["T2"], use_stereo=True)
    reset = lambda: e.upload(m=m, P=P)                         # noqa: E731
    res["N301_n84_chain_us"] = timed(lambda: e.visual_tracks([t84], chi_r, vis_r, max_successful_updates=1), reset)

    def per_track():
        d = e.track_models([t84], download=False)[0]
        st, _ = e.visual_track(d, chi_r, mode=0)
        if st == 0:
            e.visual_track(d, vis_r, mode=1)
        e.ctx.sync()
    res["N301_n84_per_track_single_cta_us"] = timed(per_track, reset)
    reset()
    got, succ = e.visual_tracks([t84], chi_r, vis_r, max_successful_updates=1)
    res["N301_n84_updated"] = bool(got[0]["updated"])
    e.close()


if __name__ == "__main__":
    main()
