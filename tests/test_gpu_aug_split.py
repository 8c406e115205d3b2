"""GPU test: at the end of a device op list in latency mode, the pose augmentation's covariance runs on the side stream (with the outlier
checks before it) while its mean is formed on the filter's stream by one CTA. Every consumer of P issued right behind such a list must wait
for the side stream; readers of the mean alone need not. Each consumer kind runs the same sequence in a child process in latency mode and
in one with HV_EKF_NO_PDL=1 (where the augmentation stays one more cluster of the checks' launch on the filter's stream): m, P and the
outputs of the consumer must be bitwise equal."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

TRAIL = 20                  # N = 160 (the benchmark's state)
FRAMES = 4
CONSUMERS = ("predict_cov", "visual_update", "visual_check_batch", "normalize", "translate", "unaugment", "transform", "download",
             "run_device_results", "group", "predicted_mean")


# ------------------------------------------------------------------------------------------------ child side
def child(consumer, out_path):
    import torch
    from hybvio_b200 import capi
    sys.path.insert(0, HERE)
    import kalman_ref as K
    lib = capi.load()
    ctx = capi.Context()
    p = capi.EkfParams()
    lib.hv_ekf_default_params(ctypes.byref(p))
    p.camera_trail_length = TRAIL
    e = capi.Ekf(ctx, p)
    N = e.N
    e.initialize_orientation([0.3, 0.2, 9.8])
    e.set_first_sample_time(0.999)
    rng = np.random.RandomState(7)
    keep = []

    def dev(a):
        t = torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()
        keep.append(t)
        return t.data_ptr()

    def visual(n, mode):
        l = K.visual_l(n, N)
        H = rng.normal(0, 0.02, (n, l)); f = rng.normal(0, 0.5, n); y = f + rng.normal(0, 0.05, n)
        o = capi.EkfOp()
        o.kind, o.n, o.l, o.mode, o.r, o.rmse_thr = capi.OP_VISUAL, n, l, mode, 0.05, -1.0
        o.H, o.f, o.y = dev(H.ravel(order="F")), dev(f), dev(y)
        return o

    t = [1.0]

    def predicts(k):
        ops = []
        for _ in range(k):
            o = capi.EkfOp()
            o.kind, o.t = capi.OP_PREDICT, t[0]
            t[0] += 0.005
            for i in range(3):
                o.gyro[i] = 0.01 * rng.normal(); o.acc[i] = (9.8 if i == 2 else 0.0) + 0.1 * rng.normal()
            ops.append(o)
        return ops

    def frame_end():
        """visual updates, then outlier checks + [SYMMETRIZE,] AUGMENT: the list ends with the fused frame end"""
        ops = [visual(8, 1), visual(20, 1)] + [visual(n, 0) for n in (8, 8, 20)]
        sym = capi.EkfOp(); sym.kind = capi.OP_SYMMETRIZE
        aug = capi.EkfOp(); aug.kind, aug.index = capi.OP_AUGMENT, -1
        return ops + [sym, aug]

    def run(ops):
        arr = (capi.EkfOp * len(ops))(*ops)
        keep.append(arr)
        e.run_device(arr, len(ops))
        return arr

    d_mean = torch.zeros(20, dtype=torch.float64, device="cuda")
    out = {}
    for k in range(FRAMES):
        run(predicts(4))
        e.predicted_mean_device(d_mean.data_ptr())
        e.flush()
        last = frame_end()
        run(last)
        # the consumer, issued right behind the list (nothing in between synchronises)
        if consumer == "predict_cov":
            run(predicts(4)); e.predicted_mean_device(d_mean.data_ptr()); e.flush()
        elif consumer == "visual_update":
            run([visual(20, 1)])
        elif consumer == "visual_check_batch":
            run([visual(8, 0), visual(20, 0)])
        elif consumer == "normalize":
            e.normalize_quaternions(False)
        elif consumer == "translate":
            e.translate_to([0.1 * k, 0.2, 0.3])
        elif consumer == "unaugment":
            e.unaugment()
        elif consumer == "transform":
            e.transform_to([0.1, 0.2, 0.3 * k], [0.9, 0.1, 0.2, 0.3] / np.linalg.norm([0.9, 0.1, 0.2, 0.3]))
        elif consumer == "download":
            m, P = e.download()
            out[f"download{k}_m"], out[f"download{k}_P"] = m, P
        elif consumer == "run_device_results":
            st, chi2 = e.run_device_results(len(last))
            out[f"results{k}_st"], out[f"results{k}_chi2"] = st, chi2
        elif consumer == "group":
            ops = [visual(8, 1)] + predicts(2) + [visual(20, 0), visual(8, 0)]
            arr = (capi.EkfOp * len(ops))(*ops)
            keep.append(arr)
            capi.ekf_group_run_device([e], [(arr, len(ops))])
        elif consumer == "predicted_mean":
            run(predicts(3))
            out[f"mean{k}"] = e.predicted_mean()
    m, P = e.download()
    out["m"], out["P"], out["mean_dev"] = m, P, d_mean.cpu().numpy()
    np.savez(out_path, **out)
    e.close()
    ctx.close()


# ------------------------------------------------------------------------------------------------ parent side
def _run_child(consumer, out_path, env_extra):
    env = dict(os.environ, **env_extra)
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "child", consumer, out_path], capture_output=True, text=True,
                       timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0, f"child {consumer} {env_extra} failed:\n{r.stdout[-2000:]}\n{r.stderr[-3000:]}"
    return dict(np.load(out_path))


@pytest.mark.parametrize("consumer", CONSUMERS)
def test_consumer_behind_split_augmentation_matches_throughput_mode(consumer, tmp_path):
    lat = _run_child(consumer, str(tmp_path / "latency.npz"), {})
    thr = _run_child(consumer, str(tmp_path / "no_pdl.npz"), {"HV_EKF_NO_PDL": "1"})
    assert sorted(lat) == sorted(thr)
    assert np.all(np.isfinite(lat["P"])) and np.all(np.isfinite(lat["m"]))
    for key in lat:
        a, b = np.ascontiguousarray(lat[key]), np.ascontiguousarray(thr[key])
        assert a.shape == b.shape and a.tobytes() == b.tobytes(), f"{consumer}: {key} differs between latency and throughput mode"


if __name__ == "__main__" and len(sys.argv) == 4 and sys.argv[1] == "child":
    child(sys.argv[2], sys.argv[3])
