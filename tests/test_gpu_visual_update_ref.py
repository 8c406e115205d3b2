"""GPU: the visual Kalman update kernels on realistic filter states and track-model measurements (tests/visual_update_ref.py), through
every entry point that runs a dense visual update, against the extended-precision reference with its per-entry bound on m and P, chi2
within tau and the status; a check must leave the state bitwise unchanged. On failure the worst entry is named with its block of the
state, its 8-CTA column block and the kernel path."""
import ctypes
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import kalman_ref as K  # noqa: E402
import visual_update_ref as V  # noqa: E402

pytestmark = pytest.mark.gpu
R, R2, NS = V.R_VIS, V.R_CHECK, 100.0
CASES = V.cases()


def _params(trail, ms):
    from hybvio_b200 import capi
    p = capi.EkfParams()
    capi.load().hv_ekf_default_params(ctypes.byref(p))
    p.camera_trail_length, p.hybrid_map_size = trail, ms
    return p


class Gate:
    """Collects the worst ratio of every entry point of one case and fails with the entry that broke the bound."""

    def __init__(self, case):
        self.c, self.rows = case, []

    def state(self, ref, got, what, path=None):
        r, where = V.worst(ref, got[0], got[1], self.c.trail, self.c.ms)
        path = "/".join(path or self.c.path)
        self.rows.append(f"  {what:34s} {r:9.3g}  {where}  [{path}]")
        assert r <= 1.0, f"{self.c.name} {what}: per-entry ratio {r:.3g} at {where}, kernel path {path}"

    def check(self, st, c2, ref, kappa, what, n=None):
        n = n or self.c.n
        assert st == ref[0], f"{self.c.name} {what}: status {st} != {ref[0]}"
        r = K.chi2_error(ref[1], c2) / K.tau(n, kappa)
        self.rows.append(f"  {what:34s} {r:9.3g}  chi2 / tau")
        assert r <= 1.0, f"{self.c.name} {what}: chi2 error / tau = {r:.3g}"

    def report(self):
        print(f"\n{self.c.name} [{'/'.join(self.c.path)}]\n" + "\n".join(self.rows))


def _unchanged(e, m, P, what):
    m_, P_ = e.download()
    assert np.array_equal(m_, m) and np.array_equal(P_, P), f"{what} changed the state"


def _device_op(torch, capi, H, f, y, r, mode, offset):
    """One OP_VISUAL op with device pointers, H starting `offset` bytes past a 16-byte boundary (0 or 8)."""
    n, l = H.shape
    nl = n * l
    k = offset // 8
    buf = torch.zeros(nl + 2 * n + 2, dtype=torch.float64, device="cuda")
    assert buf.data_ptr() % 16 == 0
    buf[k:k + nl] = torch.from_numpy(np.asfortranarray(H).ravel(order="F")).cuda()
    buf[k + nl:k + nl + n] = torch.from_numpy(np.ascontiguousarray(f)).cuda()
    buf[k + nl + n:k + nl + 2 * n] = torch.from_numpy(np.ascontiguousarray(y)).cuda()
    base = buf.data_ptr() + offset
    ops = (capi.EkfOp * 1)()
    ops[0].kind, ops[0].n, ops[0].l, ops[0].mode, ops[0].r, ops[0].rmse_thr = capi.OP_VISUAL, n, l, mode, r, -1.0
    ops[0].H, ops[0].f, ops[0].y = base, base + 8 * nl, base + 8 * (nl + n)
    torch.cuda.synchronize()
    return ops, buf


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_dense_entry_points_within_the_per_entry_bound(hv, case):
    """visual_update; visual_check (inlier, gross outlier) and visual_check_update; a check at a second noise level followed by the
    speculative update; run_device (check + update) with H aligned and 8 bytes past a 16-byte boundary; one member of a
    group_run_device launch where the measurement fits the cluster kernel (the group runs no other)."""
    import torch
    from hybvio_b200 import capi
    c, g = case, Gate(case)
    ref = c.reference()
    checkable = c.n <= K.CHI2_MAX_N
    if checkable:
        ref_in = K.check(c.P, c.H, c.f, c.y, R, NS)
        ref_in2 = K.check(c.P, c.H, c.f, c.y, R2, NS)
        ref_out = K.check(c.P, c.H, c.f, c.y_out, R, NS)
        assert ref_in[0] == 0 and ref_in2[0] == 0 and ref_out[0] == 3
        kap2 = K.kappa_S(c.P, c.H, R2, NS)
    e = capi.Ekf(hv, _params(c.trail, c.ms))
    e.upload(c.m, c.P)
    e.visual_update(c.H, c.f, c.y, R)
    g.state(ref, e.download(), "visual_update")
    if checkable:
        e.upload(c.m, c.P)
        g.check(*e.visual_check(c.H, c.f, c.y, R), ref_in, ref.kappa, "visual_check inlier")
        g.check(*e.visual_check(c.H, c.f, c.y_out, R), ref_out, ref.kappa, "visual_check outlier")
        _unchanged(e, c.m, c.P, "a check")

        e.upload(c.m, c.P)
        st, c2, m_out = e.visual_check_update(c.H, c.f, c.y, R)
        g.check(st, c2, ref_in, ref.kappa, "visual_check_update")
        got = e.download()
        assert np.array_equal(m_out, got[0])
        g.state(ref, got, "visual_check_update")
        e.upload(c.m, c.P)
        st, c2, _ = e.visual_check_update(c.H, c.f, c.y_out, R)
        g.check(st, c2, ref_out, ref.kappa, "visual_check_update outlier")
        _unchanged(e, c.m, c.P, "an outlier")

        e.upload(c.m, c.P)                       # an update at R arms the speculative path; the check at R2 computes the update at R
        e.visual_update(c.H, c.f, c.y, R)
        e.upload(c.m, c.P)
        g.check(*e.visual_check(c.H, c.f, c.y, R2), ref_in2, kap2, "check at R2 (speculative)")
        e.visual_update(c.H, c.f, c.y, R)
        g.state(ref, e.download(), "check + speculative update")

        for off in (0, 8):
            ops, buf = _device_op(torch, capi, c.H, c.f, c.y, R, 2, off)
            e.upload(c.m, c.P)
            e.run_device(ops, 1)
            st, c2 = e.run_device_results(1)
            path = c.path if off == 0 else c.path_misaligned
            g.check(int(st[0]), float(c2[0]), ref_in, ref.kappa, f"run_device (H at +{off} B)")
            g.state(ref, e.download(), f"run_device (H at +{off} B)", path)
            del buf

    if checkable and c.path[0] == "cluster":
        # one member of a group launch (it runs measurements that fit the cluster kernel): this filter and a second one with the same state
        f2 = capi.Ekf(hv, _params(c.trail, c.ms))
        ops, buf = _device_op(torch, capi, c.H, c.f, c.y, R, 2, 0)
        e.upload(c.m, c.P); f2.upload(c.m, c.P)
        capi.ekf_group_run_device([e, f2], [(ops, 1), (ops, 1)])
        st, c2 = e.run_device_results(1)
        g.check(int(st[0]), float(c2[0]), ref_in, ref.kappa, "group_run_device")
        g.state(ref, e.download(), "group_run_device")
        f2.close()
        del buf
    e.close()
    g.report()


CHAIN = [c for c in CASES if len(c.tracks) == 1]


@pytest.mark.parametrize("case", CHAIN, ids=[c.name for c in CHAIN])
def test_chain_within_the_per_entry_bound(hv, case):
    """visual_tracks with one track (cluster form, or row-chunked where it does not fit whole) and one member of group_visual_tracks
    (where it fits the cluster kernel whole: the group has no row-chunked form),
    against the reference fed the device's own H and f (hv_ekf_track_model_download), so that the track model's tolerance does not
    enter: chi2 of the check at chi_outlier_r, m and P of the update at visual_r."""
    from hybvio_b200 import capi
    c, g = case, Gate(case)
    t = c.tracks[0]
    T1, T2 = V.rig()
    y = np.asarray(t.ip).ravel()

    def new():
        e = capi.Ekf(hv, _params(c.trail, c.ms))
        e.upload(c.m, c.P)
        e.set_camera_model(T1, T2, use_stereo=t.stereo, estimate_time_shift=t.time_shift)
        return e

    e = new()
    model = e.track_models([t.obs])[0]
    assert model["tri_status"] == 0 and model["vu_status"] == 0
    H, f = model["H"], model["f"]
    n, l = H.shape
    chunks = V.chain_chunks(n, l, c.N)
    whole = K.cluster_fits(n, l, c.N)
    path = K.kernel_path(n, l, c.N) if whole else ("row-chunked", f"{chunks} chunk(s)")
    ref = V.update(c.m, c.P, H, f, y, R, NS, c.trail, chunks)
    ref_chk = K.check(c.P, H, f, y, R2, NS)
    kap2 = K.kappa_S(c.P, H, R2, NS)
    assert ref_chk[0] == 0

    got, succ = e.visual_tracks([t.obs], R2, R, max_successful_updates=1)
    assert succ == 1 and got[0]["updated"]
    g.check(got[0]["outlier_status"], got[0]["chi2"], ref_chk, kap2, "visual_tracks check", n)
    g.state(ref, e.download(), "visual_tracks", path)

    e.close()
    if not whole:                       # the group runs only measurements that fit the cluster kernel whole
        g.report()
        return
    e = new()
    other = new()
    out = capi.ekf_group_visual_tracks([other, e], [[], [t.obs]], [dict(chi_outlier_r=R2, visual_r=R, max_successful_updates=1)] * 2)
    (res, succ) = out[1]
    assert succ == 1 and res[0]["updated"]
    g.check(res[0]["outlier_status"], res[0]["chi2"], ref_chk, kap2, "group_visual_tracks check", n)
    g.state(ref, e.download(), "group_visual_tracks", path)
    _unchanged(other, c.m, c.P, "an empty group member")
    other.close()
    e.close()
    g.report()


@pytest.mark.parametrize("kind", ["filled", "bench140", "trail30", "map14", "map47", "map80"])
def test_host_list_of_checks_across_batch_splits(hv, kind):
    """hv_ekf_run_host with 27 consecutive checks (more than one batch launch holds) of the state's cases, inliers and gross outliers
    alternating, rows 4 to 200: statuses and chi2 against the reference, the state bitwise unchanged."""
    from hybvio_b200 import capi
    cs = [c for c in CASES if c.state == kind and c.n <= K.CHI2_MAX_N]
    c0 = cs[0]
    ops = (capi.EkfOp * 27)()
    keep, exp = [], []
    for i in range(27):
        c = cs[i % len(cs)]
        y = c.y if i % 3 else c.y_out
        H, f, y = np.asfortranarray(c.H), np.ascontiguousarray(c.f), np.ascontiguousarray(y)
        keep += [H, f, y]
        ops[i].kind, ops[i].n, ops[i].l, ops[i].mode, ops[i].r, ops[i].rmse_thr = capi.OP_VISUAL, c.n, c.l, 0, R, -1.0
        ops[i].H, ops[i].f, ops[i].y = H.ctypes.data, f.ctypes.data, y.ctypes.data
        exp.append((*K.check(c.P, c.H, c.f, y, R, NS), K.tau(c.n, K.kappa_S(c.P, c.H, R, NS)), c.name))
    e = capi.Ekf(hv, _params(c0.trail, c0.ms))
    e.upload(c0.m, c0.P)
    st, c2, _ = e.run_host(ops, 27)
    worst = 0.0
    for i, (s_, c_, t, name) in enumerate(exp):
        assert st[i] == s_, f"op {i} ({name}): status {st[i]} != {s_}"
        r = K.chi2_error(c_, c2[i]) / t
        worst = max(worst, r)
        assert r <= 1.0, f"op {i} ({name}): chi2 error / tau = {r:.3g}"
    _unchanged(e, c0.m, c0.P, "a host list of checks")
    e.close()
    print(f"\n{kind}: 27 checks, worst chi2 error / tau {worst:.3g}")
