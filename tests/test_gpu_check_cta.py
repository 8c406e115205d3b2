"""GPU: the outlier checks of a batch launch (ekf_check_batch_cluster2_kernel) that fit one CTA run on one CTA each (ek2_check_cta),
larger ones on a cluster of their own. Every result word must equal the single check through hv_ekf_visual_device mode 0 (the cluster
kernel) bit for bit, through hv_ekf_run_device and hv_ekf_run_host lists, and the state must stay untouched."""
import ctypes
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import ekf_common as C
import kalman_ref as K

pytestmark = pytest.mark.gpu
R, NS = 0.05, 100.0
LIMIT, STATIC = 227 * 1024, 8 * (2 + 128 + 2 + 768) + 256     # ekf_cluster2.cu: EK2_SMEM_LIMIT, EK2_STATIC_SMEM


def _pad(w):
    return w + ((20 - (w & 15)) & 15)


def cluster_fits(n, l, N):
    """ekf_cluster2_fits(n, l, N, false)"""
    B = (N + 7) // 8
    p = (20 - (N & 15)) & 15
    LD = N + (p if p else 16)
    mt = (n + 7) >> 3
    RS = n * n if n * n <= 1024 else (64 * (mt * (mt + 1) // 2) + 7) // 8
    return 8 * (n * max(l, LD) + ((n * _pad(n + B + 1) + 1) & ~1) + LD * B + RS) + STATIC <= LIMIT


def on_one_cta(n, l, N):
    """ekf_check_on_one_cta(n, l, N): n l^2 <= 2^20 and ek2_check_cta_smem_bytes + the kernel's static shared memory fit"""
    B = (N + 7) // 8
    fits = 8 * (132 + ((n * l + 1) & ~1) + ((n * _pad(n + 1 + B) + 1) & ~1) + _pad(l) * B) + STATIC <= LIMIT
    return l <= N and n * l * l <= 1 << 20 and fits


def default_params():
    from hybvio_b200 import capi
    p = capi.EkfParams()
    capi.load().hv_ekf_default_params(ctypes.byref(p))
    return p


def _state(N, seed):
    rng = np.random.RandomState(seed)
    G = rng.normal(0, 1.0, (N, 12))
    P = np.eye(N) + 0.05 * (G @ G.T)
    return rng.normal(0, 0.3, N), np.asfortranarray(0.5 * (P + P.T))


class Checks:
    """Measurements (n, l) against one state, resident on the device and on the host, with their single-check results"""

    def __init__(self, e, shapes, P, seed):
        import torch
        from hybvio_b200 import capi
        self.shapes, self.host, self.dev = shapes, [], []
        for i, (n, l) in enumerate(shapes):
            H, f = K.make_measurement(n, l, seed + i)
            y = f + K.residual(P, H, R, NS, 40.0 if i % 4 == 3 else 0.5, seed + i)
            H, f, y = np.asfortranarray(H), np.ascontiguousarray(f), np.ascontiguousarray(y)
            self.host.append((H, f, y))
            self.dev.append(tuple(torch.from_numpy(np.ascontiguousarray(a.ravel(order="F"))).cuda() for a in (H, f, y)))
        self.ref = []
        d_res = torch.zeros(4, dtype=torch.float64, device="cuda")
        for (n, l), (dH, df, dy) in zip(shapes, self.dev):
            d_res.fill_(-7.0)
            e.visual_device(dH.data_ptr(), n, l, df.data_ptr(), dy.data_ptr(), R, -1.0, 0, d_res.data_ptr())
            torch.cuda.synchronize()
            r = d_res.cpu().numpy()
            self.ref.append((int(r[0]), r[1]))
        self.capi = capi

    def ops(self, device, extra=()):
        capi = self.capi
        ops = (capi.EkfOp * (len(self.shapes) + len(extra)))()
        for i, ((n, l), h, d) in enumerate(zip(self.shapes, self.host, self.dev)):
            ptr = [a.data_ptr() for a in d] if device else [a.ctypes.data for a in h]
            ops[i].kind, ops[i].n, ops[i].l, ops[i].mode, ops[i].r, ops[i].rmse_thr = capi.OP_VISUAL, n, l, 0, R, -1.0
            ops[i].H, ops[i].f, ops[i].y = ptr
        for j, (kind, index) in enumerate(extra):
            ops[len(self.shapes) + j].kind, ops[len(self.shapes) + j].index = kind, index
        return ops

    def assert_same(self, st, chi2, what):
        for i, ((n, l), (s_, c_)) in enumerate(zip(self.shapes, self.ref)):
            assert int(st[i]) == s_, f"{what}: op {i} (n={n}, l={l}): status {st[i]} != {s_}"
            assert np.float64(chi2[i]).view(np.uint64) == np.float64(c_).view(np.uint64), f"{what}: op {i} (n={n}, l={l}): chi2 {chi2[i]!r} != {c_!r}"


def _run_both(hv, trail, ms, shapes, seed):
    import torch
    from hybvio_b200 import capi
    N = K.state_dim(trail, ms)
    e = capi.Ekf(hv, C.params_with(default_params, trail, ms))
    m, P = _state(N, seed)
    e.upload(m, P)
    chk = Checks(e, shapes, P, seed)
    ops = chk.ops(True)
    e.run_device(ops, len(shapes))
    st, c2 = e.run_device_results(len(shapes))
    chk.assert_same(st, c2, "run_device")
    st, c2, _ = e.run_host(chk.ops(False), len(shapes))
    chk.assert_same(st, c2, "run_host")
    m_, P_ = e.download()
    assert np.array_equal(m_, m) and np.array_equal(P_, P), "a check changed the state"
    torch.cuda.synchronize()
    e.close()
    return chk


def _sweep(N):
    B = (N + 7) // 8
    ls = (B - 3, N, 37, N - 2 * B + 1)
    out = []
    for q, n in enumerate(x for x in (1, 7, 8, 9, 31, 32, 33, 84) if x <= N):
        l = ls[q % 4]
        if cluster_fits(n, l, N):
            out.append((n, l))
    return out


@pytest.mark.parametrize("trail,ms", [(6, 0), (20, 0), (20, 14)], ids=["N62", "N160", "N202"])
def test_batched_checks_match_the_cluster_kernel_bitwise(hv, trail, ms):
    """n = 1 .. 84 across the pivot blocks and the one-stage / two-stage S boundary; l below one column block, = N, odd, ending inside a
    block; every fourth check a gross outlier. All but n = 84 run on one CTA each."""
    N = K.state_dim(trail, ms)
    shapes = _sweep(N)
    assert len(shapes) >= 6 and any(on_one_cta(n, l, N) for n, l in shapes)
    chk = _run_both(hv, trail, ms, shapes, 40 + N)
    assert any(s == 3 for s, _ in chk.ref) and any(s == 0 for s, _ in chk.ref)


def test_checks_above_the_size_bound_keep_their_cluster(hv):
    """N = 160: n = 84, l = 111 is the largest l at n = 84 within n l^2 <= 2^20, l = 112 the first beyond -- one batch with both forms,
    one-CTA checks before, between and after the cluster-form ones."""
    trail, N = 20, 160
    assert on_one_cta(84, 111, N) and not on_one_cta(84, 112, N)
    shapes = [(84, 111), (8, 34), (84, 112), (20, 55), (1, 5), (84, 160), (40, 90), (33, 37), (84, 111)]
    assert all(cluster_fits(n, l, N) for n, l in shapes)
    _run_both(hv, trail, 0, shapes, 77)


def test_frame_batch_with_augmentation_keeps_its_launches(hv):
    """The bench frame's 15 checks (n = 8 / 20 / 40 on one CTA each, n = 84 on clusters), then symmetrise + augment: the launches of the
    parent layout (latency mode: the batch on the side stream and the augmentation; HV_EKF_NO_PDL=1: one launch carries both), with
    the single-check results bit for bit."""
    import torch
    from hybvio_b200 import capi
    trail, N = 20, 160
    rows = [(n, K.visual_l(n, N)) for n in (8, 20, 40, 84)]
    shapes = [rows[c % 4] for c in range(5, 20)]
    assert (84, 160) in shapes and sum(on_one_cta(n, l, N) for n, l in shapes) == 11
    e = capi.Ekf(hv, C.params_with(default_params, trail, 0))
    m, P = _state(N, 5)
    e.upload(m, P)
    chk = Checks(e, shapes, P, 500)
    ops = chk.ops(True, extra=((capi.OP_SYMMETRIZE, 0), (capi.OP_AUGMENT, -1)))
    torch.cuda.synchronize()
    before = hv.launches
    e.run_device(ops, len(shapes) + 2)
    st, c2 = e.run_device_results(len(shapes) + 2)
    assert hv.launches - before == (1 if os.environ.get("HV_EKF_NO_PDL") else 2)
    chk.assert_same(st, c2, "run_device + augmentation")
    got = e.download()
    assert np.isfinite(got[0]).all() and np.isfinite(got[1]).all()
    e.close()
