"""hv_ingest_frames (csrc/capi.cu, ingest.cu): the frames of a stereo pair or of many sessions ingested with one ingest launch per 64
frames that need colour or a remap plus the pyramid launches, from host or device memory. Every job against hv_ingest_frame on the same
input into a separate pyramid on the same context -- gray_out and every level of the pyramid (gray and gradients, padded downloads)
BYTE-identical -- over 1 .. 4 channels, the default and explicit coefficients (both clamps firing), jobs with and without a remap table
and gray jobs without one, host views with padded strides, device sources at odd pitches and base addresses 1 .. 3 bytes past alignment,
two level-0 sizes and pyramids of different depth in one call, and the golden camera tables (where the oracle and the golden outputs
agree too); the launch count of a stereo pair, of 16 and 64 sessions and of gray frames; and every refusal, which leaves the pyramids,
gray_out and the launch count as they were."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from hybvio_b200 import capi
from oracle import ingest_oracle as io

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ingest_golden.npz")
HV_ERR_INVALID = -1
COEFFS = [None, (0.9, 0.8, 0.7, 0.6), (-0.35, 1.3, 0.45, -0.2)]
WIN = 5
# (channels, coefficient set, table, extra bytes per source row, max_level) of the frames of one size
FRAMES = [(1, 0, False, 0, 3), (1, 0, False, 3, 1), (1, 0, True, 5, 2), (2, 1, False, 0, 3), (3, 0, True, 0, 0), (4, 2, True, 2, 3),
          (3, 2, False, 7, 2), (4, 0, False, 0, 1), (2, 1, True, 1, 3)]


@pytest.fixture(scope="module")
def orc():
    subprocess.check_call(["make", "-C", ROOT, "oracle"], stdout=subprocess.DEVNULL)
    return io.OracleIngest()


def remap_table(rng, w, h, invalid=0.05):
    """Random table; some taps on the last column / row / pixel with non-zero fractions, some entries without a source."""
    n = w * h
    t = np.zeros(n, io.REMAP_DTYPE)
    t["x0"] = rng.randint(0, w, n); t["y0"] = rng.randint(0, h, n)
    t["xfrac"] = rng.rand(n).astype(np.float32); t["yfrac"] = rng.rand(n).astype(np.float32)
    e = rng.choice(n, max(3, n // 50), replace=False)
    t["x0"][e[0::3]] = w - 1; t["y0"][e[1::3]] = h - 1; t["x0"][e[2::3]] = w - 1; t["y0"][e[2::3]] = h - 1
    t["xfrac"][e] = rng.uniform(0.05, 1.0, e.size).astype(np.float32); t["yfrac"][e] = rng.uniform(0.05, 1.0, e.size).astype(np.float32)
    t["x0"][rng.rand(n) < invalid] = io.INVALID
    return t


class Frame:
    """One frame: its source bytes (a host buffer of `pitch` bytes per row, non-zero padding, and the same bytes on the device `offset`
    bytes past an allocation), the batched call's ingest + pyramid and the per-frame call's ingest + pyramid, both with the table."""

    def __init__(self, hv, rng, w, h, channels, coeff, table, pitch, max_level, offset=0, img=None):
        import torch
        self.w, self.h, self.c, self.coeff, self.table = w, h, channels, coeff, table
        if img is None:
            img = rng.randint(0, 256, (h, w, channels) if channels > 1 else (h, w)).astype(np.uint8)
        buf = rng.randint(1, 256, (h, pitch)).astype(np.uint8)
        buf[:, :w * channels] = img.reshape(h, w * channels)
        shape, strides = ((h, w, channels), (pitch, channels, 1)) if channels > 1 else ((h, w), (pitch, 1))
        self.host = np.lib.stride_tricks.as_strided(buf, shape, strides)
        self.buf = buf
        dbuf = torch.full((offset + h * pitch,), 0xA5, dtype=torch.uint8, device="cuda")
        dbuf[offset:].copy_(torch.from_numpy(buf.reshape(-1)))
        self.dev = dbuf.as_strided(shape, strides, offset)
        assert self.dev.data_ptr() % 16 == offset % 16
        self.ing, self.pyr = capi.Ingest(hv, w, h), hv.pyramid(w, h, WIN, max_level)
        self.ing_s, self.pyr_s = capi.Ingest(hv, w, h), hv.pyramid(w, h, WIN, max_level)
        if table is not None:
            self.ing.set_remap(table); self.ing_s.set_remap(table)
        self.gray = np.full((h, w), 0x5A, np.uint8)

    def job(self, device):
        return capi.ingest_job(self.ing, self.dev if device else self.host, self.pyr, self.coeff, self.gray)

    def check(self, what):
        """gray_out and every level against hv_ingest_frame on the same host bytes; returns the ingested image."""
        want = self.ing_s.frame(self.host, self.pyr_s, self.coeff)
        assert self.gray.tobytes() == want.tobytes(), f"{what}: gray_out, {np.count_nonzero(self.gray != want)} pixels differ"
        assert self.pyr.levels == self.pyr_s.levels
        for lv in range(self.pyr.levels):
            g, d = self.pyr.download(lv, padded=True)
            gs, ds = self.pyr_s.download(lv, padded=True)
            assert g.tobytes() == gs.tobytes(), f"{what}: gray level {lv} differs"
            assert d.tobytes() == ds.tobytes(), f"{what}: gradients of level {lv} differ"
        return want

    def release(self):
        for x in (self.ing, self.ing_s):
            x.close()
        for p in (self.pyr, self.pyr_s):
            p.release()


def frames_of_size(hv, rng, w, h, device):
    out = []
    for i, (c, k, table, extra, ml) in enumerate(FRAMES):
        pitch, offset = w * c + extra, 0
        if device:                      # byte-aligned bases at odd pitches, and aligned ones (TMA staging for the gray jobs)
            offset = i % 4
            pitch = pitch | 1 if offset else (w * c + 15) // 16 * 16
        out.append(Frame(hv, rng, w, h, c, COEFFS[k] if c > 1 else None, remap_table(rng, w, h) if table else None, pitch, ml, offset))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True])
def test_every_job_equals_the_per_frame_call(hv, device):
    import torch
    rng = np.random.RandomState(7 + device)
    frames = frames_of_size(hv, rng, 130, 70, device) + frames_of_size(hv, rng, 257, 61, device)
    order = rng.permutation(len(frames))                      # the two sizes interleaved in the job list
    frames = [frames[i] for i in order]
    torch.cuda.synchronize()
    jobs = [f.job(device) for f in frames]
    kernel_jobs = sum(1 for f in frames if f.c > 1 or f.table is not None)
    before = hv.launches
    hv.ingest_frames(jobs, device)
    assert hv.launches - before == (kernel_jobs + 63) // 64 + 2          # one pyramid launch per size
    hv.sync()
    for i, f in enumerate(frames):
        f.check(f"job {i}: {f.w}x{f.h}, {f.c} channels, coeff {f.coeff}, table {f.table is not None}, device {device}")
    for f in frames:
        f.release()


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True])
def test_golden_camera_tables(hv, orc, device):
    """The reference's pinhole / fisheye / zoomed-out rectification of the golden frame and its two colour frames in one call."""
    import torch
    g = np.load(GOLD)
    rng = np.random.RandomState(3)
    img = g["frame"]
    h, w = img.shape
    frames = []
    for k, name in enumerate(("pinhole", "fisheye", "zoomout")):
        table = g[name + "_table"].reshape(-1).view(io.REMAP_DTYPE)
        frames.append(Frame(hv, rng, w, h, 1, None, table, w + (k if device else 0), 2, k if device else 0, img=img))
    for c in (3, 4):
        rgb = g[f"rgb{c}"]
        frames.append(Frame(hv, rng, rgb.shape[1], rgb.shape[0], c, None, None, rgb.shape[1] * c + (c if device else 0), 1, c if device else 0, img=rgb))
    torch.cuda.synchronize()
    hv.ingest_frames([f.job(device) for f in frames], device)
    hv.sync()
    for name, f in zip(("pinhole", "fisheye", "zoomout"), frames):
        out = f.check(name)
        table = f.table
        assert np.array_equal(out, orc.remap(f.host, table)), name
        t = table.reshape(h, w)
        ok = (t["x0"] == io.INVALID) | ((t["x0"] + 1 < w) & (t["y0"] + 1 < h))      # taps inside the reference's own buffer
        assert np.array_equal(out[ok], g[name + "_out"][ok]), name
    for c, f in zip((3, 4), frames[3:]):
        out = f.check(f"rgb{c}")
        assert np.array_equal(out, g[f"rgb{c}_gray"]) and np.array_equal(out, orc.gray(f.host)), c
    for f in frames:
        f.release()


def stereo_sessions(hv, rng, n, w, h, channels=1):
    frames = []
    for i in range(2 * n):
        frames.append(Frame(hv, rng, w, h, channels, None, remap_table(rng, w, h), w * channels, 3))
    return frames


@pytest.mark.gpu
@pytest.mark.parametrize("sessions,size,launches", [(1, (752, 480), 2), (16, (752, 480), 2), (64, (160, 96), 6)])
def test_launches_of_rectified_stereo_sessions(hv, sessions, size, launches):
    """A rectified stereo pair and 16 sessions: 1 ingest + 1 pyramid launch; 64 sessions (128 frames): 2 ingest + 4 pyramid launches."""
    rng = np.random.RandomState(sessions)
    frames = stereo_sessions(hv, rng, sessions, *size)
    before = hv.launches
    hv.ingest_frames([f.job(False) for f in frames])
    assert hv.launches - before == launches
    hv.sync()
    for i in sorted({0, 1, len(frames) // 2, len(frames) - 1}):
        frames[i].check(f"{sessions} sessions, frame {i}")
    for f in frames:
        f.release()


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True])
def test_gray_frames_without_tables_take_pyramid_launches_only(hv, device):
    import torch
    rng = np.random.RandomState(40)
    frames = [Frame(hv, rng, 203, 61, 1, None, None, 203 + (i % 3), 3, i % 4 if device else 0) for i in range(40)]
    torch.cuda.synchronize()
    before = hv.launches
    hv.ingest_frames([f.job(device) for f in frames], device)
    assert hv.launches - before == 2                                    # 40 frames: two pyramid launches of up to 32
    hv.sync()
    for i, f in enumerate(frames):
        f.check(f"gray frame {i}")
    for f in frames:
        f.release()


def _pyr_field_offsets(tmp_path):
    """offsetof(hv_pyr, desc.lv[0].gray / .deriv): where a test finds a pyramid's device memory to aim a source at it."""
    src, exe = tmp_path / "off.cpp", tmp_path / "off"
    src.write_text('#include <cstdio>\n#include <cstddef>\n#include "capi_internal.h"\nint main() { printf("%zu %zu\\n", '
                   'offsetof(hv_pyr, desc) + offsetof(HvPyrDesc, lv) + offsetof(HvLevel, gray), '
                   'offsetof(hv_pyr, desc) + offsetof(HvPyrDesc, lv) + offsetof(HvLevel, deriv)); return 0; }\n')
    subprocess.check_call(["g++", "-std=c++17", "-w", "-I/usr/local/cuda/include", "-I" + os.path.join(ROOT, "hybvio_b200", "csrc"), str(src), "-o", str(exe)])
    return [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]


@pytest.mark.gpu
def test_every_refusal_leaves_everything_untouched(hv, tmp_path):
    import torch
    lib = capi.load()
    rng = np.random.RandomState(5)
    w, h = 96, 40
    frames = [Frame(hv, rng, w, h, c, None, remap_table(rng, w, h) if t else None, w * c, 2) for c, t in ((3, 1), (1, 1), (1, 0))]
    for f in frames:                                            # known contents to compare against after each refusal
        f.pyr.build(np.full((h, w), 77, np.uint8))
    hv.sync()
    snap = [[f.pyr.download(lv, padded=True) for lv in range(f.pyr.levels)] for f in frames]
    other = capi.Context(0)
    ing_other, pyr_other = capi.Ingest(other, w, h), other.pyramid(w, h, WIN, 2)
    ing_small, pyr_small = capi.Ingest(hv, w - 4, h), hv.pyramid(w - 4, h, WIN, 2)
    off_gray, off_deriv = _pyr_field_offsets(tmp_path)
    level0 = ctypes.c_void_p.from_address(frames[1].pyr.h.value + off_gray).value
    deriv0 = ctypes.c_void_p.from_address(frames[2].pyr.h.value + off_deriv).value

    def jobs(device=False):
        return [f.job(device) for f in frames]

    def refused(J, n=None, device=False, what=""):
        before = hv.launches
        arr = None if J is None else (capi.IngestJob * len(J))(*J)
        rc = lib.hv_ingest_frames(arr, len(J) if n is None else n, 1 if device else 0)
        assert rc == HV_ERR_INVALID, f"{what}: {rc}"
        assert hv.launches == before, what
        hv.sync()
        for f, s in zip(frames, snap):
            assert (f.gray == 0x5A).all(), what
            for lv in range(f.pyr.levels):
                g, d = f.pyr.download(lv, padded=True)
                assert g.tobytes() == s[lv][0].tobytes() and d.tobytes() == s[lv][1].tobytes(), (what, lv)

    refused(jobs(), n=0, what="no jobs")
    refused(jobs() * 43, n=capi.INGEST_BATCH_MAX + 1, what="129 jobs")
    refused(None, n=1, what="NULL jobs")
    for field in ("ing", "src", "dst"):
        J = jobs(); setattr(J[1], field, None)
        refused(J, what=f"NULL {field}")
    for ch in (0, 5):
        J = jobs(); J[1].channels = ch
        refused(J, what=f"{ch} channels")
    J = jobs(); J[0].stride_bytes = w * 3 - 1
    refused(J, what="stride below w * channels")
    J = jobs(); J[2].ing = ing_other.h_.value
    refused(J, what="ing of another context")
    J = jobs(); J[2].dst = pyr_other.h.value
    refused(J, what="pyramid of another context")
    J = jobs(); J[1].dst = pyr_small.h.value
    refused(J, what="pyramid of another size")
    J = jobs(); J[0].ing, J[0].dst = ing_small.h_.value, pyr_small.h.value; J[0].stride_bytes = w * 3
    assert lib.hv_ingest_frames((capi.IngestJob * 3)(*J), 3, 0) == 0        # a second size is fine
    hv.sync()
    for f in frames:
        f.gray[...] = 0x5A
        f.pyr.build(np.full((h, w), 77, np.uint8))
    J = jobs(); J[2].ing = J[0].ing
    refused(J, what="the same hv_ingest twice")
    J = jobs(); J[2].dst = J[1].dst
    refused(J, what="the same pyramid twice")
    torch.cuda.synchronize()
    J = jobs(True); J[0].src = level0
    refused(J, device=True, what="a device source on another job's level 0")
    J = jobs(True); J[1].src = level0
    refused(J, device=True, what="a device source on its own level 0")
    J = jobs(True); J[1].src = deriv0; J[1].stride_bytes = 4 * w
    refused(J, device=True, what="a device source on another job's gradients")
    for x in (ing_other, ing_small):
        x.close()
    for p in (pyr_other, pyr_small):
        p.release()
    other.close()
    for f in frames:
        f.release()
