"""CPU checks of the serial frame-loop replay (tests/frame_loop_replay.py) that tests/test_gpu_frame_loop.py compares the GPU with:
the problem it poses is well conditioned (no outlier decision sits near its threshold, so the GPU's decisions must come out
identical), and its gate rejects what a wrong order of the loop's work would produce."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import frame_loop_replay as R  # noqa: E402
import bench  # noqa: E402

# (config, frame pool size, frames): the runs the GPU tests replay -- bench.py's README command (540 frames, config 2, default pool),
# the driver runs (200 frames, pool of 8), the shorter bench.py runs of configs 4 and 1 (140 frames)
WELL_POSED = [(2, 128, 600), (2, 8, 200), (4, 128, 140), (1, 128, 140)]


def cpu_inputs():
    import torch
    return bench.Inputs(torch.device("cpu"))


@pytest.mark.parametrize("cid,pool,nframes", WELL_POSED)
def test_outlier_decisions_are_well_posed(cid, pool, nframes):
    """Every check's chi2 is at least 10 % away from chi2inv95(n), and the decision pattern is the designed one: every
    designated update passes and every gross outlier (every fourth slot past the updates) is rejected, the rest pass."""
    with R.configured(cid, pool):
        inp = cpu_inputs()
        rep = R.Replay(inp, nframes, [], envelope=False)
        o = R.new_filter(inp)
        thr = np.array([o.chi2inv95(bench.ekf_rows(c)[0]) for c in range(bench.CHECKS)])
        o.close()
        margin = np.abs(rep.chi2[1:] / thr - 1.0)
        gross = np.array([c >= bench.UPDATES and c % 4 == 0 for c in range(bench.CHECKS)])
        k, c = np.unravel_index(np.argmin(margin), margin.shape)
        print(f"\nconfig {cid}, pool {pool}, {nframes} frames: closest chi2 {margin.min():.0%} from the threshold (frame {k + 1}, slot {c})")
        assert margin.min() >= 0.10
        assert np.array_equal(rep.status[1:] != 0, np.broadcast_to(gross, margin.shape))
        assert set(np.unique(rep.status[1:]).tolist()) <= {0, 3}


# fault replays: config 2, pool of 8 (the GPU driver runs), fault at FAULT_FRAME, chunk ends of the GPU tests' schedule after it
FAULT_FRAME, FAULT_RUN = 91, 100


@pytest.fixture(scope="module")
def fault_setup():
    with R.configured(2, 8):
        inp = cpu_inputs()
        marks = [int(k) for k in R.chunk_ends(R.chunk_schedule(200)) if FAULT_FRAME <= k <= FAULT_RUN]
        rep = R.Replay(inp, FAULT_RUN, marks)
        yield inp, rep, marks


def first_rejection(rep, faulty, marks):
    """The first chunk end at which the faulty replay fails the envelope or the decision comparison, or None."""
    for k in marks:
        ok = rep.gate(k, faulty.m[k], faulty.P[k])[0]
        if not ok or R.check_mismatches(rep, k, faulty.status[k], faulty.chi2[k]):
            return k
    return None


@pytest.mark.parametrize("fault", R.FAULTS)
def test_gate_rejects_a_wrong_order(fault_setup, fault):
    """One update applied twice; a check + update evaluated on the state before the update that precedes it (a check that read P
    too early); the IMU burst applied after the frame's visual list; one IMU timestamp off by 1e-7 s. Each must fail the gate at a
    chunk end after the fault; the first four are caught at the first chunk end."""
    inp, rep, marks = fault_setup
    with R.configured(2, 8):
        faulty = R.Replay(inp, FAULT_RUN, marks, fault=fault, fault_frame=FAULT_FRAME, envelope=False)
    k = first_rejection(rep, faulty, marks)
    ratios = {m: rep.gate(m, faulty.m[m], faulty.P[m])[1:3] for m in marks}
    print(f"\n{fault} at frame {FAULT_FRAME}: first rejected at chunk end {k} (chunk ends {marks}); "
          f"distance / D at {marks[0]}: m {ratios[marks[0]][0]:.3g}, P {ratios[marks[0]][1]:.3g}")
    assert k is not None
    if fault != "timestamp":
        assert k == marks[0]


def test_gate_rejects_lk_on_the_previous_frames_pyramid():
    """LK of the last frame run against the pyramids of the frame before (a rebuild the LK did not wait for): the bit-exact
    tracker comparison rejects it."""
    with R.configured(2, 8):
        inp = cpu_inputs()
        k = 13
        good, stale = R.tracker_replay(inp, k), R.tracker_replay(inp, k, stale_pyramid=True)
        assert R.tracker_mismatches(good, good) == []
        bad = R.tracker_mismatches(good, {key: v for key, v in stale.items() if key != "pyr"})
        assert "lk_next_temporal" in bad and "lk_next_stereo" in bad


def test_envelope_accepts_rounding_and_rejects_more(fault_setup):
    """The envelope's own replays are inside c D(k) by construction; a state two orders of magnitude further out is not."""
    inp, rep, marks = fault_setup
    k = marks[-1]
    with R.configured(2, 8):
        pushed = R.FilterReplay(inp, push="every")
        for _ in range(k):
            pushed.step()
        m, P = pushed.o.download()
        pushed.close()
    assert rep.gate(k, m, P)[0]
    Dm, DP = rep.D[k]
    assert not rep.gate(k, rep.m[k] * (1 + 100 * R.C_ENVELOPE * Dm), rep.P[k])[0]
    assert not rep.gate(k, rep.m[k], rep.P[k] + 100 * R.C_ENVELOPE * DP * np.abs(rep.P[k]).max())[0]
