"""CPU: cv::RNG and RANSACPointSetRegistrator::getSubset restated in Python, against the oracle's replay of the draws."""
import os

import numpy as np
import pytest

_M64 = (1 << 64) - 1


def subsets_numpy(m, iters, seed=_M64, distinct=True):
    """cv::RNG(seed) (state = (uint64)(unsigned)state * 4164903690 + (state >> 32)); each subset draws rng.uniform(0, m) = next() % m,
    drawing again while the index repeats one of the subset's (distinct=False: a fault that keeps repeats)."""
    s = seed if seed else 0xFFFFFFFF
    out = np.zeros((max(iters, 1), 5), np.int32)
    for it in range(iters):
        for i in range(5):
            while True:
                s = ((s & 0xFFFFFFFF) * 4164903690 + (s >> 32)) & _M64
                v = (s & 0xFFFFFFFF) % m
                if not distinct or v not in out[it, :i]:
                    break
            out[it, i] = v
    return out[:iters]


@pytest.fixture(scope="module")
def orc():
    import subprocess
    from oracle import essential_oracle
    if not os.path.exists(essential_oracle.ORACLE_SO):
        subprocess.check_call(["make", "-s", "-C", os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"])
    return essential_oracle.OracleEssential()


@pytest.mark.parametrize("m", [6, 7, 20, 150, 4096])
def test_oracle_draws_match_the_restatement(orc, m):
    assert np.array_equal(orc.subsets(m, 300), subsets_numpy(m, 300))
