"""CPU check of the SOR chain mode's data flow (tools/sor_schedule_model.py, run_chain): one sweep per launch,
bands on CTAs that take tickets in start order, any residency and interleaving, progress published every
1 or 4 super-steps."""
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import sor_schedule_model as model  # noqa: E402

SHAPES = [  # (W4, h, HPAD, RT): full and partial last bands, one block column, wide and narrow levels
    (5, 100, 32, 1), (1, 65, 32, 1), (12, 96, 32, 1), (9, 130, 32, 2), (4, 64, 32, 2), (3, 257, 32, 4),
    (7, 200, 64, 1), (2, 129, 64, 2),
]


@pytest.mark.parametrize("pub", [1, 4])
@pytest.mark.parametrize("R", [1, 2, None])
@pytest.mark.parametrize("shape", SHAPES, ids=["W4=%d,h=%d,HPAD=%d,RT=%d" % s for s in SHAPES])
def test_chain_reads_the_raster_scan_operands_without_deadlock(shape, R, pub):
    W4, h, HPAD, RT = shape
    for seed in range(3):
        model.run_chain(W4, h, HPAD, RT, nf=2, R=R, pub=pub, seed=seed)


def test_chain_with_one_frame_and_three_frames():
    model.run_chain(6, 150, 32, 1, nf=1, R=2, pub=4, seed=5)
    model.run_chain(6, 150, 32, 1, nf=3, R=4, pub=4, seed=6)


@pytest.mark.parametrize("shape", [(5, 100, 32, 1), (9, 130, 32, 2), (3, 257, 32, 4)])
def test_model_rejects_a_halo_wait_one_super_step_short(shape):
    """The producer and compute events of a super-step interleave separately, so a published "tl done" is seen
    while super-step tl still runs: waiting for tl + HPAD instead of tl + 1 + HPAD must read a stale top block."""
    with pytest.raises(AssertionError):
        for seed in range(3):
            model.run_chain(*shape, nf=2, R=None, pub=1, seed=seed, lag=0)
