"""The inputs of tests/test_clip_stages_at_scale_gpu.py reach the code paths that test is there for; restatements
only, no GPU.  Without this the device comparisons could pass while the scans never carried into a second pass and
the hole filling never took a second grid-stride step."""
import functools

import numpy as np
import pytest

from of_dis_b200 import preprocess

from test_clip_stages_at_scale_gpu import (INTERP_CASES, TRACK_CASES, TRAJ_N, expected_tracks, interp_inputs,
                                           kernel_limits, track_inputs, traj_inputs)


def straddles(idx, edge):
    return idx.size > 0 and idx.min() < edge <= idx.max()


@pytest.mark.parametrize("case", list(TRACK_CASES))
def test_tracker_inputs_reach_the_second_scan_pass(case):
    """In some pair the survivors sit in list slots on both sides of the keep scan's first pass, and in some pair the
    candidate cells (admitted or dropped) on both sides of the candidate scan's; every end reason occurs."""
    frames, F, B, p = track_inputs(case)
    lists, st = expected_tracks(case)
    assert p["spacing"] == 1  # a cell is a pixel
    h, w = frames.shape[1:3]
    edge = kernel_limits()["track_pass"]
    keep_pairs, cand_pairs = [], []
    for k in range(len(lists) - 1):
        prev, cur = lists[k], lists[k + 1]
        kept = np.flatnonzero(np.isin(prev["id"], cur["id"]))  # the survivors' slots in the list they were read from
        if straddles(kept, edge):
            keep_pairs.append(k)
        # the candidates after the advance: the cells no survivor occupies whose smaller eigenvalue passes
        occ = np.zeros(h * w, bool)
        surv, seeds = cur[:kept.size], cur[kept.size:]
        occ[surv["y"].astype(np.int64) * w + surv["x"].astype(np.int64)] = True
        _, _, lam = preprocess.track_seed_eigen(frames[k + 1], 1)
        cand = np.flatnonzero(~occ & (lam >= np.float32(p["min_eig"])))
        # the seeds are the first candidates in cell order; the rest are dropped, only when the list is full
        assert np.array_equal(seeds["y"].astype(np.int64) * w + seeds["x"].astype(np.int64), cand[:seeds.size])
        assert cand.size == seeds.size or cur.size == p["capacity"]
        if straddles(cand, edge):
            cand_pairs.append(k)
    assert keep_pairs and cand_pairs, (case, keep_pairs, cand_pairs)
    assert min(st["ended_leaves"], st["ended_inconsistent"], st["ended_boundary"]) > 0, st
    assert (st["dropped"] > 0) == (case == "drop"), st


@functools.lru_cache(maxsize=1)
def expected_descriptors(N):
    frames, F, B, tpp, tp = traj_inputs(N)
    return preprocess.traj_descriptors(frames, F, B, None, tpp, tp)


@pytest.mark.parametrize("N", TRAJ_N)
def test_descriptor_inputs_reach_the_second_scan_pass(N):
    """In some pair segments are emitted from list slots on both sides of traj_scan_kernel's first pass."""
    lists, records, desc, n_desc, _, jst = expected_descriptors(N)
    edge = kernel_limits()["traj_pass"]
    assert desc.shape == (records.size, 35)
    ends = np.cumsum(n_desc)
    both = []
    for k in range(n_desc.size):
        ids = records["id"][ends[k] - n_desc[k]:ends[k]]
        slots = np.searchsorted(lists[k]["id"], ids)  # the lists are sorted by id
        assert np.array_equal(lists[k]["id"][slots], ids)
        if straddles(slots, edge):
            both.append(k)
    assert both, n_desc
    assert n_desc.min() > edge and jst["rejected_camera"] > 0, (n_desc, jst)


def splat_holes_at_least(F):
    """A lower bound of the holes the splat leaves in each pair: every known source splats into at most 4 targets."""
    known = (np.abs(F[..., 0]) <= 1e9) & (np.abs(F[..., -1]) <= 1e9)
    return F.shape[1] * F.shape[2] - 4 * known.reshape(F.shape[0], -1).sum(1)


@pytest.mark.parametrize("case", list(INTERP_CASES) + ["corner"])
def test_interpolation_inputs_take_a_second_fill_step(case):
    """More holes than interp_fill_kernel's largest grid after the splat in every pair, and more rounds than the first
    batch (the lattice) or than every batch before the largest (the corner)."""
    frames0, frames1, F, B, h, w = interp_inputs(case)
    lim = kernel_limits()
    assert (splat_holes_at_least(F) > lim["fill_grid"]).all()
    nop = F.shape[3]
    alpha, beta = (0.01, 0.5) if nop == 2 else (0.0, 1.0)
    _, _, rounds = preprocess.interpolate_frames(frames0, frames1, F, B, 0.5, alpha, beta, with_rounds=True)
    assert rounds > (lim["fill_warmup"] if case == "corner" else lim["fill_first"]), rounds
