"""The clip stages at the sizes they are meant for: 1080p clips tracked at spacing 1, descriptors of more than 2^20
tracks per pair, and frames interpolated from a few sources.  Only there do the single-CTA scans of the tracker
(track_scan_kernel) and of the descriptors (traj_scan_kernel) carry their sums into a second pass, and does the hole
filling's grid-stride loop (interp_fill_kernel) take a second step.  Every list, record, descriptor float, frame,
flow and counter must be BITWISE what preprocess.track_points, preprocess.traj_descriptors and
preprocess.interpolate_frames give on the same arrays.

The level flows are set directly at sc_l = 0, where the full-resolution flow is the level flow itself, so the
restatements run on exactly the arrays built here.  tests/test_clip_stages_at_scale.py checks on the CPU that these
inputs reach the paths named above, with the thresholds read from the kernels' sources by kernel_limits()."""
import functools
import os
import re

import numpy as np
import pytest

from of_dis_b200 import params, preprocess, synth

pytestmark = pytest.mark.gpu

f32 = np.float32
LEVEL0 = "3 0 8 8 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0"  # sc_f 3, sc_l 0
H, W = 1080, 1920
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "of_dis_b200", "csrc")


def _source_ints(name, pattern):
    with open(os.path.join(CSRC, name)) as f:
        m = re.search(pattern, f.read())
    assert m, "%s no longer matches %r: update kernel_limits()" % (name, pattern)
    return [int(g) for g in m.groups()]


@functools.lru_cache(maxsize=None)
def kernel_limits():
    """The sizes at which the kernels branch, from their sources:
      track_pass   flags one pass of track_scan_kernel covers (TRACK_BLOCK flags per block, a block per thread);
      traj_pass    track slots one pass of traj_scan_kernel covers;
      fill_grid    threads of the largest interp_fill_kernel grid: a round with more holes takes a second step;
      fill_first   rounds of the hole filling's first batch, whose grid is sized by every pixel of the call;
      fill_warmup  rounds of its batches before they reach their largest size."""
    block, = _source_ints("ofdis_internal.cuh", r"constexpr int TRACK_BLOCK = (\d+);")
    track_threads, = _source_ints("track_kernels.cu", r"constexpr int TRACK_SCAN_THREADS = (\d+);")
    traj_threads, = _source_ints("traj_kernels.cu", r"constexpr int SCAN_THREADS = (\d+);")
    per_block, max_blocks = _source_ints("interp_kernels.cu",
                                         r"std::min<unsigned int>\(\(bound \+ \d+\) / (\d+), (\d+)u\)")
    fill_threads, = _source_ints("interp_kernels.cu", r"interp_fill_kernel<2><<<std::max\(blocks, 1u\), (\d+), 0")
    assert fill_threads == per_block
    first, last = _source_ints("ofdis_capi.cu", r"batch = (\d+); r < max_rounds; batch = std::min\(2 \* batch, (\d+)\)")
    warmup, b = 0, first
    while b < last:
        warmup, b = warmup + b, 2 * b
    return dict(track_pass=block * track_threads, traj_pass=block * traj_threads,
                fill_grid=max_blocks * fill_threads, fill_first=first, fill_warmup=warmup + last)


# ---- inputs ------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def clip(n, ch, stereo=False, h=H, w=W):
    """n + 1 textured uint8 frames (read-only)."""
    c = synth.synthetic_sequence(n + 1, h, w, ch, seed=7 + ch, amp=3.0, stereo=stereo)
    c.setflags(write=False)
    return c


# planted regions (rows, columns) of the tracker's and the descriptors' flows
NAN_BLOCK = (slice(100, 180), slice(200, 400))        # unknown: tracks there leave, those landing there are inconsistent
OUT_BLOCK = (slice(300, 360), slice(1700, 1800))      # moved a frame width to the right: leaves the frame
STEP_BLOCK = (slice(600, 800), slice(500, 900))       # 2.5 px further, B following: motion boundaries along its edges
BACK_BLOCK = (slice(400, 500), slice(1000, 1200))     # 3 px further with a zero backward flow: inconsistent
STILL_BLOCK = (slice(850, 950), slice(1300, 1500))    # no motion: its descriptors' segments are camera motion


def clip_flows(n, nop, h=H, w=W):
    """(F, B): n forward flows (n, h, w, nop) float32 and their backward partners.  Per pair a sub-pixel translation
    and a slow rotation about the centre with B = -F, so that most tracks survive, plus the planted blocks above, so
    that every end reason occurs."""
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    cx, cy = (w - 1) / 2, (h - 1) / 2
    F = np.empty((n, h, w, nop), f32)
    B = np.empty_like(F)
    for k in range(n):
        th, tx, ty = 2e-4 * (k + 1), 0.35 - 0.1 * k, -0.25 + 0.05 * k
        u = np.cos(th) * (x - cx) - np.sin(th) * (y - cy) + cx - x + tx
        v = np.sin(th) * (x - cx) + np.cos(th) * (y - cy) + cy - y + ty
        f = np.stack([u, v], -1)[..., :nop].astype(f32)
        f[NAN_BLOCK] = np.nan
        f[OUT_BLOCK + (0,)] += w
        f[STEP_BLOCK + (0,)] += 2.5
        f[BACK_BLOCK + (0,)] += 3.0
        f[STILL_BLOCK] = 0.0
        F[k], B[k] = f, -f
        B[k][BACK_BLOCK] = 0.0
    return F, B


def lattice_flows(n, nop, step=48, h=H, w=W):
    """(F, B) known only on every step-th row and column (NaN elsewhere): a few px of smooth motion, B = -F."""
    F = np.full((n, h, w, nop), np.nan, f32)
    y, x = np.mgrid[0:h:step, 0:w:step].astype(np.float64)
    for k in range(n):
        u = 3.0 * np.sin(4.0 * x / w + 0.5 * k) * np.cos(3.0 * y / h)
        v = 2.0 * np.cos(2.5 * x / w) * np.sin(5.0 * y / h + 0.7 * k)
        F[k, ::step, ::step] = np.stack([u, v], -1)[..., :nop]
    return F, -F


def corner_flows(h, w):
    """One pair whose only known forward flow is at pixel (0, 0)."""
    F = np.full((1, h, w, 2), np.nan, f32)
    F[0, 0, 0] = (1.0, 0.5)
    return F, -F


def track_params(nop, capacity, **kw):
    p = dict(capacity=capacity, spacing=1, alpha=0.01 if nop == 2 else 0.0, beta=0.5 if nop == 2 else 1.0,
             mb_alpha=0.01, mb_beta=0.002, min_eig=100.0)
    p.update(kw)
    return p


# name: (nop, channels, capacity, pairs).  "drop": a capacity between the survivors and the survivors plus the
# candidates, so both scans run past their first pass and seeds are dropped; "largest": the largest capacity accepted.
TRACK_CASES = {"gray": (2, 1, 1 << 22, 3), "rgb": (2, 3, 1 << 22, 3), "stereo": (1, 1, 1 << 22, 3),
               "drop": (2, 1, 1_500_000, 3), "largest": (2, 1, 1 << 24, 2)}


def track_inputs(case):
    """(frames, F, B, track params) of a TRACK_CASES entry."""
    nop, ch, cap, n = TRACK_CASES[case]
    F, B = clip_flows(n, nop)
    return clip(n, ch, stereo=nop == 1), F, B, track_params(nop, cap)


TRAJ_N = [1, 4]  # patch sizes: one pixel per cell, then 16


def traj_inputs(N):
    """(frames, F, B, track params, traj params): the cheapest descriptor (L = nt = ns = 1, dim 35) of every track of
    a 1080p clip at spacing 1 over 2 pairs; only the still block's segments are rejected."""
    F, B = clip_flows(2, 2)
    tp = dict(L=1, nt=1, N=N, ns=1, min_flow=0.4, eps=0.05, min_disp=0.1, min_var=0.0, max_var=1e9, max_dis=1e9)
    return clip(2, 1), F, B, track_params(2, 1 << 21), tp


INTERP_CASES = {"lattice-gray": (2, 1), "lattice-rgb": (1, 3)}  # nop, channels
CORNER = (144, 2048)  # h, w: more holes than fill_grid, filled from one pixel


def interp_inputs(case):
    """(frames0, frames1, F, B, h, w): two 1080p pairs on a 48-pixel lattice, or one wide pair from one corner."""
    if case == "corner":
        h, w = CORNER
        c = clip(1, 1, h=h, w=w)
        F, B = corner_flows(h, w)
    else:
        nop, ch = INTERP_CASES[case]
        h, w = H, W
        c = clip(2, ch, stereo=nop == 1)
        F, B = lattice_flows(2, nop)
    return c[:-1], c[1:], F, B, h, w


# ---- on the device -----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def api():
    from of_dis_b200 import api as _api

    _api.lib()
    return _api


def same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def assert_same(got, exp, name):
    assert got.shape == exp.shape and got.dtype == exp.dtype, (name, got.shape, exp.shape, got.dtype, exp.dtype)
    bad = got.view(np.uint8) != exp.view(np.uint8)
    if bad.any():
        raise AssertionError("%s: %d of %d bytes differ, first at byte %d"
                             % (name, int(bad.sum()), bad.size, int(np.flatnonzero(bad.reshape(-1))[0])))


def assert_lists(got, exp, name):
    assert len(got) == len(exp), (name, len(got), len(exp))
    for k, (g, e) in enumerate(zip(got, exp)):
        assert_same(g, e, "%s: list %d" % (name, k))


def level0_context(api, nop, ch, h, w, F, B):
    """A context whose slots 0 .. n-1 hold F and n .. 2n-1 B, set as level-0 flows."""
    prm = params.from_cli_numbers(LEVEL0.split(), noc=ch, nop=nop)
    n = F.shape[0]
    ctx = api.Context(prm, w, h, prm.p_samp_s, 2 * n)
    for k in range(n):
        ctx.set_flow(k, 0, F[k])
        ctx.set_flow(n + k, 0, B[k])
    full = np.empty((2 * n, h, w, nop), f32)
    ctx.get_flow_fullres(0, 2 * n, full, w, h)
    ctx.sync()
    assert same(full, np.concatenate([F, B])), "the full-resolution flows are not the level flows"
    return ctx


@functools.lru_cache(maxsize=1)
def expected_tracks(case):
    frames, F, B, p = track_inputs(case)
    return preprocess.track_points(frames, F, B, p)


def test_tracks_in_calls_of_one_and_two_pairs(api):
    """The gray clip split into calls of 1 and 2 pairs gives one call's lists and counters."""
    frames, F, B, p = track_inputs("gray")
    exp, est = expected_tracks("gray")
    ctx = level0_context(api, 2, 1, H, W, F, B)
    got = [ctx.track_begin(p, frames[0], W, H)]
    got += ctx.track_advance(0, 1, 3, frames[1:2], W, H)
    got += ctx.track_advance(1, 3, 4, frames[2:], W, H)
    assert_lists(got, exp, "two calls")
    assert ctx.track_stats() == est
    ctx.close()


@pytest.mark.parametrize("case", list(TRACK_CASES))
def test_tracks_equal_the_restatement(case, api):
    frames, F, B, p = track_inputs(case)
    nop, ch, _, n = TRACK_CASES[case]
    exp, est = expected_tracks(case)
    ctx = level0_context(api, nop, ch, H, W, F, B)
    got = [ctx.track_begin(p, frames[0], W, H)] + ctx.track_advance(0, n, n, frames[1:], W, H)
    assert_lists(got, exp, case)
    assert ctx.track_stats() == est
    ctx.close()


@pytest.mark.parametrize("N", TRAJ_N)
def test_descriptors_equal_the_restatement(N, api):
    frames, F, B, tpp, tp = traj_inputs(N)
    lists, records, desc, n_desc, tst, jst = preprocess.traj_descriptors(frames, F, B, None, tpp, tp)
    ctx = level0_context(api, 2, 1, H, W, F, B)
    got0 = ctx.traj_begin(tpp, tp, frames[0], W, H)
    got = ctx.traj_advance(0, 2, 2, frames[1:], W, H)
    assert_lists([got0] + got[0], lists, "N %d" % N)
    assert np.array_equal(got[3], n_desc), (got[3], n_desc)
    assert_same(got[1], records, "N %d records" % N)
    assert_same(got[2], desc, "N %d descriptors" % N)
    assert ctx.traj_stats() == jst and ctx.track_stats() == tst
    ctx.close()


@pytest.mark.parametrize("case", list(INTERP_CASES) + ["corner"])
def test_interpolation_equals_the_restatement(case, api):
    frames0, frames1, F, B, h, w = interp_inputs(case)
    nop, n = F.shape[3], F.shape[0]
    ch = 1 if frames0.ndim == 3 else 3
    alpha, beta = (0.01, 0.5) if nop == 2 else (0.0, 1.0)
    exp_out, exp_ut, rounds = preprocess.interpolate_frames(frames0, frames1, F, B, 0.5, alpha, beta,
                                                            with_rounds=True)
    ctx = level0_context(api, nop, ch, h, w, F, B)
    before = ctx.launch_count
    out, ut = ctx.interpolate_fullres(0, n, n, frames0, frames1, 0.5, w, h, alpha=alpha, beta=beta, with_flow=True)
    assert ctx.launch_count - before >= rounds
    assert_same(out, exp_out, "%s out" % case)
    assert_same(ut, exp_ut, "%s flow_t" % case)
    ctx.close()
