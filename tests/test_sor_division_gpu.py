"""The stereo SOR's division on the GPU (pytest -m gpu).  Both exact SOR kernels write the IEEE division B1 / A11
(solver.c:458) out by hand and guard it with a conservative exponent test; where the test fails for any pixel of a
warp, the warp redoes the work with the plain `/` (fdiv_rcp / fdiv_quot / fdiv_unsafe, of_dis_b200/csrc/
ofdis_internal.cuh).  Ordinary inputs never leave the written-out path, so these tests drive the operands out of
range on purpose:

a. ofdis_debug_div against the correctly rounded quotient, over every divisor mantissa at the edges of the range,
   every exponent pair and the special values;
b. parameter regimes that push A11 and / or B1 out of range, in every SOR path (sor_lane_kernel; sor_wave_kernel as
   one CTA, a cluster and a chain, at 1, 2 and 4 rows per thread), bitwise against the oracle, with proof from the
   oracle's planes and from the context's fallback counter that the fallback ran;
c. default parameters on fresh contexts: the fallback never runs, in particular not for the rows past the level that
   an odd-height level's last tile holds at 2 or 4 rows per thread."""
import dataclasses
import functools

import numpy as np
import pytest

from of_dis_b200 import params, preprocess, synth
from test_gpu_parity import CASES, assert_bits
from test_sor_chain_gpu import _narrow_prm

pytestmark = pytest.mark.gpu
f32 = np.float32


@pytest.fixture(scope="module")
def api():
    from of_dis_b200 import api as _api

    _api.lib()
    return _api


@pytest.fixture(scope="module")
def div_ctx(api):
    prm = _narrow_prm(1)
    ctx = api.Context(prm, 72, 64)
    yield ctx
    ctx.close()


# ---- the predicate and the reference quotient, restated from the bit patterns ---------------------------------
def out_of_range(x):
    """biased exponent outside [67, 187], i.e. not 2^-60 <= |x| < 2^61 (zeros, denormals, inf and NaN included)"""
    e = (np.ascontiguousarray(x, f32).view(np.uint32) >> 23) & 0xFF
    return (e < 67) | (e > 187)


def unsafe_pair(a, b):
    b = np.asarray(b, f32)
    nonzero = (b.view(np.uint32) & 0x7FFFFFFF) != 0
    return out_of_range(a) | (nonzero & out_of_range(b))


def correctly_rounded(a, b):
    """float32 b / a, correctly rounded: the double quotient rounded once more is exact for division (53 >= 2*24 + 2)"""
    with np.errstate(all="ignore"):
        return (np.asarray(b, np.float64) / np.asarray(a, np.float64)).astype(f32)


def check_division(ctx, a, b):
    a, b = np.ascontiguousarray(a, f32), np.ascontiguousarray(b, f32)
    q_fast, q_plain, unsafe = ctx.debug_div(a, b)
    exp = correctly_rounded(a, b)
    assert np.array_equal(unsafe, unsafe_pair(a, b)), "range test: %d pairs differ" % int((unsafe != unsafe_pair(a, b)).sum())
    safe = ~unsafe
    assert_bits(q_fast[safe], exp[safe], "written-out division inside the range")
    nan = np.isnan(exp)
    assert_bits(q_plain[~nan], exp[~nan], "plain division")
    assert np.isnan(q_plain[nan]).all()
    return int(safe.sum())


def _floats(exp_bits, mant_bits, sign_bits=0):
    bits = (np.asarray(sign_bits, np.uint32) << 31) | (np.asarray(exp_bits, np.uint32) << 23) | np.asarray(mant_bits, np.uint32)
    return np.asarray(bits, np.uint32).view(f32)


def test_division_hook_every_divisor_mantissa_at_the_edges_of_the_range(div_ctx):
    """All 2^23 divisor mantissas at biased exponents 67, 127 and 187 against numerators 1, 1 + ulp, 2 - ulp, 1.5
    and a random mantissa (random signs), at numerator exponents 67, 127 and 187: inside the range, the written-out
    division is the correctly rounded one.  One 2^23-pair chunk at a time."""
    rng = np.random.default_rng(0)
    mant = np.arange(1 << 23, dtype=np.uint32)
    checked = 0
    for ea in (67, 127, 187):
        a = _floats(ea, mant)
        for eb in (67, 127, 187):
            for mb in (0, 1, (1 << 23) - 1, 1 << 22, None):
                m = rng.integers(0, 1 << 23, mant.size, dtype=np.uint32) if mb is None else np.full(mant.size, mb, np.uint32)
                b = _floats(eb, m, rng.integers(0, 2, mant.size, dtype=np.uint32))
                checked += check_division(div_ctx, a, b)
    assert checked == 3 * 3 * 5 * (1 << 23)  # every pair of this sweep is inside the range


def test_division_hook_every_exponent_pair(div_ctx):
    """All 256 x 256 biased-exponent pairs (0 and 255 included), random mantissas and signs, 16 samples each."""
    rng = np.random.default_rng(1)
    ea, eb = np.meshgrid(np.arange(256, dtype=np.uint32), np.arange(256, dtype=np.uint32), indexing="ij")
    ea, eb = np.repeat(ea.reshape(-1), 16), np.repeat(eb.reshape(-1), 16)
    n = ea.size
    a = _floats(ea, rng.integers(0, 1 << 23, n, dtype=np.uint32), rng.integers(0, 2, n, dtype=np.uint32))
    b = _floats(eb, rng.integers(0, 1 << 23, n, dtype=np.uint32), rng.integers(0, 2, n, dtype=np.uint32))
    safe = check_division(div_ctx, a, b)
    assert 0 < safe < n


def test_division_hook_special_values(div_ctx):
    """Every pair of: +-0, the smallest and largest denormals, the smallest normal, 2^-60 and 2^61 and their
    neighbours one ulp away, 1, the largest float, +-inf and NaN."""
    def nb(x):
        x = f32(x)
        return [np.nextafter(x, f32(0)), x, np.nextafter(x, f32(np.inf))]

    tiny = np.finfo(f32).tiny
    v = [0.0, f32(1e-45), _floats(0, (1 << 23) - 1)[()], tiny, 1.0, np.finfo(f32).max, np.inf, np.nan]
    v += nb(2.0 ** -60) + nb(2.0 ** 61)
    v = np.array(v, f32)
    v = np.concatenate([v, -v])
    a, b = np.meshgrid(v, v, indexing="ij")
    safe = check_division(div_ctx, a.reshape(-1), b.reshape(-1))
    assert safe > 0


# ---- parameter regimes that drive the SOR's operands out of range --------------------------------------------
# name: (factor on tv_alpha, factor on tv_gamma and tv_delta, constant initial disparity or None = random)
REGIMES = {
    "tiny": (1e-22, 1e-22, None),        # A11 and B1 below 2^-60 everywhere
    "huge": (1e22, 1e22, None),          # A11 and B1 at 2^61 and above
    "mixed": (1e-20, 1e-20, None),       # A11 straddles 2^-60: both classes in the same tiles and warps
    "tiny_data": (1.0, 1e-22, -2.0),     # ordinary A11; B1 (= b1 in the first sweep) alone below 2^-60
    "zero_data": (1.0, 0.0, -2.0),       # B1 exactly +-0: the quotient's zero select, no fallback
}
# stereo levels: two CASES entries (refined at 128 and 100 rows), a 650-row level of 72 columns (chains) and a single
# 125-row level (odd: at 2 and 4 rows per thread the last tile holds rows past the level)
DIV_CASES = ["stereo_op4_small", "stereo_sor1_rows100", "narrow650", "odd125"]


def case_inputs(case, seed):
    if case == "narrow650":
        prm = _narrow_prm(1)
        i0, i1, _ = synth.synthetic_pair(650, 72, 1, seed=seed, amp=2.0, stereo=True)
    elif case == "odd125":
        prm = params.from_cli_numbers("0 0 6 6 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0".split(), noc=1, nop=1)
        i0, i1, _ = synth.synthetic_pair(125, 72, 1, seed=seed, amp=2.0, stereo=True)
    else:
        h, w, ch, mk, amp, stereo = CASES[case]
        prm = mk()
        i0, i1, _ = synth.synthetic_pair(h, w, ch, seed=seed, amp=amp, stereo=stereo)
    return i0, i1, prm


def division_inputs(case, regime):
    """The input pair, pyramids and parameters of `case` under `regime` (shared with tests/test_oracle.py, which pins
    the oracle at these parameters to the reference build)."""
    i0, i1, prm = case_inputs(case, {"narrow650": 60, "odd125": 62}.get(case, 31))
    sa, sd, _ = REGIMES[regime]
    prm = dataclasses.replace(prm, tv_alpha=prm.tv_alpha * sa, tv_gamma=prm.tv_gamma * sd, tv_delta=prm.tv_delta * sd)
    return i0, i1, preprocess.PairPyramids(i0, i1, prm.sc_f, prm.p_samp_s), prm


def initial_disparity(regime, pyr, prm):
    """the disparity the refinement of level sc_l starts from: random (<= 0) or the regime's constant"""
    hh, ww = pyr.level_shape(prm.sc_l)
    const = REGIMES[regime][2]
    if const is None:
        return -np.abs((np.random.default_rng(7).standard_normal((hh, ww, 1)) * 1.5).astype(f32))
    return np.full((hh, ww, 1), const, f32)


def replay_classes(st, prm):
    """Replays dis_sor_de (oracle/dis_oracle.c) on the oracle's planes of every inner iteration: the set of predicate
    values {unsafe, safe} seen over the pixels' (A11, B1) in all sweeps, and whether B1 == +-0 occurs.  The replayed
    (du) must equal the oracle's bit for bit, which pins the replay itself."""
    omega = f32(prm.tv_sor)
    classes, zero = set(), False
    for it in st["iters"]:
        sh, sv, b1 = it["sh"], it["sv"], it["b1"]
        h, w = b1.shape
        s = np.zeros((h, w), f32)  # neighbour sums in dis_sor_de's order: top, left, bottom, right
        s[1:] = s[1:] + sv[:-1]
        s[:, 1:] = s[:, 1:] + sh[:, :-1]
        s[:-1] = s[:-1] + sv[:-1]
        s[:, :-1] = s[:, :-1] + sh[:, :-1]
        A = (it["a11_pre"] + s).astype(f32)
        uA = out_of_range(A)
        du = it["du_in"].astype(f32).tolist()
        du = [[f32(x) for x in row] for row in du]
        A_, b1_, sh_, sv_, uA_ = A.tolist(), b1.tolist(), sh.tolist(), sv.tolist(), uA.tolist()
        for _ in range(prm.tv_solverit):
            for j in range(h):
                for i in range(w):
                    sg = f32(0)
                    if j > 0:
                        sg = sg - f32(sv_[j - 1][i]) * du[j - 1][i]
                    if i > 0:
                        sg = sg - f32(sh_[j][i - 1]) * du[j][i - 1]
                    if j < h - 1:
                        sg = sg - f32(sv_[j][i]) * du[j + 1][i]
                    if i < w - 1:
                        sg = sg - f32(sh_[j][i]) * du[j][i + 1]
                    B1 = f32(b1_[j][i]) - sg
                    a = f32(A_[j][i])
                    if B1 == 0:
                        zero = True
                        classes.add(bool(uA_[j][i]))
                    else:
                        e = (int(B1.view(np.uint32)) >> 23) & 0xFF
                        classes.add(bool(uA_[j][i]) or e < 67 or e > 187)
                    with np.errstate(all="ignore"):
                        du[j][i] = (f32(1) - omega) * du[j][i] + omega * (B1 / a)
        got = np.array([[float(x) for x in row] for row in du], f32)
        assert_bits(got, it["du"], "replay of dis_sor_de")
    return classes, zero


@functools.lru_cache(maxsize=None)
def regime_case(case, regime):
    """parameters, pyramids, initial disparity, the oracle's (du) after two inner iterations, its whole run, and the
    replayed predicate classes"""
    from oracle import port_driver

    port_driver.build()
    _, _, pyr, prm = division_inputs(case, regime)
    dense = initial_disparity(regime, pyr, prm)
    st = port_driver.varref_stages(pyr, prm, prm.sc_l, dense, n_iters=2)
    run = port_driver.port_run(pyr, prm)
    assert np.isfinite(st["iters"][1]["du"]).all() and np.isfinite(run).all()
    classes, zero = replay_classes(st, prm)
    return prm, pyr, dense, st["iters"][1], run, classes, zero


# SOR paths: (name, options); the chain of a small level needs 32-lane bands (sor_single_max 32), and a level of at
# most 32 lanes (odd125 at 4 rows per thread) still runs in one CTA
PATHS = [("lane", (("sor_lane", 1),))]
PATHS += [("single_rt%d" % rt, (("sor_lane", 0), ("sor_rows_per_thread", rt))) for rt in (1, 2, 4)]
PATHS += [("cluster_rt%d" % rt, (("sor_lane", 0), ("sor_single_max", 32), ("sor_rows_per_thread", rt))) for rt in (1, 2)]
PATHS += [("chain_rt%d" % rt, (("sor_lane", 0), ("sor_single_max", 32), ("sor_max_cluster", 1), ("sor_rows_per_thread", rt)))
          for rt in (1, 2, 4)]
# the 650-row level only runs as a chain (21 bands of 32 rows are too many for the lane kernel)
PATH_CASES = [(c, p) for c in DIV_CASES for p in PATHS if c != "narrow650" or p[0].startswith("chain")]
PATH_IDS = ["%s-%s" % (c, p[0]) for c, p in PATH_CASES]


def _refine_and_run(api, case, opts, prm, pyr, dense, it, run):
    """(du) after two inner iterations and the whole run (eager, graph replay) bitwise against the oracle; returns the
    fallback counts of the refinement and of the runs"""
    ctx = api.Context(prm, pyr.width, pyr.height, pyr.imgpadding, 1)
    try:
        for k, v in opts:
            ctx.set_option(k, v)
        ctx.upload_pyramids(0, pyr)
        lv = prm.sc_l
        ctx.set_flow(0, lv, dense)
        ctx.varref_refine(lv, 0, 1, n_inner=2)
        assert_bits(ctx.debug_get("dudv", 0, lv)[..., 0], it["du"], "du after two inner iterations")
        n_refine = ctx.sor_div_fallbacks(reset=True)
        for graph in (False, True):
            ctx.set_graph_mode(graph)
            ctx.run(1)
            assert_bits(ctx.get_flow(0, lv), run, "whole run, graph=%s" % graph)
        return n_refine, ctx.sor_div_fallbacks()
    finally:
        ctx.close()


@pytest.mark.parametrize("regime", list(REGIMES))
@pytest.mark.parametrize("case,path", PATH_CASES, ids=PATH_IDS)
def test_sor_division_fallback_vs_oracle(case, path, regime, api):
    prm, pyr, dense, it, run, classes, zero = regime_case(case, regime)
    n_refine, n_run = _refine_and_run(api, case, path[1], prm, pyr, dense, it, run)
    if regime == "zero_data":
        # the zero select: B1 == +-0 with A11 in range, nothing to redo
        assert zero and classes == {False}, classes
        assert n_refine == 0, n_refine
        return
    # the fallback ran: the oracle's operands fail the range test somewhere, and the kernel counted redone work
    assert True in classes, "regime %s never leaves the range: the test would be vacuous" % regime
    if regime == "mixed":
        assert classes == {True, False}, classes
    assert n_refine > 0, "no fallback counted (%s, %s)" % (path[0], regime)


# ---- no spurious fallback ----------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def default_case(case):
    from oracle import port_driver

    port_driver.build()
    i0, i1, prm = case_inputs(case, {"narrow650": 61, "odd125": 63}.get(case, 32))
    pyr = preprocess.PairPyramids(i0, i1, prm.sc_f, prm.p_samp_s)
    hh, ww = pyr.level_shape(prm.sc_l)
    dense = -np.abs((np.random.default_rng(9).standard_normal((hh, ww, 1)) * 1.5).astype(f32))
    st = port_driver.varref_stages(pyr, prm, prm.sc_l, dense, n_iters=2)
    classes, _ = replay_classes(st, prm)
    assert classes == {False}, "default parameters leave the range: pick other inputs"
    return prm, pyr, dense, st["iters"][1], port_driver.port_run(pyr, prm)


@pytest.mark.parametrize("case,path", PATH_CASES, ids=PATH_IDS)
def test_no_fallback_at_default_parameters_on_a_fresh_context(case, path, api):
    """Stereo levels of 128, 100, 650 and 125 rows with default parameters (and, in the whole runs, the coarser levels:
    64, 50 and 325 rows): no operand leaves the range (the oracle's replay says so), so no warp may take the plain
    division.  A fresh context matters: the records of the rows past an odd-height level, which the last tile holds at
    2 or 4 rows per thread, are the zeros of the workspace's memset, and A11 = 0 fails the range test if those rows
    take part in it."""
    prm, pyr, dense, it, run = default_case(case)
    n_refine, n_run = _refine_and_run(api, case, path[1], prm, pyr, dense, it, run)
    assert (n_refine, n_run) == (0, 0), "fallbacks counted: refine %d, runs %d" % (n_refine, n_run)


def test_gray_and_rgb_levels_share_the_lane_kernels_shared_memory_setting():
    """sor_lane_kernel's opt-in shared memory belongs to the kernel, which gray and RGB levels share: an RGB stereo
    level that needs less of it (32 rows, 104 KB) must not lower the setting under a gray stereo level that needs more
    (64 rows, 208 KB).  In a fresh process, so that no earlier test has raised the setting already."""
    import os
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = """if 1:
        import numpy as np
        from of_dis_b200 import api, params, preprocess, synth
        def run(rows, ch, numbers):
            prm = params.from_cli_numbers(numbers.split(), noc=ch, nop=1)
            i0, i1, _ = synth.synthetic_pair(rows, 72, ch, seed=5, amp=2.0, stereo=True)
            pyr = preprocess.PairPyramids(i0, i1, prm.sc_f, prm.p_samp_s)
            ctx = api.Context(prm, pyr.width, pyr.height, pyr.imgpadding, 1)
            ctx.set_option("sor_lane", 1)
            ctx.upload_pyramids(0, pyr)
            ctx.run(1)
            ctx.close()
        gray = "1 0 6 6 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0"  # levels of 128 and 64 rows
        run(128, 1, gray)
        run(32, 3, "0 0 6 6 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0")
        run(128, 1, gray)
    """
    subprocess.run([sys.executable, "-c", code], cwd=root, check=True, timeout=300)
