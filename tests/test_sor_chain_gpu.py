"""SOR chain mode on the GPU (pytest -m gpu): levels with more bands than a thread-block cluster holds run as a
chain of CTAs, one sweep per launch, handing the band boundary over through global memory
(of_dis_b200/csrc/sor_wave_kernel.cuh, chain mode).  Every result is checked bitwise against the oracle."""
import functools

import numpy as np
import pytest

from of_dis_b200 import params, preprocess, synth
from test_gpu_parity import CASES, CLUSTER_CASES, assert_bits

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def api():
    from of_dis_b200 import api as _api

    _api.lib()
    return _api


def _narrow_prm(nop, fb=0):
    return params.from_cli_numbers(("1 0 6 6 0.05 0.95 0 8 0.4 %d 1 0 1 10 10 5 1 3 1.6 0" % fb).split(), noc=1, nop=nop)


def _narrow_pyr(rows, nop, seed, prm):
    i0, i1, _ = synth.synthetic_pair(rows, 72, 1, seed=seed, amp=2.0, stereo=(nop == 1))
    return preprocess.PairPyramids(i0, i1, prm.sc_f, prm.p_samp_s)


@functools.lru_cache(maxsize=None)
def _small_case(name, nfr):
    """pyramids of the frames, the oracle's (du,dv) after two inner iterations of the last frame, whole-run flows"""
    from oracle import port_driver

    port_driver.build()
    h, w, ch, mk, amp, stereo = CASES[name]
    prm = mk()
    pyrs = []
    for s in range(nfr):
        i0, i1, _ = synth.synthetic_pair(h, w, ch, seed=31 + s, amp=amp, stereo=stereo)
        pyrs.append(preprocess.PairPyramids(i0, i1, prm.sc_f, prm.p_samp_s))
    hh, ww = pyrs[0].level_shape(prm.sc_l)
    dense = (np.random.default_rng(7).standard_normal((hh, ww, prm.nop)) * 1.5).astype(np.float32)
    if stereo:
        dense = -np.abs(dense)
    st = port_driver.varref_stages(pyrs[-1], prm, prm.sc_l, dense, n_iters=2)["iters"][1]
    return prm, pyrs, dense, st, [port_driver.port_run(p, prm) for p in pyrs]


@pytest.mark.parametrize("pdl", [0, 1])
@pytest.mark.parametrize("max_cluster,rt", [(1, 1), (1, 2), (2, 1), (2, 2)])
@pytest.mark.parametrize("name", CLUSTER_CASES)
def test_chain_on_small_levels_vs_oracle(name, max_cluster, rt, pdl, api):
    """sor_max_cluster 1 / 2 with 32-lane single-CTA plans on the levels of the cluster tests (56..136 rows, 1..5
    sweeps, flow and stereo): with 1, every level beyond 32 lanes is a chain -- of one band, except the 136-row RGB
    level at one row per thread (128 + 8 rows); with 2 the plans are clusters of two bands or single CTAs.  The
    one-sweep-per-launch path and the plan switch are checked here; chains that hand rows from band to band for every
    (mode, rows per thread) are test_multi_band_chains_every_instantiation_vs_oracle.  Three frames per launch; (du,dv)
    after two inner iterations and the whole run, eager and graph replay, with and without programmatic dependent
    launch."""
    prm, pyrs, dense, it, runs = _small_case(name, 3)
    ctx = api.Context(prm, pyrs[0].width, pyrs[0].height, pyrs[0].imgpadding, 3)
    for k, v in (("sor_lane", 0), ("sor_single_max", 32), ("sor_max_cluster", max_cluster), ("sor_rows_per_thread", rt),
                 ("pdl", pdl)):
        ctx.set_option(k, v)
    for f, p in enumerate(pyrs):
        ctx.upload_pyramids(f, p)
    lv = prm.sc_l
    ctx.set_flow(2, lv, dense)
    ctx.varref_refine(lv, 0, 3, n_inner=2)
    dudv = ctx.debug_get("dudv", 2, lv)
    assert_bits(dudv[..., 0], it["du"], "du")
    if prm.nop == 2:
        assert_bits(dudv[..., 1], it["dv"], "dv")
    for graph in (False, True):
        ctx.set_graph_mode(graph)
        for rep in range(2):
            ctx.run(3)
            for f in range(3):
                assert_bits(ctx.get_flow(f, lv), runs[f], "graph=%s replay %d frame %d" % (graph, rep, f))
    ctx.close()


@functools.lru_cache(maxsize=None)
def _narrow_case(nop, rows, nfr):
    from oracle import port_driver

    port_driver.build()
    prm = _narrow_prm(nop)
    pyrs = [_narrow_pyr(rows, nop, 60 + s, prm) for s in range(nfr)]
    dense = (np.random.default_rng(8).standard_normal((rows, 72, nop)) * 1.5).astype(np.float32)
    if nop == 1:
        dense = -np.abs(dense)
    st = port_driver.varref_stages(pyrs[-1], prm, prm.sc_l, dense, n_iters=2)["iters"][1]
    return prm, pyrs, dense, st, [port_driver.port_run(p, prm) for p in pyrs]


@pytest.mark.parametrize("pdl", [0, 1])
@pytest.mark.parametrize("max_cluster", [1, 2])
@pytest.mark.parametrize("nop,rt", [(2, 1), (2, 2), (2, 4), (1, 1), (1, 2), (1, 4)])
def test_multi_band_chains_every_instantiation_vs_oracle(nop, rt, max_cluster, pdl, api):
    """A 650-row level, 72 columns, with sor_max_cluster 1 or 2: a chain in every (mode, rows per thread), i.e. every
    chain instantiation -- flow: 6 bands of 128 x 1 rows, 3 of 128 x 2, 3 of 64 x 4; stereo: 3 bands of 256 x 1,
    128 x 2, 64 x 4 --, each with a partial last band.  Three frames per launch; (du,dv) after two inner iterations
    and the whole run, eager and graph replay, with and without programmatic dependent launch."""
    prm, pyrs, dense, it, runs = _narrow_case(nop, 650, 3)
    ctx = api.Context(prm, pyrs[0].width, pyrs[0].height, pyrs[0].imgpadding, 3)
    for k, v in (("sor_lane", 0), ("sor_max_cluster", max_cluster), ("sor_rows_per_thread", rt), ("pdl", pdl)):
        ctx.set_option(k, v)
    for f, p in enumerate(pyrs):
        ctx.upload_pyramids(f, p)
    lv = prm.sc_l
    ctx.set_flow(2, lv, dense)
    ctx.varref_refine(lv, 0, 3, n_inner=2)
    dudv = ctx.debug_get("dudv", 2, lv)
    assert_bits(dudv[..., 0], it["du"], "du")
    if nop == 2:
        assert_bits(dudv[..., 1], it["dv"], "dv")
    for graph in (False, True):
        ctx.set_graph_mode(graph)
        for rep in range(2):
            ctx.run(3)
            for f in range(3):
                assert_bits(ctx.get_flow(f, lv), runs[f], "graph=%s replay %d frame %d" % (graph, rep, f))
    ctx.close()


# flow: 128-row bands (one row per thread), stereo: 256-row bands (two rows per thread) -- 2150 rows are 17 bands,
# 2200 and 4500 end with a partial band, 16384 is the tallest level a context accepts
@pytest.mark.parametrize("nop,rows", [(2, 2150), (2, 2200), (2, 4500), (2, 16384), (1, 4500), (1, 16384)])
def test_levels_beyond_any_cluster_default_options_vs_oracle(nop, rows, api, oracle_port):
    prm = _narrow_prm(nop)
    pyr = _narrow_pyr(rows, nop, 13, prm)
    ctx = api.Context(prm, pyr.width, pyr.height, pyr.imgpadding, 1)
    ctx.upload_pyramids(0, pyr)
    ctx.run(1)
    assert_bits(ctx.get_flow(0, prm.sc_l), oracle_port.port_run(pyr, prm), "run h=%d" % rows)
    ctx.close()


def test_chain_with_more_ctas_than_fit_at_once_vs_oracle(api, oracle_port):
    """8 frames of a 9000-row level: 8 x 71 chain CTAs of one sweep, far more than the GPU holds at once, so tickets
    are drawn while earlier bands still run."""
    prm = _narrow_prm(2)
    pyrs = [_narrow_pyr(9000, 2, 40 + s, prm) for s in range(2)]
    exp = [oracle_port.port_run(p, prm) for p in pyrs]
    ctx = api.Context(prm, pyrs[0].width, pyrs[0].height, pyrs[0].imgpadding, 8)
    for f in range(8):
        ctx.upload_pyramids(f, pyrs[f % 2])
    for graph in (False, True):
        ctx.set_graph_mode(graph)
        ctx.run(8)
        for f in range(8):
            assert_bits(ctx.get_flow(f, prm.sc_l), exp[f % 2], "graph=%s frame %d" % (graph, f))
    ctx.close()


def test_forward_backward_consistency_on_a_chained_level_vs_oracle(api, oracle_port):
    """usefbcon: the last level refines the forward frames only (every second internal frame) -- as a chain."""
    prm = _narrow_prm(2, fb=1)
    pyrs = [_narrow_pyr(2200, 2, 50 + s, prm) for s in range(2)]
    ctx = api.Context(prm, pyrs[0].width, pyrs[0].height, pyrs[0].imgpadding, 2)
    for f, p in enumerate(pyrs):
        ctx.upload_pyramids(f, p)
    ctx.run(2)
    for f, p in enumerate(pyrs):
        assert_bits(ctx.get_flow(f, prm.sc_l), oracle_port.port_run(p, prm), "fbcon frame %d" % f)
    ctx.close()


def test_uhd_flow_at_level_0_chain_equals_cluster(api):
    """4K UHD gray flow refined at level 0 (3840 x 2176 after padding): the default plan (a chain of 17 bands of 128
    rows) and the 16-CTA cluster of 9 bands of 256 rows (two rows per thread) give the same bits, and the flow is
    close to the synthetic ground truth."""
    prm = params.from_cli_numbers("5 0 12 12 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0".split(), noc=1)
    i0, i1, gt = synth.synthetic_pair(2160, 3840, 1, seed=5)
    pyr = preprocess.PairPyramids(i0, i1, prm.sc_f, prm.p_samp_s)
    ctx = api.Context(prm, pyr.width, pyr.height, pyr.imgpadding, 1)
    ctx.upload_pyramids(0, pyr)
    ctx.run(1)
    chain = ctx.get_flow(0, prm.sc_l)
    try:
        ctx.set_option("sor_max_cluster", 16)
    except api.OfdisError:
        ctx.close()
        pytest.skip("device grants no 16-CTA clusters")
    ctx.set_option("sor_rows_per_thread", 2)
    ctx.run(1)
    assert_bits(ctx.get_flow(0, prm.sc_l), chain, "cluster vs chain")
    ctx.close()
    full = preprocess.postprocess(chain, prm.sc_l, pyr.padw, pyr.padh, pyr.width_org, pyr.height_org)
    epe = np.sqrt(((full - gt) ** 2).sum(-1)).mean()
    assert epe < 0.5, epe
