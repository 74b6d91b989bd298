"""ofdis_set_option("patch_lanes"): the P = 8 gray patch kernel (patch_p8c1_kernel) with 8 lanes per patch (one
template column each) or 4 (two adjacent columns each, 8 patches per warp).  Both settings, bitwise against the
oracle: the patch stage (p, pweight, conv, cnt and the dense flow, with and without initialisation from the
coarser level) and the whole run, over flow and stereo, patnorm 0/1, the four cost functions, early exit, outlier
resets, forward-backward consistency, patch counts that leave the last warp and CTA partly empty, and a batch of
frames with graph replay."""
import numpy as np
import pytest

from of_dis_b200 import params, preprocess, synth

pytestmark = pytest.mark.gpu


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def assert_bits(got, exp, name):
    got, exp = np.asarray(got), np.asarray(exp)
    assert got.shape == exp.shape, (name, got.shape, exp.shape)
    if got.dtype.kind == "f":
        bad = bits(got) != bits(exp)
        if bad.any():
            d = np.abs(got.astype(np.float64) - exp.astype(np.float64))
            raise AssertionError("%s: %d of %d values differ bitwise, max-abs %.3e, first at %s" %
                                 (name, int(bad.sum()), bad.size, float(np.nanmax(d)), np.argwhere(bad)[0]))
    else:
        assert np.array_equal(got, exp), name


@pytest.fixture(scope="module")
def api():
    from of_dis_b200 import api as _api

    _api.lib()
    return _api


# CLI numbers: sc_f sc_l max_iter min_iter dp_thresh dr_thresh res_thresh P patove usefbcon patnorm costfct usetvref
# alpha gamma delta innerit solverit omega verbosity.  P = 8 and gray everywhere: the kernel under test.
OP = "3 1 12 12 0.05 0.95 0 8 0.4 0 {pn} {cf} 1 10 10 5 1 3 1.6 0"
CASES = {
    # name: (nop, numbers, (h, w), amp)
    "flow_pn1_l2": (2, OP.format(pn=1, cf=0), (120, 200), 6.0),
    "flow_pn0_l2": (2, OP.format(pn=0, cf=0), (120, 200), 6.0),
    "flow_pn1_l1": (2, OP.format(pn=1, cf=1), (120, 200), 6.0),
    "flow_pn1_pseudo_huber": (2, OP.format(pn=1, cf=2), (120, 200), 6.0),
    "flow_pn0_pseudo_huber": (2, OP.format(pn=0, cf=2), (120, 200), 6.0),
    "flow_pn1_cost3": (2, OP.format(pn=1, cf=3), (120, 200), 6.0),
    "flow_early_exit": (2, "3 1 16 2 0.05 0.95 0.5 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0", (120, 200), 6.0),
    "flow_outlier_resets": (2, OP.format(pn=1, cf=0), (120, 200), 30.0),
    "flow_fbcon": (2, "3 1 8 8 0.05 0.95 0 8 0.4 1 1 0 1 10 10 5 1 3 1.6 0", (120, 200), 3.0),
    # 44 x 60 at level 0: 15 x 11 = 165 patches, the last warp of 8 (lanes 4) and of 4 (lanes 8) patches and the
    # last CTA of 32 partly empty
    "flow_partial_groups": (2, "2 0 12 12 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0", (44, 60), 4.0),
    "stereo_pn1_l2": (1, OP.format(pn=1, cf=0), (120, 200), 6.0),
    "stereo_pn0_l1": (1, OP.format(pn=0, cf=1), (120, 200), 6.0),
    "stereo_pn1_pseudo_huber": (1, OP.format(pn=1, cf=2), (120, 200), 6.0),
    "stereo_pn1_cost3": (1, OP.format(pn=1, cf=3), (120, 200), 6.0),
    "stereo_early_exit": (1, "3 1 16 2 0.05 0.95 0.5 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0", (120, 200), 6.0),
    "stereo_outlier_resets": (1, OP.format(pn=1, cf=0), (120, 200), 30.0),
    "stereo_fbcon": (1, "3 1 8 8 0.05 0.95 0 8 0.4 1 1 0 1 10 10 5 1 3 1.6 0", (120, 200), 3.0),
    "stereo_partial_groups": (1, "2 0 12 12 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0", (44, 60), 4.0),
}


@pytest.mark.parametrize("lanes", [4, 8])
@pytest.mark.parametrize("name", list(CASES))
def test_patch_stage_and_whole_run_vs_oracle(name, lanes, api, oracle_port):
    nop, numbers, (h, w), amp = CASES[name]
    prm = params.from_cli_numbers(numbers.split(), noc=1, nop=nop)
    stereo = nop == 1
    i0, i1, _ = synth.synthetic_pair(h, w, 1, seed=7, amp=amp, stereo=stereo)
    pyr = preprocess.PairPyramids(i0, i1, prm.sc_f, prm.p_samp_s)
    ctx = api.Context(prm, pyr.width, pyr.height, pyr.imgpadding, 1)
    ctx.set_option("patch_lanes", lanes)
    ctx.upload_pyramids(0, pyr)
    ctx.run(1)
    assert_bits(ctx.get_flow(0, prm.sc_l), oracle_port.port_run(pyr, prm), "run")
    ctx.close()
    if name.endswith("_partial_groups"):
        info = api.Context(prm, pyr.width, pyr.height, pyr.imgpadding, 1)
        li = info.level_info(prm.sc_l)
        info.close()
        n_p = li["nopw"] * li["noph"]
        assert n_p % 8 and n_p % 32, n_p
    if prm.usefbcon:  # the patch-stage checker is the plain grid; the merge is covered by the whole run above
        return
    ctx = api.Context(prm, pyr.width, pyr.height, pyr.imgpadding, 1)
    ctx.set_option("patch_lanes", lanes)
    ctx.upload_pyramids(0, pyr)
    lv = prm.sc_l
    hh, ww = pyr.level_shape(lv + 1)
    rng = np.random.default_rng(3)
    fp = (rng.standard_normal((hh, ww, prm.nop)) * (amp / 3)).astype(np.float32)
    if stereo:
        fp = -np.abs(fp)
    for init in (True, False):
        exp = oracle_port.port_level_patches(pyr, prm, lv, fp if init else None)
        ctx.set_flow(0, lv + 1, fp)
        ctx.patgrid_optimize(lv, 0, 1, init)
        ctx.patgrid_aggregate(lv, 0, 1)
        got = ctx.get_patches(0, lv)
        for k in ("p", "pweight", "conv", "cnt"):
            assert_bits(got[k], exp[k], "patch.%s (init from coarser: %s)" % (k, init))
        assert_bits(ctx.get_flow(0, lv), exp["dense"], "dense (init from coarser: %s)" % init)
    ctx.close()


@pytest.mark.parametrize("lanes", [4, 8, 0])
def test_batch_of_frames_and_graph_replay(lanes, api, oracle_port):
    """20 frames in one launch (more than 16: the default takes 4 lanes per patch there), 4 distinct pairs:
    eager against the oracle, graph replay against eager."""
    prm = params.from_cli_numbers(OP.format(pn=1, cf=0).split(), noc=1, nop=2)
    nfr, ndist = 20, 4
    pyrs = []
    for s in range(ndist):
        i0, i1, _ = synth.synthetic_pair(120, 200, 1, seed=30 + s, amp=6.0)
        pyrs.append(preprocess.PairPyramids(i0, i1, prm.sc_f, prm.p_samp_s))
    ctx = api.Context(prm, pyrs[0].width, pyrs[0].height, pyrs[0].imgpadding, nfr)
    ctx.set_option("patch_lanes", lanes)
    packed = np.stack([ctx.pack_frame(pyrs[f % ndist]) for f in range(nfr)])
    ctx.upload_packed(0, nfr, packed)
    ctx.run(nfr)
    eager = [ctx.get_flow(f, prm.sc_l) for f in range(nfr)]
    for d in range(ndist):
        assert_bits(eager[d], oracle_port.port_run(pyrs[d], prm), "pair %d" % d)
    for f in range(nfr):
        assert_bits(eager[f], eager[f % ndist], "frame %d" % f)
    ctx.set_graph_mode(True)
    ctx.run(nfr)
    ctx.run(nfr)
    for f in range(nfr):
        assert_bits(ctx.get_flow(f, prm.sc_l), eager[f], "graph frame %d" % f)
    ctx.close()


def test_option_values(api):
    prm = params.from_cli_numbers(OP.format(pn=1, cf=0).split(), noc=1, nop=2)
    ctx = api.Context(prm, 64, 64, prm.p_samp_s, 1)
    for v in (0, 4, 8):
        ctx.set_option("patch_lanes", v)
    for v in (1, 2, 16, -1):
        with pytest.raises(Exception):
            ctx.set_option("patch_lanes", v)
    ctx.close()
