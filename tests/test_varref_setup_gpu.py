"""varref_setup_kernel against the oracle, bitwise: the derivative planes and the mask of a refinement without inner
iterations, and after one inner iteration also the SOR records and (du,dv) that the set-up kernel's first inner
iteration produced.  Gray and RGB, flow and stereo, each record layout (block wavefront, lane wavefront, fast mode),
1, 2 and 4 rows per thread (chosen by the frame count), levels whose last tile is partial in x and y, levels
narrower and shorter than the stages' halo, and the forward-only last level of usefbcon."""
import dataclasses

import numpy as np
import pytest

from of_dis_b200 import params, preprocess, synth

pytestmark = pytest.mark.gpu

CLI = "0 0 8 4 0.05 0.95 0 4 0.4 0 1 0 1 10 10 5 1 3 1.6 0"
# (h, w, frames, rows per thread assemble_rows_per_thread picks)
GEOMS = {"70x45_r1": (45, 70, 2, 1), "70x45_r2": (45, 70, 29, 2), "70x45_r4": (45, 70, 43, 4),
         "8x5_r1": (5, 8, 3, 1), "8x4_r1": (4, 8, 2, 1)}
KINDS = {"gray_flow": (1, 2), "rgb_flow": (3, 2), "gray_stereo": (1, 1), "rgb_stereo": (3, 1)}
MODES = {"wave": dict(sor_lane=0), "lane": dict(sor_lane=1), "fast": dict(sor_fast=1)}
N_PYR = 3  # distinct image pairs, cycled over the frames


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def assert_bits(got, exp, name):
    got, exp = np.asarray(got, np.float32), np.asarray(exp, np.float32)
    assert got.shape == exp.shape, (name, got.shape, exp.shape)
    bad = bits(got) != bits(exp)
    if bad.any():
        raise AssertionError("%s: %d of %d values differ bitwise, first at %s" %
                             (name, int(bad.sum()), bad.size, np.argwhere(bad)[0]))


@pytest.fixture(scope="module")
def api():
    from of_dis_b200 import api as _api

    _api.lib()
    return _api


def expected_records(it, nop):
    """the record fields debug_get("rec") returns, from the oracle's first inner iteration"""
    f32 = np.float32
    sh, sv = it["sh"], it["sv"]
    vt = np.zeros_like(sv)
    vt[1:] = sv[:-1]
    if nop == 2:
        return [it["a11_inv"], it["a12_inv"], it["a22_inv"], it["b1"], it["b2"], sh, sv, vt]
    hl = np.zeros_like(sh)
    hl[:, 1:] = sh[:, :-1]
    s = np.zeros_like(sh)  # sum of the neighbours' weights: top, left, bottom, right (zero where absent)
    for term in (vt, hl, sv, sh):
        s = (s + term).astype(f32)
    return [(it["a11_pre"] + s).astype(f32), it["b1"], sh, sv, vt]


def run_case(api, oracle_port, prm, h, w, nfr, opts, check_dudv):
    pyrs = []
    for s in range(N_PYR):
        i0, i1, _ = synth.synthetic_pair(h, w, prm.noc, seed=31 + s, amp=3.0, stereo=prm.nop == 1)
        pyrs.append(preprocess.PairPyramids(i0, i1, prm.sc_f, prm.p_samp_s))
    ctx = api.Context(prm, w, h, pyrs[0].imgpadding, nfr)
    try:
        for k, v in opts.items():
            ctx.set_option(k, v)
        for f in range(nfr):
            ctx.upload_pyramids(f, pyrs[f % N_PYR])
        lv = prm.sc_l
        rng = np.random.default_rng(7)
        flows = []
        for f in range(nfr):
            fl = (rng.standard_normal((h, w, prm.nop)) * 1.5).astype(np.float32)
            if prm.nop == 1:
                fl = -np.abs(fl)
            flows.append(fl)
        checked = sorted({0, 1, nfr - 1})
        oprm = dataclasses.replace(prm, usefbcon=0)
        exp = {f: oracle_port.varref_stages(pyrs[f % N_PYR], oprm, lv, flows[f], n_iters=1) for f in checked}
        for n_inner in (0, 1):
            for f in range(nfr):
                ctx.set_flow(f, lv, flows[f])
            ctx.varref_refine(lv, 0, nfr, n_inner=n_inner)
            ctx.sync()
            for f in checked:
                st, tag = exp[f], "frame %d n_inner %d" % (f, n_inner)
                for k in ("Ix", "Iy", "Iz", "Ixx", "Ixy", "Iyy", "Ixz", "Iyz"):
                    assert_bits(ctx.debug_get(k, f, lv), st[k], "%s %s" % (k, tag))
                assert_bits(ctx.debug_get("mask", f, lv)[0], st["mask"], "mask " + tag)
                if n_inner == 0:
                    continue
                it = st["iters"][0]
                rec = ctx.debug_get("rec", f, lv)
                for idx, e in enumerate(expected_records(it, prm.nop)):
                    assert_bits(rec[..., idx], e, "rec field %d %s" % (idx, tag))
                if check_dudv:
                    dudv = ctx.debug_get("dudv", f, lv)
                    assert_bits(dudv[..., 0], it["du"], "du " + tag)
                    if prm.nop == 2:
                        assert_bits(dudv[..., 1], it["dv"], "dv " + tag)
    finally:
        ctx.close()


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("geom", list(GEOMS))
def test_setup_and_first_iteration_vs_oracle(geom, kind, mode, api, oracle_port):
    h, w, nfr, rows = GEOMS[geom]
    noc, nop = KINDS[kind]
    prm = params.from_cli_numbers(CLI.split(), noc=noc, nop=nop)
    assert api.debug_sor_plan(w, h, nop, noc, prm.tv_solverit, nfr)["assemble_rows"] == rows
    # the red-black SOR of fast mode is not the reference's solver: its (du,dv) are checked by test_fast_mode.py
    run_case(api, oracle_port, prm, h, w, nfr, MODES[mode], check_dudv=mode != "fast")


@pytest.mark.parametrize("kind", ["gray_flow", "rgb_stereo"])
def test_setup_on_the_forward_only_last_level_of_usefbcon(kind, api, oracle_port):
    """usefbcon refines only the forward frames (every second internal frame) on the last level"""
    noc, nop = KINDS[kind]
    prm = dataclasses.replace(params.from_cli_numbers(CLI.split(), noc=noc, nop=nop), usefbcon=1)
    run_case(api, oracle_port, prm, 45, 70, 3, {}, check_dudv=True)
