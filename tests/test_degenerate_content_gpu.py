"""Degenerate image content on the GPU (pytest -m gpu): flat images, stripes, ramps, a 1-pixel checkerboard, a
rectangle moving on a flat background, independent noise, saturated and inverted frames, an RGB pair with one flat
channel, and one frame that tiles several of these together.  Smooth textured pairs never reach the data-dependent
fallbacks of the patch stage (PatClass::ComputeHessian + Eigen's LLT, patch.cpp:71-88), which every patch kernel
restates on its own; these inputs do:

    A  flow, det H == 0 with H00 == 0: both diagonals get +1e-10
    B  flow, det H == 0 with H00 > 0: the +1e-10 is absorbed, H stays singular
    C  flow, the Cholesky pivot H11 - L10^2 <= 0: L11 keeps H11
    D  stereo, H00 == 0

and with them patches that stop at cnt == 0 on an exactly zero residual, ratio tests that divide 0 by 0, flows of
exactly +0 and -0, and warps in which converged patches sit beside patches that still iterate.

For every (family, parameter set) -- parameter sets that route to each patch kernel: patch_p8c1_kernel with 8 and 4
lanes per patch, patch_p12_kernel (gray and RGB) and patch_optimize_kernel (P = 6, 16, and P = 8 RGB), flow and
stereo -- bitwise against the oracle (+0 and -0 differ): the patch stage at sc_l with and without initialisation from
a coarser flow, the refinement's planes after two inner iterations with both SOR kernels, and the whole run.  Then a
batch of more than 16 frames with the families mixed (the defaults switch to 4 lanes per patch and no dependent
launch there), eager and graph replay, and the device pyramid of 8-bit frames on flat and checkerboard content.

tests/test_oracle.py proves that the families reach the fallbacks on every patch kernel (the oracle's branch query)
and pins the oracle to the reference build on all of them (golden/reference_digests.json)."""
import dataclasses

import numpy as np
import pytest

from of_dis_b200 import params, preprocess
from test_gpu_parity import _frames_u8, assert_bits

pytestmark = pytest.mark.gpu
f32 = np.float32


# ---- the input families: deterministic numpy, (h, w) or (h, w, 3) uint8 pairs ----------------------------------
def _texture(h, w, seed):
    """a smooth seeded texture in [0, 255]: a sum of eight plane waves"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    acc = np.zeros((h, w))
    for _ in range(8):
        fx, fy = rng.uniform(-0.3, 0.3, 2)
        acc += np.sin(fx * x + fy * y + rng.uniform(0, 2 * np.pi))
    return (acc - acc.min()) / (acc.max() - acc.min()) * 255.0


def _moving_texture(h, w, seed, contrast=1.0):
    """a textured pair, I1 = I0 moved by (+2, +1) pixels (contrast > 1 saturates at 0 and 255)"""
    t = _texture(h + 8, w + 8, seed)
    t = np.clip((t - 127.5) * contrast + 127.5, 0, 255)
    return t[4:4 + h, 4:4 + w], t[3:3 + h, 2:2 + w]


def _gray_family(name, h, w):
    y, x = np.mgrid[0:h, 0:w]
    if name == "constant":
        return np.full((h, w), 128.0), np.full((h, w), 128.0)
    if name == "brightness":  # flat, brighter in the second frame
        return np.full((h, w), 100.0), np.full((h, w), 140.0)
    if name == "zero":
        return np.zeros((h, w)), np.zeros((h, w))
    if name == "checker":  # 1-pixel checkerboard, moved by one pixel: its gradients are zero, its levels >= 1 flat
        return ((x + y) & 1) * 255.0, ((x + y + 1) & 1) * 255.0
    if name == "vstripes":  # intensity varies along x only: gy == 0 (8-pixel period: gx != 0 on level 1 too)
        return ((x // 4) & 1) * 180.0 + 40, (((x + 1) // 4) & 1) * 180.0 + 40
    if name == "hramp":
        s = 230.0 / (w + 4)
        return 10 + s * x, 10 + s * (x + 2.5)
    if name == "hstripes":  # intensity varies along y only: gx == 0
        return ((y // 3) & 1) * 200.0 + 20, (((y + 1) // 3) & 1) * 200.0 + 20
    if name == "diag":  # 45-degree stripes, a function of x + y: gx == gy
        return (((x + y) // 3) & 1) * 200.0 + 30, (((x + y + 2) // 3) & 1) * 200.0 + 30
    if name == "rect":  # bright rectangle on a flat background, moved by (+3, +2)
        a, b = np.full((h, w), 60.0), np.full((h, w), 60.0)
        a[h // 4:h // 2, w // 4:w // 2] = 210
        b[h // 4 + 2:h // 2 + 2, w // 4 + 3:w // 2 + 3] = 210
        return a, b
    if name == "noise":  # independent uniform noise: nothing matches
        rng = np.random.default_rng(h * 1000 + w)
        return rng.integers(0, 256, (h, w)).astype(np.float64), rng.integers(0, 256, (h, w)).astype(np.float64)
    if name == "saturated":
        return _moving_texture(h, w, 5, contrast=5.0)
    if name == "inverted":  # a scene cut: the second frame is the negative of the first
        a, _ = _moving_texture(h, w, 6)
        return a, 255.0 - a
    if name == "textured":  # the regular case, for the mixed frame
        return _moving_texture(h, w, 7)
    if name == "mixed":  # 2 x 3 tiles: flat, stripes both ways, 45-degree stripes, texture, noise
        names = [["constant", "vstripes", "hstripes"], ["diag", "textured", "noise"]]
        a, b = np.zeros((h, w)), np.zeros((h, w))
        ys, xs = [0, h // 2, h], [0, w // 3, 2 * w // 3, w]
        for r in range(2):
            for c in range(3):
                ta, tb = _gray_family(names[r][c], ys[r + 1] - ys[r], xs[c + 1] - xs[c])
                a[ys[r]:ys[r + 1], xs[c]:xs[c + 1]] = ta
                b[ys[r]:ys[r + 1], xs[c]:xs[c + 1]] = tb
        return a, b
    raise KeyError(name)


def family_pair(name, h, w, ch):
    """The uint8 pair of family `name`: gray, or RGB with the same pattern in every channel ("one_flat_channel":
    channels 0 and 2 textured, channel 1 flat)."""
    if name == "one_flat_channel":
        assert ch == 3
        a0, b0 = _moving_texture(h, w, 8)
        a2, b2 = _moving_texture(h, w, 9)
        flat = np.full((h, w), 90.0)
        a, b = np.stack([a0, flat, a2], -1), np.stack([b0, flat, b2], -1)
    else:
        a, b = _gray_family(name, h, w)
        if ch == 3:
            a, b = np.repeat(a[..., None], 3, -1), np.repeat(b[..., None], 3, -1)
    q = lambda v: np.ascontiguousarray(np.clip(np.rint(v), 0, 255).astype(np.uint8))  # noqa: E731
    return q(a), q(b)


FAMILIES = ["constant", "brightness", "zero", "checker", "vstripes", "hramp", "hstripes", "diag", "rect", "noise",
            "saturated", "inverted", "one_flat_channel", "mixed"]

# ---- parameter sets, one or more per patch kernel --------------------------------------------------------------
# CLI numbers: sc_f sc_l max_iter min_iter dp_thresh dr_thresh res_thresh P patove usefbcon patnorm costfct usetvref
# alpha gamma delta innerit solverit omega verbosity.  name: (kernel, nop, channels, numbers, options, (h, w));
# level sizes: 96 x 160 -> 48 x 80 at sc_l = 1; 104 x 184 -> 13 x 23 at level 3; 99 x 165 is padded to 104 x 168.
# Sets with min_iter < max_iter evaluate the ratio tests, which divide 0 by 0 where a patch does not move (dp == 0).
ROUTES = {
    "p8_l8_flow": ("p8c1_l8", 2, 1, "3 1 12 12 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0", (("patch_lanes", 8),), (96, 160)),
    "p8_l4_flow": ("p8c1_l4", 2, 1, "3 1 12 4 0.05 0.95 0 8 0.4 0 0 2 1 10 10 5 1 3 1.6 0", (("patch_lanes", 4),), (104, 184)),
    "p8_l8_stereo": ("p8c1_l8", 1, 1, "3 1 12 3 0.05 0.95 0 8 0.4 0 1 1 1 10 10 5 1 3 1.6 0", (("patch_lanes", 8),), (99, 165)),
    "p8_l4_stereo": ("p8c1_l4", 1, 1, "3 1 12 12 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0", (("patch_lanes", 4),), (96, 160)),
    "p12_gray_flow": ("p12", 2, 1, "3 1 12 12 0.05 0.95 0 12 0.75 0 1 2 1 10 10 5 1 3 1.6 0", (), (104, 184)),
    "p12_gray_stereo": ("p12", 1, 1, "3 1 12 2 0.05 0.95 0 12 0.75 0 0 0 1 10 10 5 1 3 1.6 0", (), (96, 160)),
    "p12_rgb_flow": ("p12", 2, 3, "3 1 12 4 0.05 0.95 0 12 0.75 0 1 1 1 10 10 5 1 3 1.6 0", (), (96, 160)),
    "p12_rgb_stereo": ("p12", 1, 3, "3 1 12 12 0.05 0.95 0 12 0.75 0 1 0 1 10 10 5 1 3 1.6 0", (), (99, 165)),
    "p6_flow": ("generic", 2, 1, "3 1 8 8 0.05 0.95 0 6 0.5 0 0 0 1 10 10 5 2 5 1.5 0", (), (96, 160)),
    "p16_stereo_res_thresh": ("generic", 1, 1, "2 1 16 2 0.05 0.95 0.5 16 0.5 0 1 1 1 10 10 5 1 3 1.6 0", (), (104, 184)),
    "p8_rgb_flow_fbcon": ("generic", 2, 3, "3 1 8 8 0.05 0.95 0 8 0.4 1 1 0 1 10 10 5 1 3 1.6 0", (), (104, 184)),
    "p8_rgb_stereo": ("generic", 1, 3, "3 1 12 12 0.05 0.95 0 8 0.4 0 1 2 1 10 10 5 1 3 1.6 0", (), (96, 160)),
}

# (family, route) pairs: one_flat_channel is RGB only
CASES = [(f, r) for r in ROUTES for f in FAMILIES if f != "one_flat_channel" or ROUTES[r][2] == 3]
CASE_IDS = ["%s-%s" % c for c in CASES]


def degenerate_inputs(family, route):
    """(i0, i1, pyramids, parameters) of one case (shared with tests/test_oracle.py and tests/golden/make_golden.py)"""
    _, nop, ch, numbers, _, (h, w) = ROUTES[route]
    prm = params.from_cli_numbers(numbers.split(), noc=ch, nop=nop)
    i0, i1 = family_pair(family, h, w, ch)
    return i0, i1, preprocess.PairPyramids(i0, i1, prm.sc_f, prm.p_samp_s), prm


def stage_params(prm):
    """the parameters of the per-stage checks: the plain grid (the forward-backward merge is covered by the run)"""
    return dataclasses.replace(prm, usefbcon=0)


def coarser_flow(pyr, prm):
    """the flow of level sc_l + 1 the patch stage starts from: seeded, with a band of exact +0 and one of exact -0"""
    h, w = pyr.level_shape(prm.sc_l + 1)
    fl = (np.random.default_rng(4).standard_normal((h, w, prm.nop)) * 1.5).astype(f32)
    if prm.nop == 1:
        fl = -np.abs(fl)
    fl[:h // 3] = f32(0.0)
    fl[h // 3:2 * h // 3, :w // 2] = f32(-0.0)
    return fl


# ---- GPU tests ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def api():
    from of_dis_b200 import api as _api

    _api.lib()
    return _api


def _context(api, prm, pyr, opts, nfr=1):
    ctx = api.Context(prm, pyr.width, pyr.height, pyr.imgpadding, nfr)
    for k, v in opts:
        ctx.set_option(k, v)
    return ctx


@pytest.mark.parametrize("family,route", CASES, ids=CASE_IDS)
def test_patch_stage_refinement_and_run_vs_oracle(family, route, api, oracle_port):
    opts = ROUTES[route][4]
    _, _, pyr, prm = degenerate_inputs(family, route)
    sprm = stage_params(prm)
    lv = prm.sc_l
    fp = coarser_flow(pyr, prm)
    ctx = _context(api, sprm, pyr, opts)
    try:
        ctx.upload_pyramids(0, pyr)
        # patch stage (K1-K4) at sc_l; the dense flow of the initialised one feeds the refinement
        for init in (False, True):
            exp = oracle_port.port_level_patches(pyr, sprm, lv, fp if init else None)
            ctx.set_flow(0, lv + 1, fp)
            ctx.patgrid_optimize(lv, 0, 1, init)
            ctx.patgrid_aggregate(lv, 0, 1)
            got = ctx.get_patches(0, lv)
            for k in ("p", "pweight", "conv", "cnt"):
                assert_bits(got[k], exp[k], "patch.%s (init from coarser: %s)" % (k, init))
            dense = ctx.get_flow(0, lv)
            assert_bits(dense, exp["dense"], "dense (init from coarser: %s)" % init)
        # refinement (K5-K12) after two inner iterations, block and lane SOR
        st = oracle_port.varref_stages(pyr, sprm, lv, dense, n_iters=2)
        it = st["iters"][1]
        for lane in (0, 1):
            ctx.set_option("sor_lane", lane)
            ctx.set_flow(0, lv, dense)
            ctx.varref_refine(lv, 0, 1, n_inner=2)
            for k in ("Ix", "Iy", "Iz", "Ixx", "Ixy", "Iyy", "Ixz", "Iyz"):
                assert_bits(ctx.debug_get(k, 0, lv), st[k], "deriv.%s (sor_lane %d)" % (k, lane))
            assert_bits(ctx.debug_get("mask", 0, lv)[0], st["mask"], "mask (sor_lane %d)" % lane)
            rec = ctx.debug_get("rec", 0, lv)
            if prm.nop == 2:
                keys = ("a11_inv", "a12_inv", "a22_inv", "b1", "b2", "sh", "sv")
            else:
                keys = (None, "b1", "sh", "sv")
            for idx, key in enumerate(keys):
                if key:
                    assert_bits(rec[..., idx], it[key], "rec.%s (sor_lane %d)" % (key, lane))
            dudv = ctx.debug_get("dudv", 0, lv)
            assert_bits(dudv[..., 0], it["du"], "du (sor_lane %d)" % lane)
            if prm.nop == 2:
                assert_bits(dudv[..., 1], it["dv"], "dv (sor_lane %d)" % lane)
    finally:
        ctx.close()
    # whole run, with the route's own parameters (forward-backward merge included)
    ctx = _context(api, prm, pyr, opts)
    try:
        ctx.upload_pyramids(0, pyr)
        ctx.run(1)
        assert_bits(ctx.get_flow(0, prm.sc_l), oracle_port.port_run(pyr, prm), "run")
    finally:
        ctx.close()


@pytest.mark.parametrize("route", ["p8_l8_flow", "p8_l4_stereo", "p12_gray_flow"])
def test_batch_of_more_than_16_mixed_frames_eager_and_graph(route, api, oracle_port):
    """20 frames in one launch, one family per frame (every gray family, some twice), default options -- above 16
    frames those are 4 lanes per patch and no programmatic dependent launch: every frame against the oracle, graph
    replay against eager."""
    fams = [f for f in FAMILIES if f != "one_flat_channel"]
    nfr = 20
    pyrs = [degenerate_inputs(fams[f % len(fams)], route)[2] for f in range(nfr)]
    prm = degenerate_inputs(fams[0], route)[3]
    ctx = _context(api, prm, pyrs[0], (), nfr)
    try:
        ctx.upload_packed(0, nfr, np.stack([ctx.pack_frame(p) for p in pyrs]))
        ctx.run(nfr)
        eager = [ctx.get_flow(f, prm.sc_l) for f in range(nfr)]
        for f in range(len(fams)):
            assert_bits(eager[f], oracle_port.port_run(pyrs[f], prm), "frame %d (%s)" % (f, fams[f]))
        for f in range(len(fams), nfr):
            assert_bits(eager[f], eager[f % len(fams)], "frame %d" % f)
        ctx.set_graph_mode(True)
        for rep in range(2):
            ctx.run(nfr)
            for f in range(nfr):
                assert_bits(ctx.get_flow(f, prm.sc_l), eager[f], "graph replay %d, frame %d" % (rep, f))
    finally:
        ctx.close()


@pytest.mark.parametrize("size", [(96, 160), (101, 163)])
@pytest.mark.parametrize("ch", [1, 3])
@pytest.mark.parametrize("family", ["constant", "brightness", "zero", "checker"])
def test_device_pyramid_of_flat_and_checkerboard_frames(family, ch, size, api):
    """ofdis_upload_frames_u8 builds preprocess.PairPyramids bit for bit on flat frames and the 1-pixel checkerboard
    (whose box mean is a flat 127.5 from level 1 on), even and odd frame sizes."""
    prm = params.from_cli_numbers("3 1 8 8 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0".split(), noc=ch)
    h, w = size
    pairs = [family_pair(family, h, w, ch)]
    pyrs = [preprocess.PairPyramids(a, b, prm.sc_f, prm.p_samp_s) for a, b in pairs]
    if family == "checker":
        P = pyrs[0].imgpadding
        assert (pyrs[0].i0[1][P + 1:-P - 1, P + 1:-P - 1] == f32(127.5)).all()
    ctx = api.Context(prm, pyrs[0].width, pyrs[0].height, pyrs[0].imgpadding, 1)
    try:
        ctx.upload_frames_u8(0, 1, _frames_u8(pairs), w, h)
        for lv in range(prm.sc_l, prm.sc_f + 1):
            for which, exp in enumerate((pyrs[0].i0[lv], pyrs[0].i0x[lv], pyrs[0].i0y[lv], pyrs[0].i1[lv])):
                assert_bits(ctx.get_level(0, lv, which), exp, "level %d array %d" % (lv, which))
    finally:
        ctx.close()
