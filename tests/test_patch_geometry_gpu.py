"""Image paddings wider than the patch, and patch sizes outside the parameter sweeps, on the GPU (pytest -m gpu).

ofdis_create takes any imgpadding >= p_samp_s, as the reference's OFClass does, and the padding enters the address
arithmetic of every kernel that reads a padded image: the patch kernels' template and window bases (and the P = 8
gray kernel's paired loads, whose alignment comes from the address), the warp of the refinement, Sobel and the device
pyramids, the swapped copies of usefbcon and the packed-frame offsets.  A kernel that used P where it means the
padding, or the reverse, would pass every test that pads by P.  Every read of the reference lies within P of the
image, so the flow at any padding is the flow at padding P: the oracle on PairPyramids(..., pad) is the exact answer,
and the GPU's result must also equal the oracle at pad = P.

ofdis_create also takes any even p_samp_s >= 2 with noc * P^2 % 4 == 0.  The patch size picks the patch kernel and,
for the generic kernel (patch_optimize_kernel), the threads per CTA (256 down to 32) and the fold of the partial sums
(full packets of 8, and a tail of 4 where noc * P^2 % 8 == 4; P = 2 gray has the tail only).  SIZE_CASES reaches
every one of these (tests/test_patch_geometry.py asserts it with generic_launch, which restates the launcher), up to
the largest sizes ofdis_create accepts: RGB P = 30 and gray P = 52, each with a coarsest level narrower than the
patch.

Checks, all bitwise against the oracle: the patch stage at sc_l from a prescribed coarser flow, the refinement's
planes after two inner iterations, and the whole run -- at paddings P+1, P+2, P+3 and 2P on every patch kernel, and at
every patch size of SIZE_CASES; every upload path at a padding other than P, pyramid arrays and flows; a batch of more
than 16 frames with graph replay; the Python OFClass mirror.  tests/test_patch_geometry.py pins the oracle to the
reference build on all of these inputs (golden/reference_digests.json)."""
import dataclasses
import types

import numpy as np
import pytest

from of_dis_b200 import params, preprocess, synth
from test_gpu_parity import _frames_u8, assert_bits
from test_initflow_gpu import set_direction

pytestmark = pytest.mark.gpu
f32 = np.float32


# ---- the launcher's arithmetic (patch_kernels.cu launch_patch_optimize, ofdis_internal.cuh patch_generic_threads) --
def patch_kernel(noc, P):
    """the patch kernel that launch_patch_optimize takes for a patch size (the padding is always >= P, so the P = 12
    kernel's gate pad >= 12 always holds)"""
    if P == 8 and noc == 1:
        return "p8c1"
    if P == 12:
        return "p12"
    return "generic"


def generic_launch(noc, P):
    """patch_optimize_kernel's launch: (threads per CTA, dynamic shared memory in bytes, noc * P^2 % 8, full packets
    of 8 values per lane nk).  Five columns of NK slots per thread, NK = nk plus one for a tail of 4; 256 threads,
    halved while that exceeds 200 KB, down to 32."""
    n = noc * P * P
    nk = n // 8
    NK = nk + (1 if n % 8 >= 4 else 0)
    threads = 256
    while threads > 32 and 5 * NK * threads * 4 > 200 * 1024:
        threads //= 2
    return threads, 5 * NK * threads * 4, n % 8, nk


# ---- cases ---------------------------------------------------------------------------------------------------------
# CLI numbers: sc_f sc_l max_iter min_iter dp_thresh dr_thresh res_thresh P patove usefbcon patnorm costfct usetvref
# alpha gamma delta innerit solverit omega verbosity.  Level sizes: 104 x 184 -> 13 x 23 at level 3 (odd width, so an
# odd padded width at every padding); 99 x 165 and 101 x 163 are padded to multiples of 2^sc_f.
# name: (patch kernel and options, nop, channels, numbers, options, (h, w))
PAD_ROUTES = {
    "p8_l8_flow_fb": ("p8c1_l8", 2, 1, "3 1 10 10 0.05 0.95 0 8 0.4 1 1 0 1 10 10 5 1 3 1.6 0", (("patch_lanes", 8),), (104, 184)),
    "p8_l4_stereo_fb": ("p8c1_l4", 1, 1, "3 1 12 4 0.05 0.95 0 8 0.4 1 1 1 1 10 10 5 1 3 1.6 0", (("patch_lanes", 4),), (96, 168)),
    "p8_l4_flow": ("p8c1_l4", 2, 1, "3 1 12 12 0.05 0.95 0 8 0.4 0 0 2 1 10 10 5 1 3 1.6 0", (("patch_lanes", 4),), (104, 184)),
    "p12_gray_flow_fb": ("p12", 2, 1, "3 1 12 12 0.05 0.95 0 12 0.75 1 1 2 1 10 10 5 1 3 1.6 0", (), (104, 184)),
    "p12_rgb_stereo": ("p12", 1, 3, "3 1 12 4 0.05 0.95 0 12 0.75 0 1 0 1 10 10 5 1 3 1.6 0", (), (96, 160)),
    "p12_rgb_flow_fb": ("p12", 2, 3, "2 0 8 8 0.05 0.95 0 12 0.6 1 1 1 1 10 10 5 1 3 1.6 0", (), (72, 120)),
    "p6_rgb_flow_fb": ("generic", 2, 3, "3 1 8 8 0.05 0.95 0 6 0.5 1 0 0 1 10 10 5 2 5 1.5 0", (), (104, 184)),
    "p16_gray_stereo_fb": ("generic", 1, 1, "2 0 12 3 0.05 0.95 0 16 0.5 1 1 1 1 10 10 5 1 3 1.6 0", (), (88, 152)),
    "p16_gray_flow": ("generic", 2, 1, "3 1 16 2 0.05 0.95 0.5 16 0.5 0 1 0 1 10 10 5 1 3 1.6 0", (), (104, 184)),
}
# paddings relative to the patch size: odd and even, and one twice the patch
PADS = {"P+1": lambda P: P + 1, "P+2": lambda P: P + 2, "P+3": lambda P: P + 3, "2P": lambda P: 2 * P}
PAD_CASES = [(r, p) for r in PAD_ROUTES for p in PADS]
PAD_IDS = ["%s-%s" % c for c in PAD_CASES]

# name: (nop, channels, numbers, (h, w)); the padding is P.  Generic launches (generic_launch): P = 2 gray 256 threads,
# n % 8 == 4 with nk == 0 (the tail only); P = 2 RGB 256, 4, one packet and a tail; RGB 14: 128, 4; RGB 18: 64, 4;
# RGB 20: 64, 0; RGB 22, 26 and 30: 32, 4; RGB 24: 32, 0; gray 14: 256, 4; gray 18: 128, 4; gray 24: 128, 0;
# gray 36 and 52: 32, 0.  RGB 30 and gray 52 are the largest sizes ofdis_create accepts.
SIZE_CASES = {
    "p2_gray_flow": (2, 1, "3 1 8 8 0.05 0.95 0 2 0.5 0 1 0 1 10 10 5 1 3 1.6 0", (64, 96)),
    "p2_rgb_stereo_fb": (1, 3, "3 1 8 4 0.05 0.95 0 2 0 1 1 1 1 10 10 5 1 3 1.6 0", (64, 96)),
    "p14_rgb_flow_fb": (2, 3, "3 1 8 8 0.05 0.95 0 14 0.5 1 1 0 1 10 10 5 1 3 1.6 0", (96, 160)),
    "p18_rgb_stereo": (1, 3, "3 1 8 8 0.05 0.95 0 18 0.5 0 1 2 1 10 10 5 1 3 1.6 0", (96, 160)),
    "p20_rgb_flow": (2, 3, "2 1 8 4 0.05 0.95 0 20 0.6 0 0 1 1 10 10 5 1 3 1.6 0", (96, 160)),
    "p22_rgb_stereo_fb": (1, 3, "2 0 6 6 0.05 0.95 0 22 0.5 1 1 0 1 10 10 5 1 3 1.6 0", (64, 96)),
    "p24_rgb_flow_fb": (2, 3, "2 0 8 8 0.05 0.95 0 24 0.5 1 1 0 1 10 10 5 1 3 1.6 0", (80, 128)),
    "p26_rgb_flow": (2, 3, "2 0 8 3 0.05 0.95 0 26 0.5 0 1 1 1 10 10 5 1 3 1.6 0", (80, 128)),
    "p30_rgb_flow_fb": (2, 3, "3 1 8 8 0.05 0.95 0 30 0.5 1 1 0 1 10 10 5 1 3 1.6 0", (96, 160)),
    "p14_gray_stereo_fb": (1, 1, "3 1 12 12 0.05 0.95 0 14 0.5 1 1 0 1 10 10 5 1 3 1.6 0", (96, 160)),
    "p18_gray_flow_fb": (2, 1, "3 1 10 4 0.05 0.95 0 18 0.5 1 0 2 1 10 10 5 1 3 1.6 0", (96, 160)),
    "p24_gray_stereo": (1, 1, "2 0 8 8 0.05 0.95 0 24 0.5 0 1 0 1 10 10 5 1 3 1.6 0", (80, 128)),
    "p36_gray_flow_fb": (2, 1, "2 0 8 8 0.05 0.95 0 36 0.5 1 1 1 1 10 10 5 1 3 1.6 0", (80, 128)),
    "p52_gray_flow": (2, 1, "2 0 8 8 0.05 0.95 0 52 0.5 0 1 0 1 10 10 5 1 3 1.6 0", (96, 160)),
}

# every upload path at a padding other than P: name: (nop, channels, numbers, padding, (h, w)); three pairs of a clip
UPLOAD_CASES = {
    "p8_gray_flow_pad11": (2, 1, "3 1 8 8 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 11, (99, 165)),
    "p6_rgb_flow_fb_pad12": (2, 3, "3 1 8 8 0.05 0.95 0 6 0.5 1 0 0 1 10 10 5 2 5 1.5 0", 12, (101, 163)),
    "p12_gray_stereo_pad13": (1, 1, "3 1 12 4 0.05 0.95 0 12 0.75 0 1 1 1 10 10 5 1 3 1.6 0", 13, (96, 170)),
}
UPLOAD_PAIRS = 3
# every route into the device pyramids: the host pyramids (upload_pyramids, upload_packed), host images with the
# gradients (and usefbcon's swapped copies) derived on the device, float images of level sc_l, and 8-bit frames
ROUTES = ("upload_pyramids", "upload_packed", "upload_packed_images", "upload_finest_level", "upload_frames_u8",
          "upload_sequence_u8", "upload_sequence_bidir_u8")

# a batch of more than 16 frames (4 lanes per patch, no dependent launch, the other SOR plans): BATCH_DISTINCT pairs
# cycled over BATCH_FRAMES slots, padding 2P
BATCH_CLI = "3 1 8 8 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0"
BATCH_FRAMES, BATCH_DISTINCT, BATCH_SIZE = 18, 6, (96, 160)


# ---- inputs (shared with tests/test_patch_geometry.py and tests/golden/make_golden.py) ----------------------------
def pad_inputs(route, pad_name):
    """(i0, i1, pyramids at the padding, pyramids at padding P, parameters) of one padding case"""
    _, nop, ch, numbers, _, (h, w) = PAD_ROUTES[route]
    prm = params.from_cli_numbers(numbers.split(), noc=ch, nop=nop)
    i0, i1, _ = synth.synthetic_pair(h, w, ch, seed=300 + list(PAD_ROUTES).index(route), amp=4.0, stereo=(nop == 1))
    pad = PADS[pad_name](prm.p_samp_s)
    return (i0, i1, preprocess.PairPyramids(i0, i1, prm.sc_f, pad), preprocess.PairPyramids(i0, i1, prm.sc_f, prm.p_samp_s),
            prm)


def size_inputs(name):
    """(i0, i1, pyramids, parameters) of one patch-size case"""
    nop, ch, numbers, (h, w) = SIZE_CASES[name]
    prm = params.from_cli_numbers(numbers.split(), noc=ch, nop=nop)
    i0, i1, _ = synth.synthetic_pair(h, w, ch, seed=320 + list(SIZE_CASES).index(name), amp=4.0, stereo=(nop == 1))
    return i0, i1, preprocess.PairPyramids(i0, i1, prm.sc_f, prm.p_samp_s), prm


def upload_inputs(name):
    """(parameters, padding, clip of UPLOAD_PAIRS + 1 frames, pyramids of the forward pairs, of the backward pairs)"""
    nop, ch, numbers, pad, (h, w) = UPLOAD_CASES[name]
    prm = params.from_cli_numbers(numbers.split(), noc=ch, nop=nop)
    frames = synth.synthetic_sequence(UPLOAD_PAIRS + 1, h, w, ch, seed=340 + list(UPLOAD_CASES).index(name), amp=3.0,
                                      stereo=(nop == 1))
    fwd = [preprocess.PairPyramids(frames[t], frames[t + 1], prm.sc_f, pad) for t in range(UPLOAD_PAIRS)]
    bwd = [preprocess.PairPyramids(frames[t + 1], frames[t], prm.sc_f, pad) for t in range(UPLOAD_PAIRS)]
    return prm, pad, frames, fwd, bwd


def batch_inputs():
    """(parameters, the distinct pairs, their pyramids at padding 2P)"""
    prm = params.from_cli_numbers(BATCH_CLI.split())
    pairs = [synth.synthetic_pair(*BATCH_SIZE, 1, seed=360 + d, amp=4.0)[:2] for d in range(BATCH_DISTINCT)]
    return prm, pairs, [preprocess.PairPyramids(a, b, prm.sc_f, 2 * prm.p_samp_s) for a, b in pairs]


def stage_params(prm):
    """the parameters of the per-stage checks: the plain grid (the forward-backward merge is covered by the run)"""
    return dataclasses.replace(prm, usefbcon=0)


def coarser_flow(pyr, prm):
    """the seeded flow of level sc_l + 1 the patch stage starts from"""
    h, w = pyr.level_shape(prm.sc_l + 1)
    fl = (np.random.default_rng(8).standard_normal((h, w, prm.nop)) * 2).astype(f32)
    return -np.abs(fl) if prm.nop == 1 else fl


# ---- GPU tests ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def api():
    from of_dis_b200 import api as _api

    _api.lib()
    return _api


def _context(api, prm, pyr, opts=(), nfr=1):
    ctx = api.Context(prm, pyr.width, pyr.height, pyr.imgpadding, nfr)
    for k, v in opts:
        ctx.set_option(k, v)
    return ctx


def check_stages_and_run(api, oracle_port, pyr, prm, opts, refine):
    """The patch stage at sc_l from coarser_flow, the refinement's planes after two inner iterations (refine) and the
    whole run, in a context of the pyramids' padding, bitwise against the oracle.  Returns (patch stage, run flow)."""
    sprm = stage_params(prm)
    lv = prm.sc_l
    ctx = _context(api, sprm, pyr, opts)
    try:
        ctx.upload_pyramids(0, pyr)
        exp = oracle_port.port_level_patches(pyr, sprm, lv, coarser_flow(pyr, prm))
        ctx.set_flow(0, lv + 1, coarser_flow(pyr, prm))
        ctx.patgrid_optimize(lv, 0, 1, True)
        ctx.patgrid_aggregate(lv, 0, 1)
        got = ctx.get_patches(0, lv)
        for k in ("p", "pweight", "conv", "cnt"):
            assert_bits(got[k], exp[k], "patch." + k)
        got["dense"] = ctx.get_flow(0, lv)
        assert_bits(got["dense"], exp["dense"], "dense")
        if refine:
            st = oracle_port.varref_stages(pyr, sprm, lv, got["dense"], n_iters=2)
            ctx.varref_refine(lv, 0, 1, n_inner=2)
            for k in ("Ix", "Iy", "Iz", "Ixx", "Ixy", "Iyy", "Ixz", "Iyz"):
                assert_bits(ctx.debug_get(k, 0, lv), st[k], "deriv." + k)
            assert_bits(ctx.debug_get("mask", 0, lv)[0], st["mask"], "mask")
            rec = ctx.debug_get("rec", 0, lv)
            it = st["iters"][1]
            keys = ("a11_inv", "a12_inv", "a22_inv", "b1", "b2", "sh", "sv") if prm.nop == 2 else (None, "b1", "sh", "sv")
            for idx, key in enumerate(keys):
                if key:
                    assert_bits(rec[..., idx], it[key], "rec." + key)
            dudv = ctx.debug_get("dudv", 0, lv)
            assert_bits(dudv[..., 0], it["du"], "du")
            if prm.nop == 2:
                assert_bits(dudv[..., 1], it["dv"], "dv")
    finally:
        ctx.close()
    ctx = _context(api, prm, pyr, opts)
    try:
        ctx.upload_pyramids(0, pyr)
        ctx.run(1)
        flow = ctx.get_flow(0, prm.sc_l)
    finally:
        ctx.close()
    assert_bits(flow, oracle_port.port_run(pyr, prm), "run")
    return got, flow


@pytest.mark.parametrize("route,pad", PAD_CASES, ids=PAD_IDS)
def test_wider_padding_stages_and_run_vs_oracle(route, pad, api, oracle_port):
    """Every patch kernel at paddings P+1, P+2, P+3 and 2P: the oracle on the pyramids of that padding, and the
    oracle at padding P (the same context geometry otherwise)."""
    _, _, pyr, pyr_p, prm = pad_inputs(route, pad)
    assert pyr.imgpadding != prm.p_samp_s
    got, flow = check_stages_and_run(api, oracle_port, pyr, prm, PAD_ROUTES[route][4], refine=True)
    exp = oracle_port.port_level_patches(pyr_p, stage_params(prm), prm.sc_l, coarser_flow(pyr_p, prm))
    for k in ("p", "pweight", "conv", "cnt", "dense"):
        assert_bits(got[k], exp[k], "patch.%s against padding P" % k)
    assert_bits(flow, oracle_port.port_run(pyr_p, prm), "run against padding P")


@pytest.mark.parametrize("name", list(SIZE_CASES))
def test_patch_sizes_stages_and_run_vs_oracle(name, api, oracle_port):
    """Patch sizes 2 to 52: every thread count and fold of the generic patch kernel, the largest sizes accepted."""
    _, _, pyr, prm = size_inputs(name)
    check_stages_and_run(api, oracle_port, pyr, prm, (), refine=False)


def _levels(prm, pyr):
    for lv in range(prm.sc_l, prm.sc_f + 1):
        for which, arr in enumerate((pyr.i0[lv], pyr.i0x[lv], pyr.i0y[lv], pyr.i1[lv])):
            yield lv, which, arr


def swapped(pyr):
    """the pyramids of the swapped pair: what a usefbcon context holds in the backward frame of a pair"""
    return types.SimpleNamespace(i0=pyr.i1, i0x=pyr.i1x, i0y=pyr.i1y, i1=pyr.i0, i1x=pyr.i0x, i1y=pyr.i0y)


def _check_slots(ctx, prm, pyrs, exp, path, f0=0, backward=False):
    """every level and array of slots f0.. == their pyramids, with `backward` (usefbcon) also every array of their
    backward frames == the swapped pair's; after a run, every flow == exp (None: not checked; exp None: no run)"""
    for f, p in enumerate(pyrs):
        for lv, which, arr in _levels(prm, p):
            assert_bits(ctx.get_level(f0 + f, lv, which), arr, "%s: slot %d level %d array %d" % (path, f0 + f, lv, which))
    if backward:
        from of_dis_b200 import api

        set_direction(api, ctx, 1)
        try:
            for f, p in enumerate(pyrs):
                for lv, which, arr in _levels(prm, swapped(p)):
                    assert_bits(ctx.get_level(f0 + f, lv, which), arr,
                                "%s: backward frame of slot %d level %d array %d" % (path, f0 + f, lv, which))
        finally:
            set_direction(api, ctx, -1)
    if exp is None:
        return
    ctx.run(ctx.max_frames)
    for f, e in enumerate(exp):
        if e is not None:
            assert_bits(ctx.get_flow(f0 + f, prm.sc_l), e, "%s: flow of slot %d" % (path, f0 + f))


def upload_by_route(ctx, route, f0, pyrs, frames=None):
    """Uploads pairs t < len(pyrs) into slots f0 + t by `route` (one of ROUTES); pyrs[t]: the pair's pyramids at the
    context's padding, frames: the 8-bit clip whose frames t, t + 1 are pair t (the 8-bit routes only).
    upload_sequence_bidir_u8 also uploads the swapped pairs into slots f0 + n + t."""
    n, lv, pad = len(pyrs), ctx.prm.sc_l, ctx.pad
    if route == "upload_pyramids":
        for t, p in enumerate(pyrs):
            ctx.upload_pyramids(f0 + t, p)
    elif route == "upload_packed":
        ctx.upload_packed(f0, f0 + n, np.stack([ctx.pack_frame(p) for p in pyrs]))
    elif route == "upload_packed_images":
        ctx.upload_packed_images(f0, f0 + n, np.ascontiguousarray(
            np.stack([ctx.pack_frame(p)[:ctx.packed_images_frame_floats] for p in pyrs])))
    elif route == "upload_finest_level":
        ctx.upload_finest_level(f0, f0 + n, np.ascontiguousarray(
            np.stack([np.stack([p.i0[lv][pad:-pad, pad:-pad], p.i1[lv][pad:-pad, pad:-pad]]) for p in pyrs])))
    else:
        h, w = frames.shape[1:3]
        if route == "upload_frames_u8":
            ctx.upload_frames_u8(f0, f0 + n, _frames_u8([(frames[t], frames[t + 1]) for t in range(n)]), w, h)
        elif route == "upload_sequence_u8":
            ctx.upload_sequence_u8(f0, f0 + n, np.ascontiguousarray(frames[:n + 1]), w, h)
        else:
            assert route == "upload_sequence_bidir_u8", route
            ctx.upload_sequence_bidir_u8(f0, n, np.ascontiguousarray(frames[:n + 1]), w, h)


@pytest.mark.parametrize("name", list(UPLOAD_CASES))
def test_every_upload_path_at_a_wider_padding(name, api, oracle_port):
    """upload_pyramids, upload_packed (not with usefbcon), upload_packed_images, upload_finest_level, upload_frames_u8,
    upload_sequence_u8 and upload_sequence_bidir_u8 into contexts padded by more than P: every slot's pyramid arrays
    == PairPyramids(..., pad) bit for bit, and every flow == the oracle's."""
    from test_bidir_gpu import _right_camera_oracle

    prm, pad, frames, fwd, bwd = upload_inputs(name)
    assert pad != prm.p_samp_s
    n = UPLOAD_PAIRS
    exp = [oracle_port.port_run(p, prm) for p in fwd]
    # stereo: the backward slots run as the right camera (the oracle's level loop as the right camera, without usefbcon)
    exp_bwd = [oracle_port.port_run(p, prm) if prm.nop == 2 else
               (_right_camera_oracle(p, prm) if not prm.usefbcon else None) for p in bwd]
    for route in ROUTES:
        if route == "upload_packed" and prm.usefbcon:
            continue
        bidir = route == "upload_sequence_bidir_u8"
        ctx = _context(api, prm, fwd[0], (), 2 * n if bidir else n)
        try:
            upload_by_route(ctx, route, 0, fwd, frames)
            _check_slots(ctx, prm, fwd + bwd if bidir else fwd, exp + exp_bwd if bidir else exp, route)
        finally:
            ctx.close()


def test_batch_of_more_than_16_frames_at_twice_the_padding_eager_and_graph(api, oracle_port):
    """18 frames padded by 2P in one launch (4 lanes per patch and no dependent launch above 16 frames), from the packed
    upload: every distinct pair against the oracle, every slot against its pair, graph replay against eager."""
    prm, pairs, pyrs = batch_inputs()
    exp = [oracle_port.port_run(p, prm) for p in pyrs]
    ctx = _context(api, prm, pyrs[0], (), BATCH_FRAMES)
    try:
        ctx.upload_packed(0, BATCH_FRAMES, np.stack([ctx.pack_frame(pyrs[f % BATCH_DISTINCT]) for f in range(BATCH_FRAMES)]))
        ctx.run(BATCH_FRAMES)
        for f in range(BATCH_FRAMES):
            assert_bits(ctx.get_flow(f, prm.sc_l), exp[f % BATCH_DISTINCT], "eager, frame %d" % f)
        ctx.set_graph_mode(True)
        for rep in range(2):
            ctx.run(BATCH_FRAMES)
            for f in range(BATCH_FRAMES):
                assert_bits(ctx.get_flow(f, prm.sc_l), exp[f % BATCH_DISTINCT], "graph replay %d, frame %d" % (rep, f))
    finally:
        ctx.close()


@pytest.mark.parametrize("route", ["p8_l8_flow_fb", "p12_rgb_stereo"])
def test_ofclass_mirror_with_a_wider_padding(route, api, oracle_port):
    """api.OFClass, the reference-shaped constructor, with imgpadding = P + 3 (usefbcon's six arrays included)."""
    _, _, pyr, _, prm = pad_inputs(route, "P+3")
    out = np.zeros(pyr.level_shape(prm.sc_l) + (prm.nop,), f32)
    api.OFClass(pyr.i0, pyr.i0x, pyr.i0y, pyr.i1, pyr.i1x, pyr.i1y, pyr.imgpadding, out, None, pyr.width, pyr.height,
                prm.sc_f, prm.sc_l, prm.max_iter, prm.min_iter, prm.dp_thresh, prm.dr_thresh, prm.res_thresh,
                prm.p_samp_s, prm.patove, prm.usefbcon, prm.costfct, prm.noc, prm.patnorm, prm.usetvref, prm.tv_alpha,
                prm.tv_gamma, prm.tv_delta, prm.tv_innerit, prm.tv_solverit, prm.tv_sor, 0, nop=prm.nop)
    assert_bits(out, oracle_port.port_run(pyr, prm), "OFClass, imgpadding %d" % pyr.imgpadding)
