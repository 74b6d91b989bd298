"""The device pyramids (pyr_from_u8_kernel, pyr_from_level_kernel, pyr_down_kernel, swap_images_kernel, sobel_kernel)
against the host pyramid, bitwise, on the GPU (pytest -m gpu).

For every geometry of tests/test_device_pyramid.py and every upload route that takes it, every array of every level
of every slot -- borders included, and with usefbcon also each slot's backward frame, which holds the swapped pair --
must equal preprocess.PairPyramids of the pair the slot holds.  The uploads go into a sub-range of the slots; the
slots outside it hold a sentinel pyramid that must come through unchanged.  Float images that round (and the deep
levels of large 8-bit frames) hold the device to build_pyramid's evaluation order, which tests/test_device_pyramid.py
proves those inputs can tell apart.  Finally every configuration of tests/test_batched_configs_gpu.py runs from the
8-bit upload, every slot bitwise the oracle's flow of its pair."""
import numpy as np
import pytest

from of_dis_b200 import preprocess
from test_batched_configs_gpu import CONFIGS, batched_inputs, oracle_flows, slot_pair
from test_device_pyramid import GEOMETRIES, bidir_range, clip_u8, float_pair, geometry_params, level_pyramids
from test_gpu_parity import _frames_u8, assert_bits
from test_patch_geometry_gpu import ROUTES, _check_slots, swapped, upload_by_route

pytestmark = pytest.mark.gpu
FLOAT_ROUTES = ("upload_packed_images", "upload_finest_level")


@pytest.fixture(scope="module")
def api():
    from of_dis_b200 import api as _api

    _api.lib()
    return _api


def _sentinel(g, prm):
    a, b = clip_u8(g, 2, 99)
    return preprocess.PairPyramids(a, b, prm.sc_f, g["pad"])


def _check_route(api, g, prm, route, pyrs, frames, sentinel):
    """`route` uploads pyrs (forward pairs) into its slot range of a context whose every slot first held the
    sentinel; then every slot's arrays (and backward frames) == its pair's, the others' the sentinel's"""
    if route == "upload_sequence_bidir_u8":
        f0, n = bidir_range(g)
        held = pyrs[:n] + [swapped(p) for p in pyrs[:n]]
    else:
        f0, n = g["f0"], g["n"]
        held = pyrs[:n]
    ctx = api.Context(prm, g["size"][1], g["size"][0], g["pad"], g["nfr"])
    try:
        for f in range(g["nfr"]):
            ctx.upload_pyramids(f, sentinel)
        upload_by_route(ctx, route, f0, pyrs[:n], frames)
        exp = [sentinel] * f0 + held + [sentinel] * (g["nfr"] - f0 - len(held))
        _check_slots(ctx, prm, exp, None, route, backward=bool(prm.usefbcon))
    finally:
        ctx.close()


def _routes(g, prm, routes=ROUTES):
    for r in routes:
        if r == "upload_packed" and prm.usefbcon:
            continue  # a packed frame has no gradients of the second image
        if r == "upload_sequence_bidir_u8" and bidir_range(g) is None:
            continue
        yield r


@pytest.mark.parametrize("name", list(GEOMETRIES))
def test_every_route_builds_the_host_pyramid_of_8bit_frames(name, api):
    g = GEOMETRIES[name]
    prm = geometry_params(g)
    n = max(g["n"], bidir_range(g)[1] if bidir_range(g) else 0)
    frames = clip_u8(g, n + 1, 3)
    pyrs = [preprocess.PairPyramids(frames[t], frames[t + 1], prm.sc_f, g["pad"]) for t in range(n)]
    sentinel = _sentinel(g, prm)
    for route in _routes(g, prm):
        _check_route(api, g, prm, route, pyrs, frames, sentinel)


@pytest.mark.parametrize("name", [k for k in GEOMETRIES if not k.startswith("deep_")])
def test_float_images_build_the_host_pyramid(name, api):
    """upload_finest_level and upload_packed_images of float images that round (test_device_pyramid.float_image):
    levels and gradients bitwise build_pyramid of the same float level."""
    g = GEOMETRIES[name]
    prm = geometry_params(g)
    n = min(g["n"], 3)
    pyrs = [level_pyramids(*float_pair(g, 50 + 2 * t), prm, g["pad"]) for t in range(n)]
    sentinel = _sentinel(g, prm)
    for route in FLOAT_ROUTES:
        _check_route(api, g, prm, route, pyrs, None, sentinel)


@pytest.mark.parametrize("name", list(CONFIGS))
def test_8bit_upload_runs_as_the_oracle(name, api, oracle_port):
    """The configurations of test_batched_configs_gpu.py from upload_frames_u8: every slot's level flow bitwise the
    oracle's flow of its pair (the pairs are independent, not a clip)."""
    cfg = CONFIGS[name]
    prm, pairs, pyrs = batched_inputs(name)
    exp = oracle_flows(name, oracle_port)
    nfr = cfg["nfr"]
    h, w = cfg["size"]
    ctx = api.Context(prm, pyrs[0].width, pyrs[0].height, pyrs[0].imgpadding, nfr)
    try:
        ctx.upload_frames_u8(0, nfr, _frames_u8([pairs[slot_pair(f)] for f in range(nfr)]), w, h)
        ctx.run(nfr)
        out = np.empty((nfr,) + exp[0].shape, np.float32)
        ctx.get_flow_batch(0, nfr, out)
        ctx.sync()
        for f in range(nfr):
            assert_bits(out[f], exp[slot_pair(f)], "slot %d" % f)
    finally:
        ctx.close()
