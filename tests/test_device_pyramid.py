"""The geometries and inputs the device pyramids are checked on (tests/test_device_pyramid_gpu.py), and the proof on
the host that those inputs can tell one evaluation order from another.

The device builds the pyramid of every 8-bit and float upload with the arithmetic of preprocess.build_pyramid: the 2x2
box mean ((a + b) + (c + d)) * 0.25 and the Sobel/8 sums (t0 * 0.125 + t1 * 0.25) + t2 * 0.125 of the row
differences, and (p0 * 0.125 + p1 * 0.25) + p2 * 0.125 of the smoothed rows before their difference.  On the
shallow levels of 8-bit frames every intermediate is a short dyadic rational that float32 holds exactly, so any
association order gives the same bits there and a bitwise check proves nothing about the order.  Full-mantissa
float images and the deep levels (8 and beyond) of large 8-bit frames round, and there the order decides the bits:
this file asserts that other orders differ from build_pyramid on those inputs and agree with it on the shallow ones,
and that build_pyramid is the operation itself -- within the float32 rounding of its expression of a float64 box
mean and Sobel/8."""
import numpy as np
import pytest

from of_dis_b200 import params, preprocess
from test_batched_configs_gpu import random_batched_config

f32 = np.float32
U = 2.0 ** -24  # float32's unit roundoff
N_RANDOM = 18


# ---- geometries ----------------------------------------------------------------------------------------------------
def _cli(sc_f, sc_l, P=8, fb=0, tvref=1):
    """the 20 command-line numbers (run_dense.cpp) of a pyramid geometry"""
    return [sc_f, sc_l, 8, 8, 0.05, 0.95, 0.0, P, 0.4, fb, 1, 0, tvref, 10.0, 10.0, 5.0, 1, 3, 1.6, 0]


def _odd_padding(rng, sc_f):
    """an odd divisibility padding below 2^sc_f: floor(pad / 2) and ceil(pad / 2) differ (0 where sc_f is 0)"""
    return int(rng.integers(0, 1 << (sc_f - 1))) * 2 + 1 if sc_f else 0


def _geometry(numbers, ch, nop, size, nfr, f0, n, pad, org=None, rng=None):
    """size: the context's (rows, columns) of level 0; org: the 8-bit frames' (rows, columns), by default size less an
    odd padding in both directions; pairs t < n go into slots f0 + t of a context of nfr slots padded by `pad`."""
    if org is None:
        org = tuple(s - _odd_padding(rng, numbers[0]) for s in size)
    return dict(numbers=numbers, ch=ch, nop=nop, size=size, org=org, nfr=nfr, f0=f0, n=n, pad=pad)


def random_geometry(seed):
    """The level geometries, channels, flow kind and frames per launch of random_batched_config(seed) with odd
    divisibility paddings, usefbcon on every third draw (and where the draw has it), the padding P, P + 1 or P + 2,
    and the uploads into its stage sub-range [f0, f1)."""
    cfg = random_batched_config(seed)
    rng = np.random.default_rng(7000 + seed)
    numbers = list(cfg["numbers"])
    numbers[9] = 1 if seed % 3 == 0 else numbers[9]
    f0, f1, _ = cfg["stage"]
    return _geometry(numbers, cfg["ch"], cfg["nop"], cfg["size"], cfg["nfr"], f0, f1 - f0, numbers[7] + seed % 3,
                     rng=rng)


def _named(sc_f, sc_l, ch, size, nfr, f0, n, fb=0, P=8, tvref=1, org=None, seed=0):
    return _geometry(_cli(sc_f, sc_l, P, fb, tvref), ch, 2, size, nfr, f0, n, P + 1, org, np.random.default_rng(seed))


NAMED = {
    "coarsest_2_columns": _named(3, 0, 1, (56, 16), 4, 1, 2, fb=1, seed=1),
    "coarsest_4_rows": _named(4, 1, 3, (64, 208), 3, 1, 1, seed=2),
    "sc_l0_sc_f5": _named(5, 0, 1, (160, 224), 3, 1, 1, fb=1, seed=3),
    "sc_l2_sc_f5": _named(5, 2, 3, (192, 288), 5, 2, 2, seed=4),
    "sc_l3_sc_f5": _named(5, 3, 1, (128, 160), 4, 1, 2, fb=1, P=4, seed=5),
    "tall_2602_rows": _named(1, 0, 1, (2602, 26), 3, 1, 1, fb=1, seed=6),
    # the deep levels of large frames, whose Sobel sums (levels >= 8) and box means (>= 9) round; one pair each
    "deep_sc_f9_2048x1024": _named(9, 0, 1, (2048, 1024), 2, 0, 1, tvref=0, org=(2048, 1024)),
    "deep_sc_f10_4096x2048": _named(10, 2, 1, (4096, 2048), 2, 0, 1, tvref=0, org=(4096, 2048)),
    # the deepest level the 8-bit uploads start from
    "rgb_sc_l8": _named(9, 8, 3, (2048, 1536), 3, 1, 1, fb=1, seed=7),
    "frames_64": _named(1, 0, 1, (24, 40), 64, 1, 63, seed=8),
    # odd frame counts of the sequence uploads: n pairs from n + 1 frames, the two-way upload into 2n slots
    "clip_n1": _named(2, 0, 1, (44, 60), 4, 1, 1, fb=1, seed=9),
    "clip_n2": _named(2, 1, 3, (52, 68), 6, 1, 2, seed=10),
    "clip_n5": _named(3, 1, 1, (72, 88), 12, 1, 5, fb=1, seed=11),
}

GEOMETRIES = {"random_%d" % s: random_geometry(s) for s in range(N_RANDOM)}
GEOMETRIES.update(NAMED)


def geometry_params(g):
    return params.from_cli_numbers(g["numbers"], noc=g["ch"], nop=g["nop"])


def bidir_range(g):
    """(f0, n) of the two-way sequence upload: n pairs into slots f0.., their swapped pairs into f0 + n..; None where
    the context has fewer than two slots"""
    n = min(g["n"], g["nfr"] // 2)
    return (min(g["f0"], g["nfr"] - 2 * n), n) if n else None


def clip_u8(g, n_frames, seed):
    """n_frames uniformly random 8-bit frames of the geometry's full resolution: the most rounding at deep levels"""
    shape = (n_frames,) + tuple(g["org"]) + ((g["ch"],) if g["ch"] == 3 else ())
    return np.random.default_rng(seed).integers(0, 256, shape, dtype=np.uint8)


# ---- float images that round ---------------------------------------------------------------------------------------
def float_image(shape, seed):
    """A float32 level image whose box means and Sobel sums round: full-mantissa values in [0, 255), planted
    negative values, magnitudes of 1e6, a block of -0 and +0, a block of subnormals (with its neighbours), and a
    constant first row, last row, first column and last column."""
    rng = np.random.default_rng(seed)
    img = rng.uniform(0, 255, shape).astype(f32)
    h, w = shape[:2]
    flat = img.reshape(h * w, -1)
    k = max(1, h * w // 16)
    flat[rng.choice(h * w, k, replace=False)] = -rng.uniform(0, 255, (k, flat.shape[1])).astype(f32)
    flat[rng.choice(h * w, k, replace=False)] = (rng.choice([-1, 1], (k, 1)) *
                                                 rng.uniform(1e6, 2e6, (k, flat.shape[1]))).astype(f32)
    y, x = int(rng.integers(0, h - 3)), int(rng.integers(0, w - 3))
    img[y:y + 4, x:x + 4] = np.where(rng.random((4, 4) + shape[2:]) < 0.5, f32(-0.0), f32(0.0))
    y, x = int(rng.integers(0, h - 3)), int(rng.integers(0, w - 3))
    img[y:y + 4, x:x + 4] = (rng.uniform(-1, 1, (4, 4) + shape[2:]) * 2.0 ** -127).astype(f32)  # below 2^-126
    img[0], img[-1] = img[0, 0], img[-1, -1]
    img[:, 0], img[:, -1] = f32(37.25), img[1, -1]
    return img


def float_pair(g, seed):
    """(a, b): float images of level sc_l of the geometry's context"""
    prm = geometry_params(g)
    shape = (g["size"][0] >> prm.sc_l, g["size"][1] >> prm.sc_l) + ((g["ch"],) if g["ch"] == 3 else ())
    return float_image(shape, seed), float_image(shape, seed + 1)


def level_pyramids(a, b, prm, pad):
    """PairPyramids of float images a, b of level sc_l, indexed by level (None below sc_l)"""
    p = preprocess.PairPyramids(a, b, prm.sc_f - prm.sc_l, pad)
    for k in ("i0", "i0x", "i0y", "i1", "i1x", "i1y"):
        setattr(p, k, [None] * prm.sc_l + getattr(p, k))
    return p


# inputs of the order checks: float images of a few geometries, and the deep 8-bit frames
FLOAT_INPUTS = {name: (name, 40 + i) for i, name in enumerate(["coarsest_2_columns", "sc_l2_sc_f5", "clip_n5",
                                                               "random_1", "random_4"])}
DEEP = ["deep_sc_f9_2048x1024", "deep_sc_f10_4096x2048"]


def _float_levels(name, seed):
    """[(level image, dx, dy)] of build_pyramid on the float image of FLOAT_INPUTS[name], unpadded"""
    g = GEOMETRIES[name]
    prm = geometry_params(g)
    a, _ = float_pair(g, seed)
    imgs, dxs, dys = preprocess.build_pyramid(a, prm.sc_f - prm.sc_l, 0)
    return list(zip(imgs, dxs, dys))


def _deep_levels(name):
    g = GEOMETRIES[name]
    img = clip_u8(g, 1, 1)[0].astype(f32)
    return list(zip(*preprocess.build_pyramid(img, g["numbers"][0], 0)))


def _shallow_levels():
    """the 8-bit inputs the suite already checked the device pyramids on: levels 0..7"""
    from of_dis_b200 import synth

    out = []
    for ch, size in ((1, (436, 1024)), (3, (121, 203))):
        i0, _, _ = synth.synthetic_pair(size[0], size[1], ch, seed=11)
        img, _, _ = preprocess.pad_to_multiple(i0, 4)
        out.append(list(zip(*preprocess.build_pyramid(img.astype(f32), 4, 0))))
    return out


# ---- other association orders --------------------------------------------------------------------------------------
def _quads(x):
    return x[0::2, 0::2], x[0::2, 1::2], x[1::2, 0::2], x[1::2, 1::2]


BOX_ORDERS = {
    "left_to_right": lambda a, b, c, d: (((a + b) + c) + d) * f32(0.25),
    "columns_first": lambda a, b, c, d: ((a + c) + (b + d)) * f32(0.25),
    "right_to_left": lambda a, b, c, d: (a + (b + (c + d))) * f32(0.25),
}


def _reflect(img):
    return np.pad(img, ((1, 1), (1, 1)) + (((0, 0),) if img.ndim == 3 else ()), mode="reflect")


def _gx_right(p):
    t = p[:, 2:] - p[:, :-2]
    return t[:-2] * f32(0.125) + (t[1:-1] * f32(0.25) + t[2:] * f32(0.125))


def _gx_outer(p):
    t = p[:, 2:] - p[:, :-2]
    return (t[:-2] * f32(0.125) + t[2:] * f32(0.125)) + t[1:-1] * f32(0.25)


def _gy_right(p):
    s = p[:, :-2] * f32(0.125) + (p[:, 1:-1] * f32(0.25) + p[:, 2:] * f32(0.125))
    return s[2:] - s[:-2]


def _gy_difference_first(p):
    d = p[2:] - p[:-2]
    return (d[:, :-2] * f32(0.125) + d[:, 1:-1] * f32(0.25)) + d[:, 2:] * f32(0.125)


SOBEL_ORDERS = {"gx_right_to_left": (0, _gx_right), "gx_outer_taps_first": (0, _gx_outer),
                "gy_right_to_left": (1, _gy_right), "gy_difference_first": (1, _gy_difference_first)}


def _differs(got, exp):
    return bool((np.asarray(got, f32).view(np.uint32) != np.asarray(exp, f32).view(np.uint32)).any())


def _box_differs(order, levels):
    return any(_differs(BOX_ORDERS[order](*_quads(levels[i - 1][0])), levels[i][0]) for i in range(1, len(levels)))


def _sobel_differs(order, levels):
    k, fn = SOBEL_ORDERS[order]
    return any(_differs(fn(_reflect(img)), (dx, dy)[k]) for img, dx, dy in levels)


# ---- tests ---------------------------------------------------------------------------------------------------------
def test_the_geometries_reach_every_named_case():
    gs = list(GEOMETRIES.values())
    prms = [geometry_params(g) for g in gs]
    for g, prm in zip(gs, prms):
        h, w = g["size"]
        assert h % (1 << prm.sc_f) == 0 and w % (1 << prm.sc_f) == 0
        assert preprocess.pad_to_multiple(np.zeros(g["org"], np.uint8), prm.sc_f)[0].shape == (h, w)
        assert 1 <= g["n"] and 0 <= g["f0"] and g["f0"] + g["n"] <= g["nfr"]
        assert (h >> prm.sc_f) >= 4 and (w >> prm.sc_f) >= 2
    for name in GEOMETRIES:
        if name.startswith("random_") and GEOMETRIES[name]["numbers"][0] > 0:
            g = GEOMETRIES[name]
            assert all((s - o) % 2 == 1 for s, o in zip(g["size"], g["org"])), name
    coarsest = [(g["size"][0] >> p.sc_f, g["size"][1] >> p.sc_f) for g, p in zip(gs, prms)]
    assert any(c[1] == 2 for c in coarsest) and any(c[0] == 4 for c in coarsest)
    for sc_l in (0, 2, 3):
        assert any(p.sc_l == sc_l and 1 <= p.sc_f <= 5 for p in prms)
    assert any(g["size"][0] >> p.sc_l > 2048 and g["size"][1] >> p.sc_l <= 64 for g, p in zip(gs, prms))
    assert NAMED["deep_sc_f9_2048x1024"]["org"] == (2048, 1024) and geometry_params(NAMED["deep_sc_f9_2048x1024"]).sc_f == 9
    assert NAMED["deep_sc_f10_4096x2048"]["org"] == (4096, 2048) and geometry_params(NAMED["deep_sc_f10_4096x2048"]).sc_f == 10
    assert any(p.sc_l == 8 and p.noc == 3 for p in prms)
    assert max(g["nfr"] for g in gs) == 64
    assert 3 * sum(p.usefbcon for p in prms) >= len(prms)
    assert {1, 2, 5} <= {g["n"] for g in gs} and {1, 2, 5} <= {bidir_range(g)[1] for g in gs if bidir_range(g)}
    assert all(g["f0"] > 0 for g in gs if g["nfr"] > 2)


@pytest.mark.parametrize("order", list(BOX_ORDERS))
def test_other_box_mean_orders_differ_on_float_images(order):
    for name, seed in FLOAT_INPUTS.values():
        assert _box_differs(order, _float_levels(name, seed)), name


@pytest.mark.parametrize("order", list(SOBEL_ORDERS))
def test_other_sobel_orders_differ_on_float_images(order):
    for name, seed in FLOAT_INPUTS.values():
        assert _sobel_differs(order, _float_levels(name, seed)), name


@pytest.mark.parametrize("name", DEEP)
def test_deep_levels_of_8bit_frames_round(name):
    """The Sobel sums of the dy orders round from level 8 on, and on 4096 x 2048 frames a left-to-right box sum
    from level 9 on: the deep 8-bit cases tell those orders apart where levels 0..7 cannot.  (The gx orders and
    the other box orders agree with build_pyramid on them; the float images tell those apart.)"""
    levels = _deep_levels(name)
    for order in ("gy_right_to_left", "gy_difference_first"):
        assert not _sobel_differs(order, levels[:8]), order
        assert _sobel_differs(order, levels[8:]), order
    assert not _box_differs("left_to_right", levels[:8])
    if len(levels) > 10:
        assert _box_differs("left_to_right", levels[7:])


def test_the_shallow_8bit_inputs_do_not_discriminate():
    """Why the float and deep inputs exist: on the 8-bit frames and levels the suite checked the device pyramids on,
    every order gives build_pyramid's bits."""
    for levels in _shallow_levels():
        for order in BOX_ORDERS:
            assert not _box_differs(order, levels), order
        for order in SOBEL_ORDERS:
            assert not _sobel_differs(order, levels), order


def _box64(x):
    a, b, c, d = (q.astype(np.float64) for q in _quads(x))
    return (a + b + c + d) / 4, (np.abs(a) + np.abs(b) + np.abs(c) + np.abs(d)) / 4


def _sobel64(img):
    """float64 reflect-101 Sobel / 8: (dx, dy) and the |kernel|-weighted sums of the operands' magnitudes"""
    p = _reflect(img).astype(np.float64)
    q = np.abs(p)
    wt = (0.125, 0.25, 0.125)
    dx = sum(wt[i] * (p[i:i + p.shape[0] - 2, 2:] - p[i:i + p.shape[0] - 2, :-2]) for i in range(3))
    dy = sum(wt[i] * (p[2:, i:i + p.shape[1] - 2] - p[:-2, i:i + p.shape[1] - 2]) for i in range(3))
    mx = sum(wt[i] * (q[i:i + q.shape[0] - 2, 2:] + q[i:i + q.shape[0] - 2, :-2]) for i in range(3))
    my = sum(wt[i] * (q[2:, i:i + q.shape[1] - 2] + q[:-2, i:i + q.shape[1] - 2]) for i in range(3))
    return dx, dy, mx, my


@pytest.mark.parametrize("name", list(FLOAT_INPUTS))
def test_build_pyramid_is_the_float64_box_mean_and_sobel(name):
    """Each level of build_pyramid on the float images against a float64 box mean of the level before it, each
    gradient against a float64 reflect-101 Sobel / 8 of its level.  The box mean ((a + b) + (c + d)) * 0.25 rounds
    three sums, each by at most U of its magnitude, and the product where it is subnormal by 2^-150; the Sobel sums
    round two products' sum, its sum with the third and -- before (gx) or after (gy) the weights -- the differences,
    at most three roundings of U on any path, and each of the six products where it is subnormal by 2^-150."""
    levels = _float_levels(*FLOAT_INPUTS[name])
    for lv, (img, dx, dy) in enumerate(levels):
        if lv:
            exact, mag = _box64(levels[lv - 1][0])
            bound = 3 * U * (1 + U) ** 2 * mag + 2.0 ** -150
            assert np.all(np.abs(img - exact) <= bound), (name, lv)
        ex, ey, mx, my = _sobel64(img)
        for got, exact, mag, what in ((dx, ex, mx, "dx"), (dy, ey, my, "dy")):
            bound = 3 * U * (1 + U) ** 3 * mag + 6 * 2.0 ** -150
            err = np.abs(got - exact)
            assert np.all(err <= bound), (name, lv, what, float((err / np.maximum(bound, 1e-300)).max()))
