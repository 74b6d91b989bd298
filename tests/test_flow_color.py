"""Color-coded flows (ofdis_flow_color_fullres) on the CPU: preprocess.atan2_f32 against float64 atan2,
preprocess.flow_to_color against an independent float64 restatement of Middlebury's computeColor / MotionToColor,
the exact edge cases of the contract for flow and stereo, and the batch command's --color grammar."""
import os
import subprocess

import numpy as np
import pytest

from of_dis_b200 import api, preprocess

f32 = np.float32
PI_F = f32(np.pi)


def bits(a):
    return np.asarray(a, f32).view(np.uint32)


# ---- atan2_f32 ------------------------------------------------------------------------------------------------------
def test_atan2_f32_accuracy_and_range():
    ang = np.linspace(-np.pi, np.pi, 400_001)
    worst = 0.0
    for m in (1e-45, 1e-42, 1e-39, 1.2e-38, 1e-30, 1e-12, 1e-3, 0.7, 1.0, 3.0, 1e3, 1e6, 1e9):
        y, x = (m * np.sin(ang)).astype(f32), (m * np.cos(ang)).astype(f32)
        got = preprocess.atan2_f32(y, x)
        assert got.dtype == f32
        assert np.all(np.abs(got) <= PI_F)
        ref = np.arctan2(y.astype(np.float64), x.astype(np.float64))
        worst = max(worst, float(np.abs(got.astype(np.float64) - ref).max()))
    # independent magnitudes for y and x, subnormal to 1e9, both signs
    rng = np.random.default_rng(1)
    mag = lambda n: (10.0 ** rng.uniform(-45, 9, n)).astype(f32) * rng.choice(f32([-1, 1]), n)  # noqa: E731
    y, x = mag(1_000_000), mag(1_000_000)
    got = preprocess.atan2_f32(y, x)
    assert np.all(np.abs(got) <= PI_F)
    worst = max(worst, float(np.abs(got.astype(np.float64) - np.arctan2(y.astype(np.float64), x.astype(np.float64))).max()))
    assert worst <= 1e-6, worst


def test_atan2_f32_signed_zeros_and_axes():
    half = PI_F * f32(0.5)
    # (y, x, C's atan2) -- a list, since a dict would merge the keys 0.0 and -0.0
    cases = [(0.0, -1.0, PI_F), (-0.0, -1.0, -PI_F), (0.0, 1.0, f32(0.0)), (-0.0, 1.0, f32(-0.0)),
             (0.0, -0.0, PI_F), (-0.0, -0.0, -PI_F), (0.0, 0.0, f32(0.0)), (-0.0, 0.0, f32(-0.0)),
             (1.0, 0.0, half), (-1.0, 0.0, -half), (1.0, -0.0, half), (-1.0, -0.0, -half)]
    for y, x, exp in cases:
        got = preprocess.atan2_f32(f32(y), f32(x))
        assert bits(got) == bits(exp), (y, x, float(got), float(exp))
        assert bits(got) == bits(np.arctan2(f32(y), f32(x))), (y, x)  # C's values
    assert float(half) == float(np.float32(np.pi / 2))


# ---- flow_to_color --------------------------------------------------------------------------------------------------
def middlebury_f64(flow, max_motion=0.0):
    """Middlebury's flow-code (colorcode.cpp computeColor, color-flow's MotionToColor) in float64, written from the
    published algorithm: its own wheel, the maximum radius of the known pixels (1 where it is 0) or max_motion."""
    ncols = 55
    wheel = []
    for n, f in ((15, lambda i: (255, 255 * i // 15, 0)), (6, lambda i: (255 - 255 * i // 6, 255, 0)),
                 (4, lambda i: (0, 255, 255 * i // 4)), (11, lambda i: (0, 255 - 255 * i // 11, 255)),
                 (13, lambda i: (255 * i // 13, 0, 255)), (6, lambda i: (255, 0, 255 - 255 * i // 6))):
        wheel += [f(i) for i in range(n)]
    wheel = np.array(wheel, np.float64)
    assert len(wheel) == ncols
    u, v = flow[..., 0].astype(np.float64), flow[..., 1].astype(np.float64)
    known = (np.abs(u) <= 1e9) & (np.abs(v) <= 1e9)
    u, v = np.where(known, u, 0.0), np.where(known, v, 0.0)
    maxrad = np.sqrt(u * u + v * v).max(initial=0.0)
    if max_motion > 0:
        maxrad = max_motion
    if maxrad == 0:
        maxrad = 1.0
    fx, fy = u / maxrad, v / maxrad
    rad = np.sqrt(fx * fx + fy * fy)
    a = np.arctan2(-fy, -fx) / np.pi
    fk = (a + 1.0) / 2.0 * (ncols - 1)
    k0 = fk.astype(int)
    k1 = (k0 + 1) % ncols
    f = fk - k0
    out = np.zeros(flow.shape[:-1] + (3,), np.int32)
    for b in range(3):
        col = (1 - f) * wheel[k0, b] / 255.0 + f * wheel[k1, b] / 255.0
        col = np.where(rad <= 1, 1 - rad * (1 - col), col * 0.75)
        out[..., b] = np.where(known, (255.0 * col).astype(int), 0)
    return out


@pytest.mark.parametrize("max_value", [0.0, 3.5])
def test_flow_to_color_matches_middlebury_in_float64(max_value):
    rng = np.random.default_rng(2)
    n = 1_000_000
    flow = (rng.standard_normal((1000, n // 1000, 2)) * rng.choice([0.3, 2.0, 20.0], (1000, 1, 1))).astype(f32)
    axes = np.array([[1, 0], [-1, 0], [0, 1], [0, -1], [2, 0], [0, -2], [0.5, 0], [0, 0.5]], f32) * 3
    flow[0, :len(axes)] = axes
    got, scale = preprocess.flow_to_color(flow, max_value)
    assert got.dtype == np.uint8 and got.shape == flow.shape[:-1] + (3,) and scale.dtype == f32
    exp = middlebury_f64(flow, max_value)
    diff = np.abs(got.astype(np.int32) - exp)
    assert diff.max() <= 1, diff.max()
    assert (diff > 0).mean() < 1e-2  # float32 rounding at the truncations, not a systematic offset


def test_flow_to_color_edges():
    big = np.nextafter(f32(1e9), f32(np.inf))
    assert f32(1e9) == 1e9
    unknown = [np.nan, -np.nan, np.inf, -np.inf, big, -big]
    flow = np.zeros((4, 8, 2), f32)
    flow[0, :6, 0] = unknown
    flow[1, :6, 1] = unknown
    flow[2, 0] = (1e9, 0)
    flow[2, 1] = (0, -1e9)
    flow[3, :] = (0, 0)
    rgb, scale = preprocess.flow_to_color(flow)
    assert (rgb[0, :6] == 0).all() and (rgb[1, :6] == 0).all()
    assert scale == f32(1e9)
    assert rgb[2, :2].any(axis=-1).all()  # exactly 1e9 is known, and colored
    assert (rgb[3] == 255).all() and (rgb[0, 6:] == 255).all()  # zero flow is white
    # all-zero and all-unknown slots have scale 1
    assert preprocess.flow_to_color(np.zeros((3, 4, 2), f32))[1] == 1
    allnan = np.full((2, 3, 4, 2), np.nan, f32)
    allnan[1] = np.inf
    rgb, scale = preprocess.flow_to_color(allnan)
    assert (scale == 1).all() and (rgb == 0).all()
    # u < 0, v = 0: a = atan2_f32(-0, 1) / PI_F = -0, fk = 27, f = 0, so col is wheel entry 27 itself; beyond the
    # scale it is darkened by 0.75, on the scale it stays within rounding of the entry
    rgb, _ = preprocess.flow_to_color(np.array([[[-1, 0], [-2, 0]]], f32), max_value=1.0)
    w = preprocess.COLOR_WHEEL[27]
    assert w.tolist() == [0, 209, 255]
    assert rgb[0, 1].tolist() == [int(f32(255) * (f32(c) / f32(255) * f32(0.75))) for c in w]
    assert np.abs(rgb[0, 0].astype(int) - w).max() <= 1


def test_flow_to_color_batch_and_tiny_max_value():
    rng = np.random.default_rng(3)
    flows = rng.normal(0, 5, (3, 6, 7, 2)).astype(f32)
    rgb, scale = preprocess.flow_to_color(flows)
    for k in range(3):
        r1, s1 = preprocess.flow_to_color(flows[k])
        assert (r1 == rgb[k]).all() and bits(s1) == bits(scale[k])
    # max_value 1e-30: fx, fy overflow to inf, the angle of the unscaled flow stays finite -> darkened wheel colors
    rgb, scale = preprocess.flow_to_color(flows, 1e-30)
    assert (scale == f32(1e-30)).all()
    assert (rgb <= 191).all() and rgb.max() > 0


# ---- disp_to_color --------------------------------------------------------------------------------------------------
def test_disp_color_bins():
    wt, cum = preprocess.disp_color_bins()
    assert cum[0] == 0 and cum[7] == f32(1.0)
    assert (np.diff(cum) > 0).all()
    assert wt[0] == f32(1000) / f32(114)


def test_disp_to_color_edges():
    wt, cum = preprocess.disp_color_bins()
    scale = f32(10)
    d = np.array([10, 0, -0.0, -1, np.nan, np.nextafter(f32(1e9), f32(np.inf)), np.inf, 5, 1e9], f32)
    rgb, s = preprocess.disp_to_color(-d[:, None, None], max_value=float(scale))  # this library's sign: F = -d
    assert s == scale
    # d = scale: val = 1 is in no bin (cum[7] == 1.0f), so the "else 6" branch; in float32, (1 - cum[6]) * wt[6] is
    # 1 - 3.6e-7, so w is not 0 and blue truncates to 254: white but for one step of blue
    w6 = f32(1) - (f32(1) - cum[6]) * wt[6]
    assert 0 < w6 < 1e-6
    assert rgb[0, 0].tolist() == [255, 255, int((w6 * f32(0) + (f32(1) - w6) * f32(1)) * f32(255))] == [255, 255, 254]
    assert (rgb[1:6] == 0).all()  # 0, -0, negative, NaN, > 1e9 are black (0 and -0 are valid: black by the map)
    assert (rgb[6] == 0).all()
    assert rgb[8, 0].tolist() == rgb[0, 0].tolist()  # 1e9 is valid and beyond the scale: val = 1 as well
    # values exactly at each cum boundary fall into the next bin: w = 1 there, so the bin's own map entry
    for i in range(1, 7):
        v = cum[i]
        got, _ = preprocess.disp_to_color(np.array([[[-v]]], f32), max_value=1.0)
        exp = (preprocess.DISP_COLOR_MAP[i, :3] * 255).tolist()
        assert got[0, 0].tolist() == exp, (i, got[0, 0].tolist(), exp)
    # the swapped sign: +F is the disparity
    F = np.array([[[3.0], [-3.0]]], f32)
    a, _ = preprocess.disp_to_color(F, max_value=6.0)
    b, _ = preprocess.disp_to_color(F, max_value=6.0, swapped=True)
    assert (a[0, 1] == b[0, 0]).all() and (a[0, 0] == 0).all() and (b[0, 1] == 0).all() and a[0, 1].any()
    # the automatic scale is at least 1: all disparities below 1 keep their colors below white
    small = -np.full((1, 4, 4, 1), 0.25, f32)
    rgb, s = preprocess.disp_to_color(small)
    assert s[0] == 1
    rgb2, _ = preprocess.disp_to_color(small, max_value=1.0)
    assert (rgb == rgb2).all()
    assert preprocess.disp_to_color(-np.full((2, 2, 1), 7.5, f32))[1] == f32(7.5)
    # per-slot swapped marks of a batch
    batch = np.stack([F, -F])
    rgb, _ = preprocess.disp_to_color(batch, 6.0, swapped=[False, True])
    assert (rgb[0] == rgb[1]).all()


def test_color_export():
    assert "ofdis_flow_color_fullres" in api.EXPORTS


# ---- batch front-end: --color grammar (refused before the device is touched) ------------------------------------------
@pytest.fixture(scope="module")
def bindir():
    from of_dis_b200 import build

    return build.build_host()


@pytest.mark.parametrize("exe", ["run_OF_INT_batch", "run_DE_RGB_batch"])
def test_batch_command_color_grammar(bindir, tmp_path, exe):
    path = os.path.join(bindir, exe)
    lst = tmp_path / "list.txt"
    lst.write_text("")
    r = subprocess.run([path], capture_output=True, text=True)
    assert r.returncode == 2 and "--color-max" in r.stderr
    for args in (["--color-max", "2"], ["--color", "--color-max", "0"], ["--color", "--color-max", "-1"],
                 ["--color", "--color-max", "inf"], ["--color", "--color-max", "nan"],
                 ["--color", "--color-max", "1e39"], ["--color", "--color-max", "2x"], ["--color", "--color-max"],
                 ["--color", "--color-max", "1", "--color-max", "2"]):
        r = subprocess.run([path, str(lst)] + args, capture_output=True, text=True)
        assert r.returncode == 2, (args, r.stderr)
    # an empty list with valid options does nothing and succeeds
    for args in (["--color"], ["--color", "--color-max", "0.5", "--kitti", "--batch", "2"]):
        r = subprocess.run([path, str(lst)] + args, capture_output=True, text=True)
        assert r.returncode == 0, (args, r.stderr)
