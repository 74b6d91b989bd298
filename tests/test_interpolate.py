"""preprocess.interpolate_frames (the restatement of ofdis_interpolate_fullres) against a slow per-pixel loop written
from the header's contract, its behaviour on cases with a known answer, and the argument checks of
api.Context.interpolate_fullres that run before the device is touched."""
import ctypes
import math

import numpy as np
import pytest

from of_dis_b200 import api, params, preprocess

f32 = np.float32
INF = f32(np.inf)


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32 if a.dtype == np.float32 else np.uint8)


def _bil(img, xs, ys):
    h, w, nc = img.shape
    x0, y0 = int(math.floor(xs)), int(math.floor(ys))
    x1, y1 = min(x0 + 1, w - 1), min(y0 + 1, h - 1)
    fx, fy = f32(xs - f32(x0)), f32(ys - f32(y0))
    gx, gy = f32(1) - fx, f32(1) - fy
    out = []
    for c in range(nc):
        r0 = f32(f32(img[y0, x0, c]) * gx) + f32(f32(img[y0, x1, c]) * fx)
        r1 = f32(f32(img[y1, x0, c]) * gx) + f32(f32(img[y1, x1, c]) * fx)
        out.append(f32(f32(r0 * gy) + f32(r1 * fy)))
    return out


def _inside(x, y, w, h):
    return bool(x >= 0 and x <= f32(w - 1) and y >= 0 and y <= f32(h - 1))


def slow_interpolate(i0, i1, F, B, t, alpha, beta, order=None):
    """The header's five steps, one pixel at a time; sources are visited in `order` (default: raster order)."""
    h, w, nop = F.shape
    I0, I1 = i0.reshape(h, w, -1), i1.reshape(h, w, -1)
    t = f32(t)
    m0, _ = preprocess.consistency_check(F, B, alpha, beta)
    m1, _ = preprocess.consistency_check(B, F, alpha, beta)
    best = {}
    for s in (range(h * w) if order is None else order):
        Y, X = divmod(int(s), w)
        u = F[Y, X, 0]
        v = F[Y, X, 1] if nop == 2 else f32(0)
        if not (abs(u) <= f32(1e9) and abs(v) <= f32(1e9)):
            continue
        xs, ys = f32(f32(X) + u), f32(f32(Y) + v)
        if _inside(xs, ys, w, h):
            b = _bil(I1, xs, ys)
            c = f32(0)
            for ch in range(I0.shape[2]):
                c = f32(c + abs(f32(I0[Y, X, ch]) - b[ch]))
        else:
            c = INF
        key = (int(np.array(c, f32).view(np.uint32)) << 32) | (Y * w + X)
        px, py = f32(f32(X) + f32(t * u)), f32(f32(Y) + f32(t * v))
        if not (px > -1 and px < w and py > -1 and py < h):
            continue
        tx, ty = int(math.floor(px)), int(math.floor(py))
        for yy in ([ty, ty + 1] if py > math.floor(py) else [ty]):
            for xx in ([tx, tx + 1] if px > math.floor(px) else [tx]):
                if 0 <= xx < w and 0 <= yy < h and key < best.get((yy, xx), 1 << 64):
                    best[(yy, xx)] = key
    ut = np.zeros((h, w, nop), f32)
    stamp = np.full((h, w), -1)
    for (yy, xx), key in best.items():
        sy, sx = divmod(key & 0xFFFFFFFF, w)
        ut[yy, xx] = F[sy, sx]
        stamp[yy, xx] = 0
    if not best:
        stamp[:] = 0
    r = 0
    while (stamp < 0).any():
        r += 1
        for y in range(h):
            for x in range(w):
                if stamp[y, x] >= 0:
                    continue
                s, k = [f32(0)] * nop, 0
                for yy, xx in ((y, x - 1), (y, x + 1), (y - 1, x), (y + 1, x)):
                    if 0 <= xx < w and 0 <= yy < h and 0 <= stamp[yy, xx] < r:
                        s = [f32(s[c] + ut[yy, xx, c]) for c in range(nop)]
                        k += 1
                if k:
                    ut[y, x] = [f32(s[c] / f32(k)) for c in range(nop)]
                    stamp[y, x] = r
    out = np.zeros(I0.shape, np.uint8)
    for Y in range(h):
        for X in range(w):
            u = ut[Y, X, 0]
            v = ut[Y, X, 1] if nop == 2 else f32(0)
            x0, y0 = f32(f32(X) - f32(t * u)), f32(f32(Y) - f32(t * v))
            x1, y1 = f32(f32(X) + f32((f32(1) - t) * u)), f32(f32(Y) + f32((f32(1) - t) * v))
            in0, in1 = _inside(x0, y0, w, h), _inside(x1, y1, w, h)
            s0 = _bil(I0, min(max(x0, f32(0)), f32(w - 1)), min(max(y0, f32(0)), f32(h - 1)))
            s1 = _bil(I1, min(max(x1, f32(0)), f32(w - 1)), min(max(y1, f32(0)), f32(h - 1)))
            o0 = in0 and m0[int(math.floor(y0 + f32(0.5))), int(math.floor(x0 + f32(0.5)))] != 0
            o1 = in1 and m1[int(math.floor(y1 + f32(0.5))), int(math.floor(x1 + f32(0.5)))] != 0
            for c in range(I0.shape[2]):
                if (in0 and not in1) or (o0 and not o1):
                    val = s0[c]
                elif (in1 and not in0) or (o1 and not o0):
                    val = s1[c]
                else:
                    val = f32(f32((f32(1) - t) * s0[c]) + f32(t * s1[c]))
                out[Y, X, c] = int(f32(min(max(val, f32(0)), f32(255))) + f32(0.5))
    return out.reshape(i0.shape), ut


def _random_case(rng, h, w, noc, nop, kind):
    shape = (h, w) if noc == 1 else (h, w, noc)
    if kind == "flat":  # ties in cost: every match costs 0
        i0 = np.full(shape, 77, np.uint8)
        i1 = i0.copy()
    else:
        i0 = rng.integers(0, 256, shape, dtype=np.uint8)
        i1 = rng.integers(0, 256, shape, dtype=np.uint8)
    F = rng.normal(0, 1.5, (h, w, nop)).astype(f32)
    B = rng.normal(0, 1.5, (h, w, nop)).astype(f32)
    if kind == "integer":  # sources that meet on the same targets
        F = np.round(F).astype(f32)
        B = np.round(B).astype(f32)
    if kind in ("special", "flat"):
        for arr in (F, B):
            m = rng.random(arr.shape[:2])
            arr[m < 0.1, 0] = np.nan
            arr[(m >= 0.1) & (m < 0.15), 0] = np.inf
            arr[(m >= 0.15) & (m < 0.2), -1] = -np.inf
            arr[(m >= 0.2) & (m < 0.25), 0] = f32(3e9)   # unknown: above 1e9
            arr[(m >= 0.25) & (m < 0.3), 0] = f32(9e8)   # known, far outside the frame
            arr[(m >= 0.3) & (m < 0.4), 0] += f32(w)     # cost +inf, target may still be inside
    return i0, i1, F, B


@pytest.mark.parametrize("t", [0.25, 0.5, 0.75])
@pytest.mark.parametrize("noc,nop", [(1, 2), (3, 2), (1, 1), (3, 1)])
@pytest.mark.parametrize("kind", ["random", "integer", "special", "flat"])
def test_restatement_matches_the_per_pixel_loop(kind, noc, nop, t):
    rng = np.random.default_rng(hash((kind, noc, nop, t)) % 2**32)
    for h, w in ((5, 7), (6, 4)):
        i0, i1, F, B = _random_case(rng, h, w, noc, nop, kind)
        alpha, beta = api.CONSISTENCY_DEFAULTS[nop]
        out, ut = preprocess.interpolate_frames(i0, i1, F, B, t, alpha, beta)
        eo, eu = slow_interpolate(i0, i1, F, B, t, alpha, beta)
        assert out.shape == i0.shape and ut.shape == F.shape
        np.testing.assert_array_equal(out, eo)
        np.testing.assert_array_equal(_bits(ut), _bits(eu))


def test_result_does_not_depend_on_the_source_order():
    rng = np.random.default_rng(3)
    i0, i1, F, B = _random_case(rng, 6, 8, 1, 2, "integer")
    alpha, beta = api.CONSISTENCY_DEFAULTS[2]
    out, ut = preprocess.interpolate_frames(i0, i1, F, B, 0.5, alpha, beta)
    for seed in range(3):
        order = np.random.default_rng(seed).permutation(6 * 8)
        eo, eu = slow_interpolate(i0, i1, F, B, 0.5, alpha, beta, order=order)
        np.testing.assert_array_equal(out, eo)
        np.testing.assert_array_equal(_bits(ut), _bits(eu))


def test_batch_equals_pairs():
    rng = np.random.default_rng(4)
    cases = [_random_case(rng, 5, 6, 3, 2, "special") for _ in range(3)]
    a0, a1, F, B = (np.stack([c[k] for c in cases]) for k in range(4))
    out, ut, rounds = preprocess.interpolate_frames(a0, a1, F, B, 0.25, 0.01, 0.5, with_rounds=True)
    for k, (i0, i1, f, b) in enumerate(cases):
        o, u = preprocess.interpolate_frames(i0, i1, f, b, 0.25, 0.01, 0.5)
        np.testing.assert_array_equal(out[k], o)
        np.testing.assert_array_equal(_bits(ut[k]), _bits(u))
    assert rounds >= 0


@pytest.mark.parametrize("t", [0.25, 0.5, 0.75])
def test_zero_flow_gives_the_rounded_blend(t):
    rng = np.random.default_rng(5)
    i0 = rng.integers(0, 256, (9, 11, 3), dtype=np.uint8)
    i1 = rng.integers(0, 256, (9, 11, 3), dtype=np.uint8)
    F = np.zeros((9, 11, 2), f32)
    out, ut = preprocess.interpolate_frames(i0, i1, F, F, t, 0.01, 0.5)
    tt = f32(t)
    blend = (f32(1) - tt) * i0.astype(f32) + tt * i1.astype(f32)
    np.testing.assert_array_equal(out, (np.fmin(np.fmax(blend, f32(0)), f32(255)) + f32(0.5)).astype(np.uint8))
    assert not ut.any()


@pytest.mark.parametrize("nop", [2, 1])
def test_integer_translation_reproduces_the_shifted_frame(nop):
    rng = np.random.default_rng(6)
    h, w, d = 10, 24, 2
    wide = rng.integers(0, 256, (h, w + 2 * d), dtype=np.uint8)
    i0 = wide[:, d:d + w].copy()
    i1 = wide[:, :w].copy()  # i1(x) = i0(x - d): motion d to the right
    F = np.zeros((h, w, nop), f32)
    F[..., 0] = d
    B = -F
    out, ut = preprocess.interpolate_frames(i0, i1, F, B, 0.5, *api.CONSISTENCY_DEFAULTS[nop])
    half = wide[:, d // 2:d // 2 + w]  # frame at t = 0.5: i0(x - d/2)
    np.testing.assert_array_equal(out[:, 2 * d:w - 2 * d], half[:, 2 * d:w - 2 * d])
    assert (ut[..., 0][:, 2 * d:w - 2 * d] == d).all()


def test_occlusion_takes_the_frame_that_sees_the_pixel():
    # a square of 200 moving 4 px to the right over a static background of 50: at t = 0.5 the band it uncovers and
    # the band it is about to cover are background, taken from the one frame that shows background there
    h, w, a, s, d = 20, 40, 10, 12, 4
    i0 = np.full((h, w), 50, np.uint8)
    i1 = i0.copy()
    i0[4:4 + s, a:a + s] = 200
    i1[4:4 + s, a + d:a + d + s] = 200
    F = np.zeros((h, w, 2), f32)
    B = np.zeros((h, w, 2), f32)
    F[4:4 + s, a:a + s, 0] = d
    B[4:4 + s, a + d:a + d + s, 0] = -d
    out, _ = preprocess.interpolate_frames(i0, i1, F, B, 0.5, 0.01, 0.5)
    rows = slice(6, 4 + s - 2)
    assert (out[rows, a:a + d // 2] == 50).all()                      # uncovered: only I1 sees the background
    assert (out[rows, a + s + d // 2:a + s + d] == 50).all()          # about to be covered: only I0 sees it
    assert (out[rows, a + d // 2 + 1:a + s + d // 2 - 1] == 200).all()  # the square, half way
    # the plain blend would have mixed the square into both bands
    assert (((i0[rows].astype(int) + i1[rows]) // 2)[:, a:a + d // 2] != 50).all()


def test_all_nan_flow_gives_zero_flow():
    rng = np.random.default_rng(7)
    i0 = rng.integers(0, 256, (6, 7), dtype=np.uint8)
    i1 = rng.integers(0, 256, (6, 7), dtype=np.uint8)
    F = np.full((6, 7, 2), np.nan, f32)
    out, ut, rounds = preprocess.interpolate_frames(i0, i1, F, F, 0.5, 0.01, 0.5, with_rounds=True)
    assert rounds == 0 and not ut.any() and not np.signbit(ut).any()
    eo, eu = slow_interpolate(i0, i1, F, F, 0.5, 0.01, 0.5)
    np.testing.assert_array_equal(out, eo)


def test_one_splatted_pixel_fills_the_frame():
    h, w = 9, 13
    rng = np.random.default_rng(8)
    i0 = rng.integers(0, 256, (h, w), dtype=np.uint8)
    i1 = rng.integers(0, 256, (h, w), dtype=np.uint8)
    F = np.full((h, w, 2), np.nan, f32)
    F[1, 2] = (2.0, -4.0)  # at t = 0.25 it lands on (2.5, 0): the targets (2, 0) and (3, 0); its cost is +inf
    out, ut, rounds = preprocess.interpolate_frames(i0, i1, F, F, 0.25, 0.01, 0.5, with_rounds=True)
    assert (ut[..., 0] == 2).all() and (ut[..., 1] == -4).all()
    # the farthest pixel from the targets is the bottom-right corner
    assert rounds == (w - 1 - 3) + (h - 1 - 0)
    eo, eu = slow_interpolate(i0, i1, F, F, 0.25, 0.01, 0.5)
    np.testing.assert_array_equal(out, eo)
    np.testing.assert_array_equal(_bits(ut), _bits(eu))


class _NoDevice(api.Context):
    """A Context whose checks run without a device: the library is never reached by a refused call."""

    def __init__(self, noc, nop):  # noqa: D401 -- no ofdis_create
        self.prm = params.operating_point(2, 64, noc=noc, nop=nop)
        self._h = ctypes.c_void_p()

    def close(self):
        pass


@pytest.mark.parametrize("noc", [1, 3])
def test_api_checks_host_arrays(noc):
    ctx = _NoDevice(noc, 2)
    h, w, n = 4, 6, 3
    frame = (h, w) if noc == 1 else (h, w, noc)
    clip = np.zeros((n + 1,) + frame, np.uint8)
    pairs = np.zeros((n, 2) + frame, np.uint8)
    bad = [
        (clip[:-1].astype(np.int16), clip[1:]),           # dtype
        (clip[:-2], clip[1:-1]),                            # frame count
        (clip[:-1, :, :-1], clip[1:, :, :-1]),              # frame shape
        (clip[:-1, :, ::-1], clip[1:, :, ::-1]),            # frames not C-contiguous
        (clip[:-1], pairs[:, 1]),                           # strides differ
        (clip[::-1][:-1], clip[::-1][1:]),                  # negative stride
    ]
    for f0, f1 in bad:
        with pytest.raises(ValueError):
            ctx.interpolate_fullres(0, n, n, f0, f1, 0.5, w, h)
    for kw in ({"out": np.zeros((n, h, w, 2), np.uint8)}, {"out": np.zeros((n,) + frame, np.float32)},
               {"with_flow": True, "flow_t": np.zeros((n, h, w, 1), np.float32)},
               {"with_flow": True, "flow_t": np.zeros((n, h, w, 2), np.float64)},
               {"out": np.zeros((n,) + frame, np.uint8)[:, ::-1]}):
        with pytest.raises(ValueError):
            ctx.interpolate_fullres(0, n, n, clip[:-1], clip[1:], 0.5, w, h, **kw)


def test_api_accepts_clip_and_pair_layouts(monkeypatch):
    # the layouts of the issue reach the library with the right frame stride
    calls = []

    class _Lib:
        def ofdis_interpolate_fullres(self, *a):
            calls.append(a)
            return 0

    monkeypatch.setattr(api, "lib", lambda: _Lib())
    ctx = _NoDevice(3, 2)
    ctx.sync = lambda: None
    h, w, n = 4, 6, 3
    hwc = h * w * 3
    clip = np.zeros((n + 1, h, w, 3), np.uint8)
    pairs = np.zeros((n, 2, h, w, 3), np.uint8)
    out, fl = ctx.interpolate_fullres(0, n, n, clip[:-1], clip[1:], 0.5, w, h, with_flow=True)
    assert out.shape == (n, h, w, 3) and fl.shape == (n, h, w, 2) and calls[-1][6] == hwc
    ctx.interpolate_fullres(0, n, n, pairs[:, 0], pairs[:, 1], 0.5, w, h)
    assert calls[-1][6] == 2 * hwc
    assert calls[-1][8:10] == api.CONSISTENCY_DEFAULTS[2]
    ctx.interpolate_fullres(0, 1, 1, clip[:1], clip[1:2], 0.5, w, h, alpha=0.0, beta=2.0)
    assert calls[-1][6] == hwc and calls[-1][8:10] == (0.0, 2.0)
