"""preprocess.confidence (ofdis_confidence_fullres's restatement) against a per-pixel loop written from the header,
its texture term against the tracker's seeding at r = 2, and the weighted fusion and tracking restatements: all-ones
weights give the unweighted results bit for bit, and weights of 0, -0, NaN and negative values skip an observation."""
import math

import numpy as np
import pytest

from of_dis_b200 import preprocess, synth

f32 = np.float32
QNAN = np.uint32(0x7FC00000).view(f32)


def bits(a):
    return np.ascontiguousarray(np.asarray(a, f32)).view(np.uint32)


def gray(I, x, y):
    p = I[y, x]
    if I.ndim == 3:
        return (f32(p[0]) + f32(p[1]) + f32(p[2])) / f32(3)
    return f32(p)


def pixel_loop(I0, I1, F, B, r, s_fb, s_tex, min_count):
    """The header's per-pixel formulas, one pixel and one window tap at a time, in float32 scalars."""
    H, W = I0.shape[:2]
    F = F.reshape(H, W, -1)
    nop = F.shape[2]
    s_fb, s_tex = f32(s_fb), f32(s_tex)
    half, quarter = f32(0.5), f32(0.25)

    def iw(qx, qy):
        u = F[qy, qx, 0]
        v = F[qy, qx, 1] if nop == 2 else f32(0)
        xs, ys = f32(qx) + u, f32(qy) + v
        if not (xs >= 0 and xs <= f32(W - 1) and ys >= 0 and ys <= f32(H - 1)):
            return None
        x0, y0 = int(math.floor(xs)), int(math.floor(ys))
        x1, y1 = min(x0 + 1, W - 1), min(y0 + 1, H - 1)
        fx, fy = f32(xs - f32(x0)), f32(ys - f32(y0))
        gx, gy = f32(1) - fx, f32(1) - fy
        r0 = gray(I1, x0, y0) * gx + gray(I1, x1, y0) * fx
        r1 = gray(I1, x0, y1) * gx + gray(I1, x1, y1) * fx
        return f32(r0 * gy + r1 * fy)

    conf = np.zeros((H, W), f32)
    terms = np.zeros((H, W, 3), f32)
    e_map = None if B is None else preprocess.consistency_check(F, B, 0.0, 0.0)[1]
    with np.errstate(all="ignore"):
        for Y in range(H):
            for X in range(W):
                win = [(min(max(X + dx, 0), W - 1), min(max(Y + dy, 0), H - 1))
                       for dy in range(-r, r + 1) for dx in range(-r, r + 1)]
                n, s0, s1, a, b, c = 0, f32(0), f32(0), f32(0), f32(0), f32(0)
                samples = []
                for qx, qy in win:
                    ix = (gray(I0, min(qx + 1, W - 1), qy) - gray(I0, max(qx - 1, 0), qy)) * half
                    iy = (gray(I0, qx, min(qy + 1, H - 1)) - gray(I0, qx, max(qy - 1, 0))) * half
                    a, b, c = f32(a + ix * ix), f32(b + ix * iy), f32(c + iy * iy)
                    w1 = iw(qx, qy)
                    if w1 is not None:
                        n += 1
                        s0, s1 = f32(s0 + gray(I0, qx, qy)), f32(s1 + w1)
                        samples.append((gray(I0, qx, qy), w1))
                d = f32(a - c)
                lam = f32((a + c) * half - f32(np.sqrt(f32(d * d * quarter + b * b))))
                z = QNAN
                if n >= min_count:
                    m0, m1 = f32(s0 / f32(n)), f32(s1 / f32(n))
                    c00, c11, c01 = f32(0), f32(0), f32(0)
                    for g0, w1 in samples:
                        p, q = f32(g0 - m0), f32(w1 - m1)
                        c00, c11, c01 = f32(c00 + p * p), f32(c11 + q * q), f32(c01 + p * q)
                    den = f32(c00 * c11)
                    if den > 0:
                        z = f32(c01 / f32(np.sqrt(den)))
                if e_map is None:
                    e, ce = QNAN, f32(1)
                else:
                    e = e_map[Y, X]
                    ce = f32(s_fb / f32(s_fb + e)) if e >= 0 else f32(0)
                cz = z if z > 0 else f32(0)
                cl = f32(lam / f32(lam + s_tex)) if lam > 0 else f32(0)
                conf[Y, X] = f32(f32(cz * ce) * cl)
                terms[Y, X] = (z, e, lam)
    return conf, terms


def pair(seed, h, w, ch, nop, specials=False):
    rng = np.random.default_rng(seed)
    shape = (h, w, ch) if ch == 3 else (h, w)
    I0 = rng.integers(0, 256, shape).astype(np.uint8)
    I1 = np.roll(I0, 1, axis=1) // 2 + rng.integers(0, 128, shape).astype(np.uint8)
    I0[:8, :8] = 77  # a flat patch: zero variance and lambda 0
    F = rng.uniform(-3, 3, (h, w, nop)).astype(f32)
    B = (-F + rng.normal(0, 0.5, F.shape)).astype(f32)
    if specials:
        for v, share in ((np.nan, 0.05), (np.inf, 0.03), (-np.inf, 0.03), (3e9, 0.03), (-0.0, 0.05)):
            F[rng.random(F.shape) < share] = v
            B[rng.random(B.shape) < share] = v
    return I0, I1, F, B


@pytest.mark.parametrize("ch,nop", [(1, 2), (3, 2), (1, 1), (3, 1)])
@pytest.mark.parametrize("r", [1, 2, 3])
@pytest.mark.parametrize("with_b", [True, False])
def test_restatement_equals_the_pixel_loop(ch, nop, r, with_b):
    I0, I1, F, B = pair(10 * ch + nop + r, 11, 14, ch, nop, specials=(r == 2))
    prm = dict(radius=r, s_fb=2.0, s_tex=50.0, min_count=max(1, (2 * r + 1) ** 2 // 2))
    got = preprocess.confidence(I0, I1, F, B if with_b else None, prm)
    exp = pixel_loop(I0, I1, F, B if with_b else None, r, prm["s_fb"], prm["s_tex"], prm["min_count"])
    assert (bits(got[0]) == bits(exp[0])).all()
    assert (bits(got[1]) == bits(exp[1])).all()
    assert (got[0] >= 0).all() and np.isnan(got[1][..., 0]).any() and (got[0] > 0).any()


@pytest.mark.parametrize("ch", [1, 3])
def test_texture_term_is_the_trackers_at_radius_2(ch):
    I0, I1, F, _ = pair(5 + ch, 19, 23, ch, 2)
    _, terms = preprocess.confidence(I0, I1, F, None, dict(radius=2, s_fb=1.0, s_tex=1.0, min_count=1))
    cx, cy, lam = preprocess.track_seed_eigen(I0, 1)  # spacing 1: one cell per pixel, seeded at the pixel
    assert (bits(terms[cy, cx, 2]) == bits(lam)).all()


def test_forward_backward_term_is_the_consistency_err():
    I0, I1, F, B = pair(3, 13, 17, 1, 2, specials=True)
    _, terms = preprocess.confidence(I0, I1, F, B, dict(radius=1, s_fb=1.0, s_tex=1.0, min_count=1))
    assert (bits(terms[..., 1]) == bits(preprocess.consistency_check(F, B, 0.01, 0.5)[1])).all()


# ---- weighted fusion and tracking ---------------------------------------------------------------------------------
CAM = dict(fx=40.0, fy=38.5, cx=15.25, cy=11.5, baseline=0.5, doffs=0.25)
TP = dict(step=1, rounds=6, min_weight=1.0, max_depth=float("inf"), huber=0.3, damping=0.0, min_corr=6,
          max_shift=0.5, min_cos=0.99, eps=0.0, integrate=1)
VP = dict(nx=37, ny=23, nz=41, origin=(-1.9, -0.9, -0.35), voxel=0.07, trunc=0.2, max_weight=6.0, color=1)


def pose(w=(0, 0, 0), t=(0, 0, 0)):
    return np.concatenate([synth.axis_angle(np.asarray(w, np.float64)), np.asarray(t, np.float64).reshape(3, 1)], 1)


def scene(seed, n, h, w):
    rng = np.random.default_rng(seed)
    vol = preprocess.fuse_new_volume(VP)
    nz, ny, nx = vol["T"].shape
    z = VP["origin"][2] + np.arange(nz)[:, None, None] * VP["voxel"]
    x = VP["origin"][0] + np.arange(nx)[None, None, :] * VP["voxel"]
    y = VP["origin"][1] + np.arange(ny)[None, :, None] * VP["voxel"]
    vol["T"][:] = np.clip((1.3 + 0.1 * np.sin(3 * x) + 0.05 * y - z) / VP["trunc"], -1, 1).astype(f32)
    vol["W"][:] = rng.choice(np.array([1.0, 2.0, 3.0], f32), vol["W"].shape)
    vol["C"][:] = rng.integers(0, 256, vol["C"].shape)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    disp = []
    for k in range(n):
        Z = 1.3 + 0.02 * np.sin(xx / 5.0 + k) + 0.003 * yy + rng.uniform(-0.01, 0.01, (h, w))
        disp.append((f32(CAM["fx"]) * f32(CAM["baseline"]) / Z - CAM["doffs"]).astype(f32))
    motions = np.stack([pose(rng.uniform(-0.005, 0.005, 3), rng.uniform(-0.02, 0.02, 3)) for _ in range(n)])
    frames = rng.integers(0, 256, (n, h, w, 3)).astype(np.uint8)
    return vol, np.stack(disp), motions, frames


def copy(vol):
    return {k: (None if v is None else v.copy()) for k, v in vol.items()}


def same_vol(a, b):
    for k in ("T", "W", "C"):
        assert np.array_equal(np.ascontiguousarray(a[k]).view(np.uint8), np.ascontiguousarray(b[k]).view(np.uint8)), k


def test_weighted_push_with_ones_is_the_push():
    vol, disp, motions, frames = scene(1, 3, 24, 31)
    poses = np.stack([pose((0.01 * k, 0, 0), (0.02 * k, 0, 0)) for k in range(3)])
    a, b = copy(vol), copy(vol)
    preprocess.fuse_integrate(a, VP, disp, poses, CAM, frames=frames)
    preprocess.fuse_integrate(b, VP, disp, poses, CAM, frames=frames, weights=np.ones(disp.shape, f32))
    same_vol(a, b)
    assert not np.array_equal(a["W"], vol["W"])


def test_weights_that_are_not_positive_skip_the_observation():
    vol, disp, motions, frames = scene(2, 2, 24, 31)
    poses = np.stack([pose((0.01 * k, 0, 0), (0.02 * k, 0, 0)) for k in range(2)])
    rng = np.random.default_rng(0)
    wts = np.ones(disp.shape, f32)
    skip = rng.random(disp.shape) < 0.4
    wts[skip] = rng.choice(np.array([0.0, -0.0, np.nan, -1.0, -np.inf, np.inf], f32), int(skip.sum()))
    masked = disp.copy()
    masked[skip] = np.nan  # an unknown disparity skips the observation in the unweighted push
    a, b = copy(vol), copy(vol)
    preprocess.fuse_integrate(a, VP, masked, poses, CAM, frames=frames)
    preprocess.fuse_integrate(b, VP, disp, poses, CAM, frames=frames, weights=wts)
    same_vol(a, b)


def test_weighted_push_formula():
    # one voxel seen by one pixel of weight c: W' = W + c, T = (T W + f c) / W', colour rounding under the push's rule
    vol, disp, motions, frames = scene(3, 1, 24, 31)
    poses = pose().reshape(1, 3, 4)
    c = f32(0.37)
    a, b = copy(vol), copy(vol)
    preprocess.fuse_integrate(a, VP, disp, poses, CAM, frames=frames, weights=np.full(disp.shape, c, f32))
    preprocess.fuse_integrate(b, VP, disp, poses, CAM, frames=frames)
    changed = b["W"] != vol["W"]
    assert changed.any() and (a["W"] != vol["W"]).sum() == changed.sum()
    W0 = vol["W"][changed]
    assert np.array_equal(a["W"][changed], np.fmin(W0 + c, f32(VP["max_weight"])))
    # f recovered from the unweighted update: T1 = (T0 W0 + f) / (W0 + 1); compare the weighted T to within rounding
    f = b["T"][changed] * (W0 + 1) - vol["T"][changed] * W0
    assert np.allclose(a["T"][changed], (vol["T"][changed] * W0 + f * c) / (W0 + c), atol=1e-5)


@pytest.mark.parametrize("integrate", [0, 1])
def test_weighted_track_with_ones_is_the_track(integrate):
    vol, disp, motions, frames = scene(4, 3, 24, 31)
    prev = pose((0.01, -0.02, 0.005), (0.02, -0.01, 0.03))
    tp = dict(TP, integrate=integrate)
    a, b = copy(vol), copy(vol)
    pa, sa = preprocess.fuse_track(a, VP, tp, disp, motions, prev, CAM, frames)
    pb, sb = preprocess.fuse_track(b, VP, tp, disp, motions, prev, CAM, frames, weights=np.ones(disp.shape, f32))
    assert np.array_equal(pa.view(np.uint64), pb.view(np.uint64))
    assert np.array_equal(sa.view(np.uint8), sb.view(np.uint8))
    same_vol(a, b)
    assert (sa["rounds"] > 0).any()


def test_weighted_track_skips_cells_and_scales_terms():
    vol, disp, motions, frames = scene(5, 1, 24, 31)
    rng = np.random.default_rng(1)
    wts = rng.uniform(0.2, 1.5, disp.shape).astype(f32)
    wts[0, 0, :12] = np.array([0.0, -0.0, np.nan, -2.0, np.inf, -np.inf] * 2, f32)
    p = preprocess.fuse_track_params(TP)
    cam = preprocess._ego_cam(CAM)
    M = pose((0.01, 0, 0), (0.01, 0, 0)).ravel()
    ok, r, G, Pw = preprocess.fuse_track_cells(vol, VP, disp[0], cam, 1, TP["min_weight"], TP["max_depth"], M)
    c = wts[0].ravel()
    A, b, cost, cnt = preprocess.fuse_track_eval(vol, VP, disp[0], cam, p, M, wts[0])
    sel = ok & (c > 0) & np.isfinite(c)
    assert cnt == int(sel.sum()) and cnt < int(ok.sum())
    terms = preprocess.fuse_track_terms(r[sel], G[sel], Pw[sel], TP["huber"], c[sel])
    ar = np.abs(r[sel])
    wt = np.where(ar <= f32(TP["huber"]), f32(1), f32(TP["huber"]) / ar).astype(f32) * c[sel]
    assert np.array_equal(terms[:, 27], (wt.astype(np.float64) * r[sel]) * r[sel])
