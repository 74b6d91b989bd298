"""preprocess.fuse_track (ofdis_fuse_track's restatement) against a scalar per-cell loop written from the header,
the trilinear gradient against finite differences, planted planar and corner volumes, the statuses, and the call's
two properties (n frames in one call equal n calls of one; integrating equals aligning then pushing)."""
import math

import numpy as np
import pytest

from of_dis_b200 import preprocess

f32 = np.float32
CAM = dict(fx=40.0, fy=38.5, cx=15.25, cy=11.5, baseline=0.5, doffs=0.25)
TP = dict(step=1, rounds=10, min_weight=1.0, max_depth=float("inf"), huber=0.3, damping=0.0, min_corr=6,
          max_shift=1.0, min_cos=0.9, eps=0.0, integrate=0)


def rot(w):
    w = np.asarray(w, np.float64)
    t = np.linalg.norm(w)
    if t == 0:
        return np.eye(3)
    k = w / t
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + math.sin(t) * K + (1 - math.cos(t)) * K @ K


def pose(w=(0, 0, 0), t=(0, 0, 0)):
    return np.concatenate([rot(w), np.asarray(t, np.float64).reshape(3, 1)], 1)


def planted(seed, p, h, w):
    """A wavy surface TSDF with planted W at and around min_weight, NaN and +-1 T, and disparities of a wavy surface
    with NaN, -0, +inf and 3e9."""
    rng = np.random.default_rng(seed)
    vol = preprocess.fuse_new_volume(p)
    nz, ny, nx = vol["T"].shape
    z = p["origin"][2] + np.arange(nz)[:, None, None] * p["voxel"]
    x = p["origin"][0] + np.arange(nx)[None, None, :] * p["voxel"]
    y = p["origin"][1] + np.arange(ny)[None, :, None] * p["voxel"]
    sdf = 1.2 + 0.1 * np.sin(3 * x) + 0.05 * y - z
    vol["T"][:] = np.clip(sdf / p["trunc"], -1, 1).astype(f32)
    vol["W"][:] = rng.choice(np.array([1.0, 2.0, 3.0], f32), vol["W"].shape)
    shape = vol["T"].shape
    below = np.nextafter(f32(1), f32(0))
    for v, share in ((np.nan, 0.01), (1.0, 0.01), (-1.0, 0.01), (-0.0, 0.01)):
        vol["T"][rng.random(shape) < share] = v
    for v, share in ((0.0, 0.02), (below, 0.02), (np.nan, 0.01)):
        vol["W"][rng.random(shape) < share] = v
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    Z = 1.2 + 0.02 * np.sin(xx / 5.0) + 0.003 * yy + rng.uniform(-0.01, 0.01, (h, w))
    d = (f32(CAM["fx"]) * f32(CAM["baseline"]) / Z - CAM["doffs"]).astype(f32)
    for v, share in ((np.nan, 0.05), (-0.0, 0.03), (np.inf, 0.02), (3e9, 0.02)):
        d[rng.random((h, w)) < share] = v
    return vol, d


def scalar_eval(vol, p, D, cam, tp, M):
    """Step 2 of the header, one cell at a time in float32 scalars, the chunk sums in cell order and the tree."""
    g = [f32(v) for v in np.asarray(M, np.float64).reshape(12)]
    T, Wt = vol["T"], vol["W"]
    nz, ny, nx = T.shape
    H, W = D.shape
    s = tp["step"]
    ncx, ncy = (W - 1) // s + 1, (H - 1) // s + 1
    fb = f32(f32(cam["fx"]) * f32(cam["baseline"]))
    fx, fy, cx, cy, doffs = (f32(cam[k]) for k in ("fx", "fy", "cx", "cy", "doffs"))
    o = [f32(v) for v in p["origin"]]
    vox, one = f32(p["voxel"]), f32(1)
    cells = ncx * ncy
    chunks = []
    count = 0
    with np.errstate(all="ignore"):
        for c0 in range(0, cells, 32):
            acc = [0.0] * 28
            for c in range(c0, min(c0 + 32, cells)):
                px, py = min((c % ncx) * s + s // 2, W - 1), min((c // ncx) * s + s // 2, H - 1)
                d = D[py, px]
                sd = d + doffs
                if not (d >= 0 and d <= f32(1e9) and sd > 0):
                    continue
                Z = fb / sd
                if not Z <= f32(tp["max_depth"]):
                    continue
                X, Y = ((f32(px) - cx) * Z) / fx, ((f32(py) - cy) * Z) / fy
                Pw, i0, fr, good = [], [], [], True
                for e, n in enumerate((nx, ny, nz)):
                    Pw.append(((g[4 * e] * X + g[4 * e + 1] * Y) + g[4 * e + 2] * Z) + g[4 * e + 3])
                    q = (Pw[e] - o[e]) / vox
                    fl = np.floor(q)
                    good = good and bool(fl >= 0 and fl <= f32(n - 2))
                    i0.append(int(fl) if good else 0)
                    fr.append(q - fl)
                if not good:
                    continue
                cc = []
                for q8 in range(8):
                    i, j, k = i0[0] + (q8 & 1), i0[1] + ((q8 >> 1) & 1), i0[2] + (q8 >> 2)
                    if not (Wt[k, j, i] >= f32(tp["min_weight"]) and abs(T[k, j, i]) < one):
                        good = False
                    cc.append(T[k, j, i])
                if not good:
                    continue
                count += 1
                gx, gy, gz = one - fr[0], one - fr[1], one - fr[2]
                x00, x10 = cc[0] * gx + cc[1] * fr[0], cc[2] * gx + cc[3] * fr[0]
                x01, x11 = cc[4] * gx + cc[5] * fr[0], cc[6] * gx + cc[7] * fr[0]
                y0, y1 = x00 * gy + x10 * fr[1], x01 * gy + x11 * fr[1]
                r = y0 * gz + y1 * fr[2]
                G = [(((cc[1] - cc[0]) * gy + (cc[3] - cc[2]) * fr[1]) * gz +
                      ((cc[5] - cc[4]) * gy + (cc[7] - cc[6]) * fr[1]) * fr[2]) / vox,
                     ((x10 - x00) * gz + (x11 - x01) * fr[2]) / vox, (y1 - y0) / vox]
                wt = float(one if abs(r) <= f32(tp["huber"]) else f32(tp["huber"]) / abs(r))
                a = [float(v) for v in G]
                w0, w1, w2 = (2.0 * float(v) for v in Pw)
                J = [(a[1] * -w2) + (a[2] * w1), (a[0] * w2) + (a[2] * -w0), (a[0] * -w1) + (a[1] * w0)] + a
                rd = float(r)
                terms = [(wt * J[i]) * J[j] for i in range(6) for j in range(i, 6)]
                terms += [-((wt * J[i]) * rd) for i in range(6)] + [(wt * rd) * rd]
                acc = [x + t for x, t in zip(acc, terms)]
            chunks.append(acc)
    while len(chunks) & (len(chunks) - 1):
        chunks.append([0.0] * 28)
    while len(chunks) > 1:
        chunks = [[x + y for x, y in zip(chunks[i], chunks[i + 1])] for i in range(0, len(chunks), 2)]
    return chunks[0], count


def scalar_solve(A, b):
    """The header's elimination: partial pivoting on the first row of the largest |a_ij|, back substitution."""
    A = [list(r) for r in A]
    b = list(b)
    k = len(b)
    for j in range(k):
        p = j
        for i in range(j + 1, k):
            if abs(A[i][j]) > abs(A[p][j]):
                p = i
        if not abs(A[p][j]) > 0:
            return None
        A[j], A[p], b[j], b[p] = A[p], A[j], b[p], b[j]
        for i in range(j + 1, k):
            f = A[i][j] / A[j][j]
            for c in range(j + 1, k):
                A[i][c] = A[i][c] - f * A[j][c]
            b[i] = b[i] - f * b[j]
    x = [0.0] * k
    for i in range(k - 1, -1, -1):
        v = b[i]
        for c in range(i + 1, k):
            v = v - A[i][c] * x[c]
        x[i] = v / A[i][i]
    return x if all(math.isfinite(v) for v in x) else None


def scalar_track(vol, p, tp, D, motion, prev, cam):
    """Steps 1, 3 and 4 of the header for one frame around scalar_eval."""
    P = [float(v) for v in np.asarray(prev).reshape(12)]
    if motion is None:
        pred = P
    else:
        m = [float(v) for v in np.asarray(motion).reshape(12)]
        Ri = [[m[4 * c + r] for c in range(3)] for r in range(3)]
        ti = [-(((m[r] * m[3]) + (m[4 + r] * m[7])) + (m[8 + r] * m[11])) for r in range(3)]
        pred = []
        for r in range(3):
            pred += [((P[4 * r] * Ri[0][c]) + (P[4 * r + 1] * Ri[1][c])) + (P[4 * r + 2] * Ri[2][c]) for c in range(3)]
            pred.append((((P[4 * r] * ti[0]) + (P[4 * r + 1] * ti[1])) + (P[4 * r + 2] * ti[2])) + P[4 * r + 3])
    M, applied, status = list(pred), 0, 0
    for r in range(tp["rounds"] + 1):
        v, cnt = scalar_eval(vol, p, D, cam, tp, M)
        cost0 = v[27] if r == 0 else cost0
        if cnt < tp["min_corr"]:
            status = 1 if r == 0 else 0
            break
        if r == tp["rounds"]:
            break
        it = iter(v)
        A = [[0.0] * 6 for _ in range(6)]
        for a in range(6):
            for bb in range(a, 6):
                A[a][bb] = A[bb][a] = next(it)
        for a in range(6):
            A[a][a] = A[a][a] + tp["damping"]
        x = scalar_solve(A, v[21:27])
        if x is None or max(abs(t) for t in x) <= tp["eps"]:
            break
        q = (x[0] * x[0] + x[1] * x[1]) + x[2] * x[2]
        K = ((0.0, -x[2], x[1]), (x[2], 0.0, -x[0]), (-x[1], x[0], 0.0))
        C = [[(((1.0 - q if i == j else 0.0) + (2.0 * (x[i] * x[j]))) + (2.0 * K[i][j])) / (1.0 + q) for j in range(3)]
             for i in range(3)]
        Mn = []
        for i in range(3):
            row = [((C[i][0] * M[j]) + (C[i][1] * M[4 + j])) + (C[i][2] * M[8 + j]) for j in range(4)]
            row[3] = row[3] + x[3 + i]
            Mn += row
        M, applied = Mn, r + 1
    if status == 0:
        dt = [M[3] - pred[3], M[7] - pred[7], M[11] - pred[11]]
        s = [((M[4 * i] * pred[4 * i]) + (M[4 * i + 1] * pred[4 * i + 1])) + (M[4 * i + 2] * pred[4 * i + 2])
             for i in range(3)]
        ok = math.sqrt((dt[0] * dt[0] + dt[1] * dt[1]) + dt[2] * dt[2]) <= tp["max_shift"] and \
            (((s[0] + s[1]) + s[2]) - 1.0) / 2.0 >= tp["min_cos"]
        status = 0 if ok else 2
    F = pred if status else M
    return np.array(F), (status, cnt, applied, cost0, v[27])


VP = dict(nx=13, ny=11, nz=17, origin=(-0.45, -0.35, 0.8), voxel=0.07, trunc=0.2, max_weight=6.0, color=0)


@pytest.mark.parametrize("rounds", [0, 1, 10])
@pytest.mark.parametrize("step", [1, 3, 8])
@pytest.mark.parametrize("seed", [0, 1])
def test_restatement_equals_the_scalar_loop(seed, step, rounds):
    h, w = 23, 31
    p = dict(VP, nx=VP["nx"] + 2 * seed, nz=VP["nz"] - 2 * seed)
    vol, d = planted(seed, p, h, w)
    tp = dict(TP, step=step, rounds=rounds, damping=0.5 * seed, huber=0.05 if seed else 0.3, max_depth=1.25 + seed)
    prev = pose((0.01, -0.02, 0.005), (0.02, -0.01, 0.03))
    motion = pose((0.003, 0.004, -0.002), (0.01, 0.0, -0.02))
    cam = preprocess._ego_cam(CAM)
    v_np = preprocess.fuse_track_eval(vol, p, d, cam, preprocess.fuse_track_params(tp), prev.ravel())
    v_sc, cnt = scalar_eval(vol, p, d, CAM, tp, prev.ravel())
    assert cnt == v_np[3] and cnt > (40 if step == 1 else 2)
    got = np.concatenate([v_np[0][np.triu_indices(6)], v_np[1], [v_np[2]]])
    assert np.array_equal(got.view(np.uint64), np.array(v_sc).view(np.uint64))
    poses, stats = preprocess.fuse_track(vol, p, tp, d[None], motion[None], prev, CAM)
    F, st = scalar_track(vol, p, tp, d, motion, prev, CAM)
    assert np.array_equal(poses[0].ravel().view(np.uint64), F.view(np.uint64))
    assert tuple(stats[0].tolist()) == st


def trilinear64(T, q):
    i0 = np.floor(q).astype(int)
    fr = q - i0
    v = 0.0
    for q8 in range(8):
        b = [(q8 >> e) & 1 for e in range(3)]
        wgt = np.prod([fr[e] if b[e] else 1 - fr[e] for e in range(3)])
        v += wgt * float(T[i0[2] + b[2], i0[1] + b[1], i0[0] + b[0]])
    return v


def test_gradient_equals_finite_differences():
    rng = np.random.default_rng(3)
    p = dict(VP, voxel=0.05)
    vol = preprocess.fuse_new_volume(p)
    vol["T"][:] = rng.uniform(-0.9, 0.9, vol["T"].shape).astype(f32)
    vol["W"][:] = 1.0
    h, w = 23, 31
    d = np.full((h, w), f32(20.0) / f32(1.1) - f32(CAM["doffs"]), f32)
    M = pose((0.02, -0.01, 0.0), (0.0, 0.0, 0.0)).ravel()
    ok, r, G, Pw = preprocess.fuse_track_cells(vol, p, d, preprocess._ego_cam(CAM), 1, 1.0, np.inf, M)
    assert ok.sum() > 100
    o = np.array(p["origin"], np.float64)
    for c in np.flatnonzero(ok)[::7]:
        q = (Pw[c].astype(np.float64) - o) / np.float64(f32(p["voxel"]))
        h_ = 1e-6
        num = [(trilinear64(vol["T"], q + h_ * np.eye(3)[e]) - trilinear64(vol["T"], q - h_ * np.eye(3)[e])) /
               (2 * h_ * float(f32(p["voxel"]))) for e in range(3)]
        assert np.allclose(G[c], num, rtol=1e-3, atol=1e-3), (c, G[c], num)
        assert abs(float(r[c]) - trilinear64(vol["T"], q)) < 1e-4


def test_planar_volume_one_round_recovers_the_offset():
    """T = (z - 1.0) / mu and every frame point on z = 1.0 + delta: one round recovers -delta in t_z.  A plane fixes
    only three of the six degrees of freedom, so N is singular and the solve needs a damping, here one that is
    negligible against N's entries (about 1e7)."""
    p = dict(nx=41, ny=31, nz=21, origin=(-1.0, -0.75, 0.5), voxel=0.05, trunc=0.2, max_weight=6.0, color=0)
    vol = preprocess.fuse_new_volume(p)
    z = p["origin"][2] + np.arange(p["nz"]) * f32(p["voxel"])
    vol["T"][:] = np.clip((z - 1.0) / 0.2, -1, 1).astype(f32)[:, None, None]
    vol["W"][:] = 1.0
    delta = 0.023
    fb = f32(f32(CAM["fx"]) * f32(CAM["baseline"]))
    d = np.full((23, 31), fb / f32(1.0 + delta) - f32(CAM["doffs"]), f32)
    tp = dict(TP, rounds=1, huber=10.0, damping=1e-6)
    poses, stats = preprocess.fuse_track(vol, p, tp, d[None], None, pose(), CAM)
    assert stats[0]["status"] == 0 and stats[0]["rounds"] == 1
    assert abs(poses[0, 2, 3] + delta) < 2e-6, poses[0]
    assert np.abs(poses[0, :, :3] - np.eye(3)).max() < 1e-5 and np.abs(poses[0, :2, 3]).max() < 1e-5


def corner_scene(h=48, w=64):
    """A room corner: side wall x = -0.8, floor y = 0.6, back wall z = 2.0, its TSDF and the depth from pose()."""
    f = 60.0 * w / 64
    cam = dict(fx=f, fy=f, cx=(w - 1) / 2, cy=(h - 1) / 2, baseline=0.5, doffs=0.0)
    p = dict(nx=64, ny=52, nz=72, origin=(-1.0, -0.9, 0.3), voxel=0.03, trunc=0.15, max_weight=6.0, color=0)
    x = p["origin"][0] + np.arange(p["nx"]) * p["voxel"]
    y = p["origin"][1] + np.arange(p["ny"]) * p["voxel"]
    z = p["origin"][2] + np.arange(p["nz"]) * p["voxel"]
    Z, Y, X = np.meshgrid(z, y, x, indexing="ij")
    sdf = np.minimum(np.minimum(2.0 - Z, 0.6 - Y), X + 0.8)
    vol = preprocess.fuse_new_volume(p)
    vol["T"][:] = np.clip(sdf / p["trunc"], -1, 1).astype(f32)
    vol["W"][:] = 1.0
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    u, v = (xx - cam["cx"]) / cam["fx"], (yy - cam["cy"]) / cam["fy"]
    with np.errstate(divide="ignore"):
        t = np.stack([np.full_like(u, 2.0), np.where(v > 0, 0.6 / v, np.inf), np.where(u < 0, -0.8 / u, np.inf)])
    depth = t.min(0)
    fb = np.float64(f32(cam["fx"]) * f32(cam["baseline"]))
    return p, vol, (fb / depth).astype(f32), cam


def test_corner_volume_recovers_a_perturbation():
    """A seeded 5 cm, 0.5 degree perturbation is recovered within 1 mm and 0.01 degree in 10 rounds.  The trilinear T
    of a cube that straddles a crease between two walls is not the distance, so about 100 of the 2852 cells keep a
    residual of up to 0.04 at the true pose; a Huber threshold of 0.01 keeps them from biasing the fit."""
    p, vol, d, cam = corner_scene()
    rng = np.random.default_rng(5)
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    tdir = rng.normal(size=3)
    tdir /= np.linalg.norm(tdir)
    start = pose(axis * math.radians(0.5), 0.05 * tdir)
    tp = dict(TP, rounds=10, huber=0.01, damping=0.0)
    poses, stats = preprocess.fuse_track(vol, p, tp, d[None], None, start, cam)
    t_err, r_err = preprocess.trajectory_errors(poses, pose()[None])
    assert stats[0]["status"] == 0 and stats[0]["rounds"] <= 10
    assert t_err[0] < 1e-3 and r_err[0] < 0.01, (t_err, r_err, stats)
    assert stats[0]["cost"] < 0.05 * stats[0]["cost0"]


def test_statuses():
    p, vol, d, cam = corner_scene(24, 32)
    start = pose((0.004, -0.003, 0.002), (0.03, -0.02, 0.02))
    empty = preprocess.fuse_new_volume(p)
    poses, stats = preprocess.fuse_track(empty, p, TP, d[None], None, start, cam)
    assert stats[0]["status"] == 1 and stats[0]["n_corr"] == 0 and stats[0]["rounds"] == 0
    assert np.array_equal(poses[0], start)
    poses, stats = preprocess.fuse_track(vol, p, dict(TP, max_shift=1e-6), d[None], None, start, cam)
    assert stats[0]["status"] == 2 and stats[0]["rounds"] > 0 and np.array_equal(poses[0], start)
    poses, stats = preprocess.fuse_track(vol, p, dict(TP, min_cos=1.0), d[None], None, start, cam)
    assert stats[0]["status"] == 2 and np.array_equal(poses[0], start)
    poses, stats = preprocess.fuse_track(vol, p, dict(TP, rounds=0), d[None], None, start, cam)
    assert stats[0]["status"] == 0 and stats[0]["rounds"] == 0 and np.array_equal(poses[0], start)
    assert stats[0]["cost"] == stats[0]["cost0"] > 0
    full = preprocess.fuse_track(vol, p, TP, d[None], None, start, cam)[1][0]
    early = preprocess.fuse_track(vol, p, dict(TP, eps=1e-4), d[None], None, start, cam)[1][0]
    none = preprocess.fuse_track(vol, p, dict(TP, eps=1e9), d[None], None, start, cam)[1][0]
    assert full["rounds"] == 10 and 0 < early["rounds"] < 10 and none["rounds"] == 0, (full, early, none)
    few = preprocess.fuse_track(vol, p, dict(TP, min_corr=10 ** 6), d[None], None, start, cam)[1][0]
    assert few["status"] == 1 and few["n_corr"] > 0


def clip3(seed):
    rng = np.random.default_rng(seed)
    p, vol, d, cam = corner_scene(24, 32)
    p = dict(p, color=1)
    vol = dict(vol, C=rng.integers(0, 256, vol["T"].shape + (3,)).astype(np.uint8))
    disp = np.stack([d, d * f32(1.01), d * f32(0.99)])
    disp[1][rng.random(d.shape) < 0.1] = np.nan
    motions = np.stack([pose(rng.uniform(-0.004, 0.004, 3), rng.uniform(-0.02, 0.02, 3)) for _ in range(3)])
    frames = rng.integers(0, 256, (3, 24, 32, 3)).astype(np.uint8)
    return p, vol, disp, motions, frames, cam


def copy(vol):
    return {k: None if v is None else v.copy() for k, v in vol.items()}


def same_vol(a, b):
    return all(np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)) for k in ("T", "W", "C"))


def test_one_call_equals_calls_of_one_and_integrating_equals_aligning_then_pushing():
    p, vol, disp, motions, frames, cam = clip3(7)
    tp = dict(TP, rounds=4, integrate=1, damping=0.1)
    prev = pose((0.002, 0.0, 0.0), (0.01, 0.0, 0.0))
    v1 = copy(vol)
    poses, stats = preprocess.fuse_track(v1, p, tp, disp, motions, prev, cam, frames)
    v2, P, got = copy(vol), prev, []
    for k in range(3):
        pk, sk = preprocess.fuse_track(v2, p, tp, disp[k:k + 1], motions[k:k + 1], P, cam, frames[k:k + 1])
        got.append((pk[0], sk[0]))
        P = pk[0]
    assert same_vol(v1, v2)
    for k in range(3):
        assert np.array_equal(got[k][0], poses[k]) and got[k][1].tobytes() == stats[k].tobytes()
    v3, P = copy(vol), prev
    for k in range(3):
        pk, sk = preprocess.fuse_track(v3, p, dict(tp, integrate=0), disp[k:k + 1], motions[k:k + 1], P, cam)
        assert np.array_equal(pk[0], poses[k]) and sk[0].tobytes() == stats[k].tobytes()
        preprocess.fuse_integrate(v3, p, disp[k:k + 1], pk, cam, tp["max_depth"], frames[k:k + 1])
        P = pk[0]
    assert same_vol(v1, v3)
    assert not same_vol(v1, vol)


def test_null_motions_equal_identity_motions():
    p, vol, disp, _, frames, cam = clip3(8)
    tp = dict(TP, rounds=3, integrate=1)
    prev = pose((0.002, 0.001, 0.0), (0.01, 0.02, 0.0))
    a = preprocess.fuse_track(copy(vol), p, tp, disp, None, prev, cam, frames)
    b = preprocess.fuse_track(copy(vol), p, tp, disp, np.stack([pose()] * 3), prev, cam, frames)
    assert np.array_equal(a[0], b[0]) and a[1].tobytes() == b[1].tobytes()


def test_trajectory_errors():
    gt = np.stack([pose(), pose((0, 0.1, 0), (1, 2, 3))])
    est = np.stack([pose((0.0, 0.0, math.radians(2.0)), (0.3, 0.4, 0.0)), gt[1]])
    t, r = preprocess.trajectory_errors(est, gt)
    assert np.allclose(t, [0.5, 0.0]) and np.allclose(r, [2.0, 0.0], atol=1e-6)


def test_relocalisation_with_exact_disparities():
    """The GPU file's re-localisation on synth.rigid_stereo_clip at KITTI's size, with the clip's exact disparities in
    the model and the frame instead of a stereo context's: 8 frames fused at their true poses, frame 8 aligned from its
    true pose perturbed by 0.15 m and 1 degree must fall to <= 25 % of both, the bound the stereo case misses."""
    from of_dis_b200 import synth

    kitti = dict(fx=721.5, fy=721.5, cx=609.6, cy=172.9, baseline=0.54, doffs=0.0)
    n = 9
    rels = [pose((0.0, math.radians(0.3 * (k % 3 - 1)), 0.0), (0.02 * (k % 2), 0.0, -0.5)) for k in range(n - 1)]
    clip = synth.rigid_stereo_clip(n - 1, 375, 1242, 1, 2, kitti, rels, block={"velocity": (0.0, 0.0, 0.0)})
    G, d = clip["abs"], clip["disp"].astype(f32)
    p = dict(nx=160, ny=55, nz=280, origin=(-8.0, -3.0, 3.0), voxel=0.1, trunc=0.3, max_weight=64.0, color=0)
    tp = dict(step=2, rounds=10, min_weight=1.0, max_depth=30.0, huber=0.2, damping=1.0, min_corr=100, max_shift=0.5,
              min_cos=math.cos(math.radians(5.0)), eps=1e-7, integrate=0)
    vol = preprocess.fuse_integrate(preprocess.fuse_new_volume(p), p, d[:8], G[:8], kitti)
    rng = np.random.default_rng(11)
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    tdir = rng.normal(size=3)
    tdir /= np.linalg.norm(tdir)
    start = np.concatenate([rot(axis * math.radians(1.0)) @ G[8][:, :3], (G[8][:, 3] + 0.15 * tdir)[:, None]], 1)
    got, st = preprocess.fuse_track(vol, p, tp, d[8:9], None, start, kitti)
    t_err, r_err = preprocess.trajectory_errors(got, G[8:9])
    assert st[0]["status"] == 0 and t_err[0] <= 0.25 * 0.15 and r_err[0] <= 0.25 * 1.0, (t_err, r_err, st)
