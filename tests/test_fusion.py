"""preprocess.fuse_integrate, fuse_extract and fuse_render against scalar per-voxel, per-edge and per-ray loops written
from include/ofdis_b200.h; chunked pushes, the skip rules, the weight cap, a fused plane, and the batch command's --fuse
refusals (no device needed)."""
import math

import numpy as np
import pytest

from of_dis_b200 import preprocess

f32 = np.float32
QNAN = np.uint32(0x7FC00000).view(np.float32)
CAM = dict(fx=40.0, fy=38.5, cx=15.25, cy=11.5, baseline=0.5, doffs=0.25)


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


def params(**kw):
    p = dict(nx=13, ny=9, nz=17, origin=(-0.7, -0.45, 0.6), voxel=0.1, trunc=0.25, max_weight=5.0, color=1)
    p.update(kw)
    return p


def scene(seed, n=3, h=24, w=32, ch=3):
    """Disparities of a slanted plane with planted NaN, -0, +inf and 3e9, poses that keep part of the volume behind and
    beside the frustum, and random frames."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    disp = []
    for k in range(n):
        Z = 1.2 + 0.02 * x + 0.01 * y + 0.05 * k + rng.uniform(-0.02, 0.02, (h, w))
        d = (f32(CAM["fx"]) * f32(CAM["baseline"]) / Z - CAM["doffs"]).astype(f32)
        d[rng.random((h, w)) < 0.05] = np.nan
        d[rng.random((h, w)) < 0.03] = -0.0
        d[rng.random((h, w)) < 0.02] = np.inf
        d[rng.random((h, w)) < 0.02] = 3e9
        disp.append(d)
    poses = np.stack([pose(rng.uniform(-0.1, 0.1, 3), rng.uniform(-0.2, 0.2, 3) + (0, 0, -0.1 * k)) for k in range(n)])
    frames = rng.integers(0, 256, (n, h, w, ch) if ch == 3 else (n, h, w)).astype(np.uint8)
    return np.stack(disp), poses, frames


# ---- scalar loops written from the header ---------------------------------------------------------------------------
def loop_integrate(vol, p, disp, poses, cam, max_depth, frames):
    T, W, C = vol["T"], vol["W"], vol["C"]
    nz, ny, nx = T.shape
    n, H, Wd = disp.shape
    c = {k: f32(cam[k]) for k in preprocess.STEREO_CAMERA_FIELDS}
    fb, mu, maxw, md = f32(c["fx"] * c["baseline"]), f32(p["trunc"]), f32(p["max_weight"]), f32(max_depth)
    o, vox = [f32(v) for v in p["origin"]], f32(p["voxel"])
    with np.errstate(all="ignore"):
        for k in range(n):
            P = poses[k].reshape(12)
            g = [f32(P[4 * c_ + r]) if c_ < 3 else None for r in range(3) for c_ in range(4)]
            for r in range(3):
                g[4 * r + 3] = f32(-(((P[r] * P[3]) + (P[4 + r] * P[7])) + (P[8 + r] * P[11])))
            for kk in range(nz):
                for j in range(ny):
                    for i in range(nx):
                        X, Y, Z = o[0] + f32(i) * vox, o[1] + f32(j) * vox, o[2] + f32(kk) * vox
                        Xc = ((g[0] * X + g[1] * Y) + g[2] * Z) + g[3]
                        Yc = ((g[4] * X + g[5] * Y) + g[6] * Z) + g[7]
                        Zc = ((g[8] * X + g[9] * Y) + g[10] * Z) + g[11]
                        if not Zc > 0:
                            continue
                        u = (c["fx"] * Xc) / Zc + c["cx"]
                        v = (c["fy"] * Yc) / Zc + c["cy"]
                        uu, vv = u + f32(0.5), v + f32(0.5)
                        if not (0 <= uu < f32(Wd) and 0 <= vv < f32(H)):
                            continue
                        px, py = int(np.floor(uu)), int(np.floor(vv))
                        d = disp[k, py, px]
                        s = d + c["doffs"]
                        if not (0 <= d <= f32(1e9) and s > 0):
                            continue
                        z = fb / s
                        if z > md:
                            continue
                        sdf = z - Zc
                        if sdf < -mu:
                            continue
                        f = min(f32(1), sdf / mu)
                        w0 = W[kk, j, i]
                        w1 = w0 + f32(1)
                        T[kk, j, i] = (T[kk, j, i] * w0 + f) / w1
                        if C is not None:
                            fr = frames[k].reshape(H, Wd, -1)[py, px]
                            for ch in range(3):
                                obs = f32(fr[ch if fr.size == 3 else 0])
                                C[kk, j, i, ch] = int(np.floor((f32(C[kk, j, i, ch]) * w0 + obs) / w1 + f32(0.5)))
                        W[kk, j, i] = min(w1, maxw)
    return vol


def loop_extract(vol, p, min_weight):
    T, W, C = vol["T"], vol["W"], vol["C"]
    nz, ny, nx = T.shape
    o, vox, mw = [f32(v) for v in p["origin"]], f32(p["voxel"]), f32(min_weight)
    out = []
    with np.errstate(all="ignore"):
        for kk in range(nz):
            for j in range(ny):
                for i in range(nx):
                    for e, (di, dj, dk) in enumerate(((1, 0, 0), (0, 1, 0), (0, 0, 1))):
                        i2, j2, k2 = i + di, j + dj, kk + dk
                        if i2 >= nx or j2 >= ny or k2 >= nz:
                            continue
                        Ta, Tb = T[kk, j, i], T[k2, j2, i2]
                        if not (W[kk, j, i] >= mw and W[k2, j2, i2] >= mw and abs(Ta) < 1 and abs(Tb) < 1
                                and (Ta > 0) != (Tb > 0)):
                            continue
                        t = Ta / (Ta - Tb)
                        P = [o[0] + f32(i) * vox, o[1] + f32(j) * vox, o[2] + f32(kk) * vox]
                        P[e] = P[e] + t * vox
                        gx = T[kk, j, min(i + 1, nx - 1)] - T[kk, j, max(i - 1, 0)]
                        gy = T[kk, min(j + 1, ny - 1), i] - T[kk, max(j - 1, 0), i]
                        gz = T[min(kk + 1, nz - 1), j, i] - T[max(kk - 1, 0), j, i]
                        L = np.sqrt((gx * gx + gy * gy) + gz * gz)
                        nrm = [g / L for g in (gx, gy, gz)] if L > 0 else [QNAN] * 3
                        col = (0, 0, 0) if C is None else tuple(C[kk, j, i] if t < f32(0.5) else C[k2, j2, i2])
                        out.append(tuple(P) + tuple(nrm) + col + (0,))
    return np.array(out, preprocess.FUSE_POINT_DTYPE)


def loop_render(vol, p, P, cam, zn, zf, st, mw, w, h):
    T, W = vol["T"], vol["W"]
    nz, ny, nx = T.shape
    c = {k: f32(cam[k]) for k in preprocess.STEREO_CAMERA_FIELDS}
    o, vox = [f32(v) for v in p["origin"]], f32(p["voxel"])
    q = P.reshape(12).astype(f32)
    zn, zf, st, mw = f32(zn), f32(zf), f32(st), f32(mw)
    depth = np.full((h, w), QNAN, f32)

    def sample(Zs, r0, r1):
        cx, cy = r0 * Zs, r1 * Zs
        idx, fr = [], []
        for e, dim in enumerate((nx, ny, nz)):
            Pw = ((q[4 * e] * cx + q[4 * e + 1] * cy) + q[4 * e + 2] * Zs) + q[4 * e + 3]
            qq = (Pw - o[e]) / vox
            fl = np.floor(qq)
            if not (fl >= 0 and fl <= f32(dim - 2)):
                return None
            idx.append(int(fl))
            fr.append(qq - fl)
        i, j, k = idx
        for dk in (0, 1):
            for dj in (0, 1):
                for di in (0, 1):
                    if not W[k + dk, j + dj, i + di] >= mw:
                        return None
        one = f32(1)

        def lx(jj, kk):
            return T[kk, jj, i] * (one - fr[0]) + T[kk, jj, i + 1] * fr[0]

        y0 = lx(j, k) * (one - fr[1]) + lx(j + 1, k) * fr[1]
        y1 = lx(j, k + 1) * (one - fr[1]) + lx(j + 1, k + 1) * fr[1]
        return y0 * (one - fr[2]) + y1 * fr[2]

    with np.errstate(all="ignore"):
        for y in range(h):
            for x in range(w):
                r0, r1 = (f32(x) - c["cx"]) / c["fx"], (f32(y) - c["cy"]) / c["fy"]
                prev = None
                for s in range(preprocess.FUSE_MAX_SAMPLES + 1):
                    Zs = zn + f32(s) * st
                    if not Zs <= zf:
                        break
                    Ts = sample(Zs, r0, r1)
                    if Ts is not None and prev is not None and prev[1] > 0 and Ts <= 0:
                        depth[y, x] = prev[0] + st * (prev[1] / (prev[1] - Ts))
                        break
                    prev = None if Ts is None else (Zs, Ts)
    return depth


def same(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_restatements_equal_the_loops(seed):
    ch = 3 if seed != 1 else 1
    p = params(color=1 if seed != 2 else 0)
    disp, poses, frames = scene(seed, ch=ch)
    a, b = preprocess.fuse_new_volume(p), preprocess.fuse_new_volume(p)
    preprocess.fuse_integrate(a, p, disp, poses, CAM, max_depth=2.0 if seed == 1 else np.inf, frames=frames)
    loop_integrate(b, p, disp, poses, CAM, 2.0 if seed == 1 else np.inf, frames)
    for k in ("T", "W", "C"):
        assert (a[k] is None and b[k] is None) or same(a[k], b[k]), k
    assert (a["W"] > 0).mean() > 0.05 and (a["W"] == 0).any()
    for mw in (1.0, 2.0):
        got, exp = preprocess.fuse_extract(a, p, mw), loop_extract(b, p, mw)
        assert len(got) > 0 and same(got, exp), mw
    h, w = 24, 32
    dep = preprocess.fuse_render(a, p, poses[:2], CAM, 0.5, 3.0, 0.05, 1.0, w, h)
    for k in range(2):
        assert same(dep[k], loop_render(b, p, poses[k], CAM, 0.5, 3.0, 0.05, 1.0, w, h)), k
    assert np.isfinite(dep).any()


def test_chunked_pushes_equal_one_push():
    p = params()
    disp, poses, frames = scene(5, n=5)
    one = preprocess.fuse_integrate(preprocess.fuse_new_volume(p), p, disp, poses, CAM, frames=frames)
    for cut in ((1, 1, 1, 1, 1), (2, 3), (4, 1)):
        v, k0 = preprocess.fuse_new_volume(p), 0
        for c in cut:
            preprocess.fuse_integrate(v, p, disp[k0:k0 + c], poses[k0:k0 + c], CAM, frames=frames[k0:k0 + c])
            k0 += c
        assert all(same(v[k], one[k]) for k in ("T", "W", "C")), cut


def test_skipped_voxels_are_untouched():
    """Behind the camera, outside the image, at the known(d) edges and beyond max_depth: the voxel keeps its bytes."""
    h, w = 24, 32
    p = params(nx=3, ny=3, nz=1, origin=(-0.05, -0.05, 1.0), voxel=0.05, trunc=0.5)
    fb = f32(CAM["fx"]) * f32(CAM["baseline"])
    base = (fb / f32(1.2) - f32(CAM["doffs"])).astype(f32)

    def push(d=base, P=pose(), md=np.inf):
        v = preprocess.fuse_new_volume(p)
        v["T"][:] = f32(0.25)
        v["W"][:] = f32(2)
        disp = np.full((1, h, w), d, f32)
        preprocess.fuse_integrate(v, p, disp, P[None], CAM, max_depth=md, frames=np.zeros((1, h, w, 3), np.uint8))
        return (v["W"] != 2).sum()

    assert push() == 9
    assert push(P=pose(t=(0, 0, 5.0))) == 0, "behind the camera"
    assert push(P=pose(t=(3.0, 0, 0))) == 0, "outside the image"
    for d in (np.nan, -1e-30, 1.0001e9, np.inf):
        assert push(d=f32(d)) == 0, d
    assert push(d=-f32(0.0)) == 9, "-0 is known"
    assert push(md=1.1) == 0, "beyond max_depth"
    assert push(md=1.3) == 9


def test_weight_caps_at_max_weight():
    p = params(max_weight=3.0)
    disp, poses, frames = scene(7, n=6)
    disp[:] = disp[:1]
    poses[:] = poses[:1]
    v = preprocess.fuse_integrate(preprocess.fuse_new_volume(p), p, disp, poses, CAM, frames=frames)
    assert v["W"].max() == 3.0 and (v["W"] == 3.0).sum() > 10


def test_a_plane_fused_from_exact_depth():
    """A fronto-parallel plane at Z = 2 seen by three cameras: points within one voxel of it, normals facing the
    camera, rendered depth within step / 2."""
    h, w = 48, 64
    cam = dict(fx=60.0, fy=60.0, cx=31.5, cy=23.5, baseline=0.5, doffs=0.0)
    p = params(nx=40, ny=30, nz=30, origin=(-1.0, -0.75, 1.3), voxel=0.05, trunc=0.2, color=0)
    poses = np.stack([pose(t=(0.0, 0, 0)), pose(t=(0.1, 0, 0)), pose((0, 0.03, 0), (-0.05, 0.02, 0.1))])
    y, x = np.mgrid[0:h, 0:w]
    disp = []
    for P in poses:
        # depth of the plane Z_world = 2 along each pixel ray of camera P
        ray = np.stack([(x - cam["cx"]) / cam["fx"], (y - cam["cy"]) / cam["fy"], np.ones_like(x, float)], -1)
        dw = ray @ P[:, :3].T
        Zc = (2.0 - P[2, 3]) / dw[..., 2]
        disp.append((f32(cam["fx"] * cam["baseline"]) / Zc).astype(f32))
    v = preprocess.fuse_integrate(preprocess.fuse_new_volume(p), p, np.stack(disp), poses, cam)
    pts = preprocess.fuse_extract(v, p, 1.0)
    assert len(pts) > 500
    assert np.abs(pts["z"] - 2.0).max() <= p["voxel"]
    assert (pts["nz"][np.isfinite(pts["nz"])] < -0.9).mean() > 0.95
    dep = preprocess.fuse_render(v, p, poses[:1], cam, 1.4, 2.8, 0.02, 1.0, w, h)[0]
    known = np.isfinite(dep)
    assert known.mean() > 0.5 and np.abs(dep[known] - 2.0).max() <= 0.01


def test_write_fused_ply(tmp_path):
    pts = np.zeros(2, preprocess.FUSE_POINT_DTYPE)
    pts["x"], pts["nz"], pts["r"], pts["b"] = (1.5, -2.0), (-1.0, 0.5), (7, 9), (200, 3)
    path = str(tmp_path / "a.ply")
    preprocess.write_fused_ply(path, pts)
    data = open(path, "rb").read()
    head, body = data.split(b"end_header\n")
    assert b"element vertex 2" in head and len(body) == 2 * 27
    rec = np.frombuffer(body, [("p", "<f4", (6,)), ("c", "u1", (3,))])
    assert (rec["p"][:, 0] == pts["x"]).all() and (rec["c"][:, 0] == pts["r"]).all() and (rec["c"][:, 2] == pts["b"]).all()


# ---- batch command: --fuse is refused where it does not apply (no device needed) ------------------------------------
CAMERA = "721.5,707,16,12,0.54,0.25"
SF = ["--scene-flow", "d.txt", "--camera", CAMERA]
GOOD = "0.1,0.3,-2,-1,1,40,20,60"


def _batch(tmp_path, exe, args):
    import subprocess

    from of_dis_b200 import build

    bindir = build.build_host()
    (tmp_path / "list.txt").write_text("\n")
    preprocess.write_pfm(str(tmp_path / "d.pfm"), np.zeros((24, 32), np.float32))
    (tmp_path / "d.txt").write_text("")
    (tmp_path / "odo").mkdir(exist_ok=True)
    return subprocess.run([str(bindir) + "/" + exe + "_batch", "list.txt"] + args, capture_output=True, text=True,
                          cwd=str(tmp_path))


@pytest.mark.parametrize("exe,args", [
    ("run_OF_INT", ["--fuse", GOOD] + SF), ("run_DE_INT", ["--odometry", "odo", "--fuse", GOOD] + SF),
    ("run_DE_RGB", ["--fuse", GOOD]), ("run_OF_INT", ["--warm-start", "--odometry", "odo", "--fuse", GOOD] + SF),
    ("run_OF_RGB", ["--odometry", "odo", "--fuse"] + SF[:0]),
    ("run_OF_INT", ["--odometry", "odo", "--fuse", "0.1,0.3,-2,-1,1,40,20"] + SF),
    ("run_OF_INT", ["--odometry", "odo", "--fuse", "0.1,0.3,-2,-1,1,40,20,60,5"] + SF),
    ("run_OF_INT", ["--odometry", "odo", "--fuse", "0,0.3,-2,-1,1,40,20,60"] + SF),
    ("run_OF_INT", ["--odometry", "odo", "--fuse", "0.1,-0.3,-2,-1,1,40,20,60"] + SF),
    ("run_OF_INT", ["--odometry", "odo", "--fuse", "0.1,0.3,-2,-1,1,0,20,60"] + SF),
    ("run_OF_INT", ["--odometry", "odo", "--fuse", "0.1,0.3,-2,-1,1,40.5,20,60"] + SF),
    ("run_OF_INT", ["--odometry", "odo", "--fuse", "0.1,0.3,-2,-1,nan,40,20,60"] + SF),
    ("run_OF_INT", ["--odometry", "odo", "--fuse", "0.1,0.3,-2,-1,1,1024,1024,1025"] + SF),
    ("run_OF_INT", ["--odometry", "odo", "--fuse", "0.1,0.3,-2,-1,1,40,20,x"] + SF)])
def test_batch_command_refuses_fuse(tmp_path, exe, args):
    r = _batch(tmp_path, exe, args)
    assert r.returncode == 2, (args, r.stdout, r.stderr)


def test_batch_command_accepts_fuse(tmp_path):
    r = _batch(tmp_path, "run_OF_RGB", ["--odometry", "odo", "--fuse", "0.1,0.3,-2,-1,1,1024,1024,1024"] + SF)
    assert r.returncode == 0, (r.stdout, r.stderr)
    assert not any(p.name.startswith("fused") for p in (tmp_path / "odo").iterdir())
