"""ofdis_fuse_*: the device volume (T, W, colour), extracted points and counts and rendered depth must equal
preprocess.fuse_integrate / fuse_extract / fuse_render bit for bit (gray and RGB contexts, colour on and off, host and
device memory, sizes that no brick divides, volumes partly behind and beside the frustum, disparities with NaN, -0,
+inf and 3e9); chunked pushes, a capacity below the count, fixed launch counts, every argument error with the volume
unchanged, a stereo context's own disparities, the quality on synth.rigid_stereo_clip, and the batch command's --fuse."""
import ctypes
import json
import math

import numpy as np
import pytest

from of_dis_b200 import params, preprocess, synth

pytestmark = pytest.mark.gpu

SMALL = "3 %d 8 8 0.05 0.95 0 8 0.4 %d 1 0 1 10 10 5 1 3 1.6 0"
CAM = dict(fx=40.0, fy=38.5, cx=15.25, cy=11.5, baseline=0.5, doffs=0.25)


@pytest.fixture(scope="module")
def api():
    from of_dis_b200 import api as _api

    _api.lib()
    return _api


def context(api, prm, h, w, max_frames, stream=None):
    scf = 1 << prm.sc_f
    W, H = (w + scf - 1) // scf * scf, (h + scf - 1) // scf * scf
    return api.Context(prm, W, H, prm.p_samp_s, max_frames, stream=stream)


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


def vparams(**kw):
    # 37 x 23 x 41: no brick or scan block divides it; x from -1.9 and z from 0.3 put part of it beside and behind
    p = dict(nx=37, ny=23, nz=41, origin=(-1.9, -0.9, 0.3), voxel=0.07, trunc=0.2, max_weight=6.0, color=1)
    p.update(kw)
    return p


def scene(seed, n, h, w, ch):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    disp = []
    for k in range(n):
        Z = 1.3 + 0.8 * np.sin(x / 9.0) * 0.3 + 0.01 * y + 0.03 * k + rng.uniform(-0.03, 0.03, (h, w))
        d = (np.float32(CAM["fx"]) * np.float32(CAM["baseline"]) / Z - CAM["doffs"]).astype(np.float32)
        d[rng.random((h, w)) < 0.05] = np.nan
        d[rng.random((h, w)) < 0.03] = -0.0
        d[rng.random((h, w)) < 0.02] = np.inf
        d[rng.random((h, w)) < 0.02] = 3e9
        disp.append(d)
    poses = np.stack([pose(rng.uniform(-0.08, 0.08, 3), rng.uniform(-0.2, 0.2, 3) + (0, 0, 0.05 * k))
                      for k in range(n)])
    frames = rng.integers(0, 256, (n, h, w, ch) if ch == 3 else (n, h, w)).astype(np.uint8)
    return np.stack(disp), poses, frames


def same(a, b, what):
    if a is None and b is None:
        return
    ab, bb = np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8)
    assert ab.shape == bb.shape and (ab == bb).all(), "%s differs" % what


def check_volume(ctx, vol, what):
    got = ctx.fuse_volume()
    for k in ("T", "W", "C"):
        same(got[k], vol[k], "%s %s" % (what, k))


@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("color", [0, 1])
@pytest.mark.parametrize("ch", [1, 3])
def test_device_equals_the_restatement(ch, color, mem, api):
    import torch

    h, w, n = 45, 61, 5
    disp, poses, frames = scene(10 * ch + color, n, h, w, ch)
    prm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=ch, nop=2)
    ctx = context(api, prm, h, w, 4)
    p = vparams(color=color)
    ctx.fuse_begin(p)
    vol = preprocess.fuse_new_volume(p)
    fr = frames if color else None
    if mem == "host":
        ctx.fuse_push(disp, poses, CAM, width_org=w, height_org=h, frames=fr, max_depth=2.5)
    else:
        dd = torch.from_numpy(disp).cuda()
        df = torch.from_numpy(frames).cuda()
        ctx.fuse_push(dd.data_ptr(), poses, CAM, width_org=w, height_org=h, frames=df.data_ptr() if color else None,
                      max_depth=2.5, memkind=api.MEM_DEVICE)
    preprocess.fuse_integrate(vol, p, disp, poses, CAM, max_depth=2.5, frames=fr)
    check_volume(ctx, vol, "push")
    assert (vol["W"] > 0).mean() > 0.05 and (vol["W"] == 0).mean() > 0.05
    for mw in (1.0, 3.0):
        exp = preprocess.fuse_extract(vol, p, mw)
        assert len(exp) > 100
        if mem == "host":
            got, total = ctx.fuse_extract(mw)
        else:
            buf = torch.zeros(len(exp) * 28 + 28, dtype=torch.uint8, device="cuda")
            _, total = ctx.fuse_extract(mw, capacity=len(exp) + 1, memkind=api.MEM_DEVICE, out=buf.data_ptr())
            got = buf.cpu().numpy()[:28 * len(exp)].view(preprocess.FUSE_POINT_DTYPE)
        assert total == len(exp)
        same(got, exp, "extract %g" % mw)
    rp = np.concatenate([poses[:2], pose((0, 0.05, 0), (0.3, -0.1, -0.4))[None]])
    exp = preprocess.fuse_render(vol, p, rp, CAM, 0.4, 2.9, 0.035, 1.0, w, h)
    if mem == "host":
        got = ctx.fuse_render(rp, CAM, z_near=0.4, z_far=2.9, step=0.035, width_org=w, height_org=h)
    else:
        out = torch.empty((3, h, w), dtype=torch.float32, device="cuda")
        ctx.fuse_render(rp, CAM, z_near=0.4, z_far=2.9, step=0.035, width_org=w, height_org=h, memkind=api.MEM_DEVICE,
                        out=out.data_ptr())
        ctx.sync()
        got = out.cpu().numpy()
    assert np.isfinite(exp).mean() > 0.2 and np.isnan(exp).any()
    same(got, exp, "render")
    ctx.close()


def test_chunks_capacity_and_launch_counts(api):
    h, w, n = 45, 61, 65
    disp, poses, frames = scene(3, n, h, w, 3)
    prm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=3, nop=2)
    ctx = context(api, prm, h, w, 64)
    p = vparams(max_weight=40.0)
    ctx.fuse_begin(p)
    before = ctx.launch_count
    ctx.fuse_push(disp, poses, CAM, width_org=w, height_org=h, frames=frames)
    launches = {"push65": ctx.launch_count - before}
    whole = ctx.fuse_volume()
    ctx.fuse_begin(p)
    for k0, k1 in ((0, 1), (1, 30), (30, 64), (64, 65)):
        before = ctx.launch_count
        ctx.fuse_push(disp[k0:k1], poses[k0:k1], CAM, width_org=w, height_org=h, frames=frames[k0:k1])
        launches["push%d" % (k1 - k0)] = ctx.launch_count - before
    vol = preprocess.fuse_integrate(preprocess.fuse_new_volume(p), p, disp, poses, CAM, frames=frames)
    check_volume(ctx, vol, "chunked")
    for k in ("T", "W", "C"):
        same(whole[k], vol[k], "one push " + k)
    exp = preprocess.fuse_extract(vol, p, 1.0)
    for cap in (0, 1, 77, len(exp) - 1):
        before = ctx.launch_count
        got, total = ctx.fuse_extract(1.0, capacity=cap)
        launches["extract"] = ctx.launch_count - before
        assert total == len(exp) and len(got) == cap
        same(got, exp[:cap], "capacity %d" % cap)
    for m in (1, 64):
        before = ctx.launch_count
        ctx.fuse_render(np.repeat(poses[:1], m, 0), CAM, z_near=0.5, z_far=2.0, step=0.05, width_org=w, height_org=h)
        launches["render%d" % m] = ctx.launch_count - before
    assert launches == {"push65": 1, "push1": 1, "push29": 1, "push34": 1, "extract": 3, "render1": 1,
                        "render64": 1}, launches
    ctx.close()


def test_argument_errors_leave_the_volume(api):
    h, w, n = 45, 61, 2
    disp, poses, frames = scene(4, n, h, w, 1)
    prm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=1, nop=2)
    ctx = context(api, prm, h, w, 1)
    L = api.lib()
    nan, inf = float("nan"), float("inf")
    p = vparams()
    cp = api.FuseParams(p["nx"], p["ny"], p["nz"], (ctypes.c_float * 3)(*p["origin"]), p["voxel"], p["trunc"],
                        p["max_weight"], 1)
    assert L.ofdis_fuse_push(ctx._h, 1, api._ptr(disp), h * w, api._ptr(poses), None, inf, None, 0, w, h, 0) == -1, \
        "no live volume"
    count = ctypes.c_long(0)
    assert L.ofdis_fuse_extract(ctx._h, 1.0, None, 0, ctypes.byref(count), 0) == -1
    assert L.ofdis_fuse_get_volume(ctx._h, None, None, None, 0) == -1
    ctx.fuse_begin(p)
    ctx.fuse_push(disp, poses, CAM, width_org=w, height_org=h, frames=frames)
    vol = ctx.fuse_volume()
    cam = api.StereoCamera(*[CAM[k] for k in preprocess.STEREO_CAMERA_FIELDS])

    def push(n=n, d=disp.ctypes.data, stride=h * w, P=poses, c=cam, md=inf, fr=frames.ctypes.data, fs=h * w, ww=w,
             hh=h, mk=0):
        cc = None if c is None else ctypes.byref(c)
        return L.ofdis_fuse_push(ctx._h, n, api._ptr(d), stride, None if P is None else api._ptr(P), cc, md,
                                 api._ptr(fr), fs, ww, hh, mk)

    def render(n=1, P=poses, c=cam, zn=0.5, zf=2.0, st=0.05, mw=1.0, out=np.empty((2, h, w), np.float32), ww=w, mk=0):
        cc = None if c is None else ctypes.byref(c)
        return L.ofdis_fuse_render(ctx._h, n, None if P is None else api._ptr(P), cc, zn, zf, st, mw, api._ptr(out),
                                   ww, h, mk)

    bad_cam = [api.StereoCamera(*[dict(CAM, **kv)[k] for k in preprocess.STEREO_CAMERA_FIELDS])
               for kv in (dict(fx=0.0), dict(fy=inf), dict(baseline=-1.0), dict(cx=nan), dict(doffs=inf))]
    badp = poses.copy()
    badp[1, 2, 3] = nan
    errs = [push(n=0), push(n=3), push(d=None), push(P=None), push(c=None), push(md=nan), push(md=0.0),
            push(stride=h * w - 1), push(fr=None), push(fs=h * w - 1), push(P=badp), push(ww=w + 64), push(ww=w - 16),
            push(d=2, mk=1)] + [push(c=c) for c in bad_cam]
    errs += [render(n=0), render(n=3), render(P=None), render(c=None), render(out=None), render(zn=0.0),
             render(zn=nan), render(st=0.0), render(st=inf), render(zf=0.4), render(zf=inf), render(mw=nan),
             render(zf=32769.5, st=0.5), render(P=badp, n=2), render(ww=w - 16), render(out=2, mk=1)]
    errs += [L.ofdis_fuse_extract(ctx._h, 1.0, None, 0, None, 0), L.ofdis_fuse_extract(ctx._h, 1.0, None, -1,
                                                                                     ctypes.byref(count), 0),
             L.ofdis_fuse_extract(ctx._h, 1.0, None, 5, ctypes.byref(count), 0),
             L.ofdis_fuse_extract(ctx._h, nan, None, 0, ctypes.byref(count), 0),
             L.ofdis_fuse_extract(ctx._h, 1.0, api._ptr(2), 5, ctypes.byref(count), 1)]
    for kv in (dict(nx=0), dict(ny=-1), dict(nz=0), dict(nx=1024, ny=1024, nz=1025), dict(voxel=0.0),
               dict(voxel=nan), dict(trunc=-1.0), dict(trunc=inf), dict(max_weight=0.5), dict(max_weight=inf),
               dict(color=2)):
        q = api.FuseParams(*[kv.get(k, getattr(cp, k)) for k, _ in api.FuseParams._fields_])
        errs.append(L.ofdis_fuse_begin(ctx._h, ctypes.byref(q)))
    q = api.FuseParams(*[getattr(cp, k) for k, _ in api.FuseParams._fields_])
    q.origin[1] = inf
    errs.append(L.ofdis_fuse_begin(ctx._h, ctypes.byref(q)))
    errs.append(L.ofdis_fuse_begin(ctx._h, None))
    assert all(e == -1 for e in errs), errs  # OFDIS_ERR_ARG
    got = ctx.fuse_volume()
    for k in ("T", "W", "C"):
        same(got[k], vol[k], "after the errors: " + k)
    assert render(n=2, zf=32768.5, st=0.5) == 0 and push(n=2, fr=frames.ctypes.data, md=inf) == 0
    ctx.fuse_begin(vparams(color=0))
    assert L.ofdis_fuse_get_volume(ctx._h, None, None, api._ptr(np.empty(10, np.uint8)), 0) == -1
    ctx.close()


def test_disparities_of_a_stereo_context_on_the_same_stream(api):
    """A stereo context writes its filtered disparities to device memory and fuses them from there, on its stream."""
    import torch

    h, w, n = 96, 160, 3
    cam = dict(fx=180.0, fy=176.5, cx=w / 2 - 0.25, cy=h / 2 + 0.5, baseline=0.54, doffs=0.25)
    rels = [pose((0.0, 0.01, 0.0), (0.03, 0.0, -0.4)), pose((0.004, -0.006, 0.002), (0.0, 0.01, -0.3))]
    clip = synth.rigid_stereo_clip(n - 1, h, w, 1, 21, cam, rels)
    stream = torch.cuda.Stream()
    prm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=1, nop=1)
    ctx = context(api, prm, h, w, 2 * n, stream=stream.cuda_stream)
    fwd = np.stack([clip["left"], clip["right"]], 1)
    ctx.upload_frames_u8(0, 2 * n, np.ascontiguousarray(np.concatenate([fwd, fwd[:, ::-1]])), w, h)
    ctx.set_swapped_slots(n, 2 * n, 1)
    ctx.run(2 * n)
    d_disp = torch.full((n, h, w), 7.0, device="cuda")
    torch.cuda.synchronize()
    ctx.disparity_fullres(0, n, n, w, h, lr_check=1, outputs=("disp",), memkind=api.MEM_DEVICE,
                          out={"disp": d_disp.data_ptr()})
    p = dict(nx=60, ny=40, nz=70, origin=(-4.0, -2.0, 2.0), voxel=0.15, trunc=0.45, max_weight=64.0, color=1)
    ctx.fuse_begin(p)
    d_frames = torch.from_numpy(np.ascontiguousarray(clip["left"])).cuda()
    torch.cuda.synchronize()
    ctx.fuse_push(d_disp.data_ptr(), clip["abs"], cam, width_org=w, height_org=h, frames=d_frames.data_ptr(),
                  memkind=api.MEM_DEVICE)
    pts, total = ctx.fuse_extract(1.0)
    maps = d_disp.cpu().numpy()
    vol = preprocess.fuse_integrate(preprocess.fuse_new_volume(p), p, maps, clip["abs"], cam, frames=clip["left"])
    check_volume(ctx, vol, "stereo context")
    exp = preprocess.fuse_extract(vol, p, 1.0)
    assert total == len(exp) > 1000
    same(pts, exp, "stereo context points")
    ctx.close()


def test_quality_on_a_synthetic_rig_clip(api):
    """synth.rigid_stereo_clip at KITTI's size with a static box; disparities of a stereo context at operating point 2
    (lr-check), 8 frames fused with the true poses at 0.1 m."""
    h, w, n = 375, 1242, 8
    cam = dict(fx=721.5, fy=721.5, cx=609.6, cy=172.9, baseline=0.54, doffs=0.0)
    rels = [pose((0.0, math.radians(0.3 * (k % 3 - 1)), 0.0), (0.02 * (k % 2), 0.0, -0.5)) for k in range(n - 1)]
    clip = synth.rigid_stereo_clip(n - 1, h, w, 1, 2, cam, rels, block={"velocity": (0.0, 0.0, 0.0)})
    prm = params.operating_point(2, w, noc=1, nop=1)
    ctx = context(api, prm, h, w, 2 * n)
    fwd = np.stack([clip["left"], clip["right"]], 1)
    ctx.upload_frames_u8(0, 2 * n, np.ascontiguousarray(np.concatenate([fwd, fwd[:, ::-1]])), w, h)
    ctx.set_swapped_slots(n, 2 * n, 1)
    ctx.run(2 * n)
    disp = ctx.disparity_fullres(0, n, n, w, h, lr_check=1, outputs=("disp",))["disp"]
    p = dict(nx=160, ny=55, nz=280, origin=(-8.0, -3.0, 3.0), voxel=0.1, trunc=0.3, max_weight=64.0, color=0)
    ctx.fuse_begin(p)
    ctx.fuse_push(disp, clip["abs"], cam, width_org=w, height_org=h)
    depth = ctx.fuse_render(clip["abs"][:1], cam, z_near=3.0, z_far=30.0, step=0.05, width_org=w, height_org=h)[0]
    pts, total = ctx.fuse_extract(1.0)
    ctx.close()
    fb = np.float32(np.float32(cam["fx"]) * np.float32(cam["baseline"]))
    true = fb / (clip["disp"][0] + np.float32(cam["doffs"]))
    with np.errstate(invalid="ignore", divide="ignore"):
        raw = np.where((disp[0] >= 0) & (disp[0] <= 1e9), fb / disp[0], np.nan)
    both = np.isfinite(depth) & np.isfinite(raw)
    ground = pts[pts["ny"] < -0.9]
    figures = dict(render_median=float(np.median(np.abs(depth[both] - true[both]))),
                   raw_median=float(np.median(np.abs(raw[both] - true[both]))), pixels=int(both.sum()),
                   ground_points=int(len(ground)), ground_median=float(np.median(np.abs(ground["y"] - 1.65))),
                   points=int(total))
    print(json.dumps(figures))
    # bounds written before the first run: the fused depth beats a single frame's raw DIS depth, and the ground lies
    # within one voxel of y = 1.65 (median).  On an H100 the medians were 0.075 m fused against 0.088 m raw and the
    # ground 0.021 m.  Only a fifth of the pixels is compared: the wall at 40 m and the ground beyond 30 m lie outside
    # the volume (a first bound of 30 % of the frame did not allow for that).
    assert figures["pixels"] > 0.1 * h * w, figures
    assert figures["render_median"] < figures["raw_median"], figures
    assert figures["ground_points"] > 1000 and figures["ground_median"] < p["voxel"], figures


def test_batch_command_fuse(tmp_path):
    """A chained clip of three pairs and an unrelated pair (two clips) through run_OF_INT_batch --scene-flow --camera
    --odometry --fuse: each fused_<clip>.ply equals the restatement on the written poses, the disparities and frames."""
    import subprocess

    from of_dis_b200 import build

    bindir = build.build_host()
    h, w, n = 91, 150, 3
    cam = dict(fx=180.0, fy=176.5, cx=w / 2 - 0.25, cy=h / 2 + 0.5, baseline=0.54, doffs=0.25)
    rels = [pose((0.0, 0.01, 0.0), (0.03, 0.0, -0.5)), pose((0.004, -0.006, 0.002), (0.0, 0.01, -0.3)),
            pose((0.0, 0.0, 0.0), (0.05, 0.0, -0.6))]
    clip = synth.rigid_stereo_clip(n, h, w, 1, 31, cam, rels)
    rng = np.random.default_rng(31)
    maps = clip["disp"].copy()
    maps[rng.random(maps.shape) < 0.03] = np.nan
    for k in range(n + 1):
        preprocess.write_pgm(str(tmp_path / ("f%d.pgm" % k)), clip["left"][k])
        preprocess.write_pfm(str(tmp_path / ("d%d.pfm" % k)), -maps[k])
    pairs = [(k, k + 1) for k in range(n)] + [(2, 0)]
    (tmp_path / "list.txt").write_text("".join("f%d.pgm f%d.pgm out%d.flo\n" % (a, b, j)
                                               for j, (a, b) in enumerate(pairs)))
    (tmp_path / "disps.txt").write_text("".join("d%d.pfm d%d.pfm\n" % ab for ab in pairs))
    (tmp_path / "odo").mkdir()
    camarg = ",".join(repr(float(cam[k])) for k in preprocess.STEREO_CAMERA_FIELDS)
    spec = "0.25,0.75,-6,-3,2,48,20,80"
    r = subprocess.run([str(bindir) + "/run_OF_INT_batch", "list.txt", "--batch", "2", "--scene-flow", "disps.txt",
                        "--camera", camarg, "--odometry", "odo", "--fuse", spec], capture_output=True, text=True,
                       cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
    p = dict(nx=48, ny=20, nz=80, origin=(-6.0, -3.0, 2.0), voxel=0.25, trunc=0.75, max_weight=64.0, color=1)
    lines = [ln.split() for ln in r.stdout.splitlines() if ln.startswith("FUSE")]
    for c, frames in ((0, [0, 1, 2, 3]), (1, [2, 0])):
        poses = preprocess.read_kitti_poses(str(tmp_path / "odo" / ("poses_%04d.txt" % c)))
        assert poses.shape == (len(frames), 3, 4)
        d = np.stack([-preprocess.read_pfm(str(tmp_path / ("d%d.pfm" % k)))[..., 0] for k in frames])
        vol = preprocess.fuse_integrate(preprocess.fuse_new_volume(p), p, d, poses, cam, max_depth=np.inf,
                                        frames=clip["left"][frames])
        pts = preprocess.fuse_extract(vol, p, 1.0)
        assert len(pts) > 100
        exp = tmp_path / ("exp%d.ply" % c)
        preprocess.write_fused_ply(str(exp), pts)
        assert (tmp_path / "odo" / ("fused_%04d.ply" % c)).read_bytes() == exp.read_bytes(), c
        assert lines[c] == ["FUSE", "clip", str(c), "frames", str(len(frames)), "points", str(len(pts))], lines
