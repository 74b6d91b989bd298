"""ofdis_fuse_track: the poses (float64 bits), the stats and the whole volume after the call must equal
preprocess.fuse_track bit for bit (gray and RGB, colour on and off, host and device memory, volumes beside and behind
the camera, planted disparities and planted T and W, n = 1 and max_frames + 1, damping 0 and above); the call's two
properties on the device, every argument error with the volume and outputs unchanged, the launch count, a stereo
context's own disparities, and the quality on synth.rigid_stereo_clip."""
import ctypes
import json
import math

import numpy as np
import pytest

from of_dis_b200 import params, preprocess, synth

pytestmark = pytest.mark.gpu

f32 = np.float32
SMALL = "3 %d 8 8 0.05 0.95 0 8 0.4 %d 1 0 1 10 10 5 1 3 1.6 0"
CAM = dict(fx=40.0, fy=38.5, cx=15.25, cy=11.5, baseline=0.5, doffs=0.25)
TP = dict(step=1, rounds=6, min_weight=1.0, max_depth=float("inf"), huber=0.3, damping=0.0, min_corr=6,
          max_shift=0.5, min_cos=0.99, eps=0.0, integrate=1)


@pytest.fixture(scope="module")
def api():
    from of_dis_b200 import api as _api

    _api.lib()
    return _api


def context(api, prm, h, w, max_frames, stream=None):
    scf = 1 << prm.sc_f
    W, H = (w + scf - 1) // scf * scf, (h + scf - 1) // scf * scf
    return api.Context(prm, W, H, prm.p_samp_s, max_frames, stream=stream)


def pose(w=(0, 0, 0), t=(0, 0, 0)):
    return np.concatenate([synth.axis_angle(np.asarray(w, np.float64)), np.asarray(t, np.float64).reshape(3, 1)], 1)


def vparams(**kw):
    # 37 x 23 x 41: x from -1.9 puts part of it beside the frustum, z from -0.35 its first slices behind the camera
    # (which stays within a few cm of z = 0.03), so the push's Zc <= 0 skip runs inside a tracking call
    p = dict(nx=37, ny=23, nz=41, origin=(-1.9, -0.9, -0.35), voxel=0.07, trunc=0.2, max_weight=6.0, color=1)
    p.update(kw)
    return p


def scene(seed, n, h, w, ch, p):
    """A wavy surface at about 1.3 m: its planted TSDF (W at and around min_weight, NaN and +-1 T), disparities of
    the surface seen from drifting poses with NaN, -0, +inf and 3e9, the true motions and frames."""
    rng = np.random.default_rng(seed)
    vol = preprocess.fuse_new_volume(p)
    nz, ny, nx = vol["T"].shape
    z = p["origin"][2] + np.arange(nz)[:, None, None] * p["voxel"]
    x = p["origin"][0] + np.arange(nx)[None, None, :] * p["voxel"]
    y = p["origin"][1] + np.arange(ny)[None, :, None] * p["voxel"]
    vol["T"][:] = np.clip((1.3 + 0.1 * np.sin(3 * x) + 0.05 * y - z) / p["trunc"], -1, 1).astype(f32)
    vol["W"][:] = rng.choice(np.array([1.0, 2.0, 3.0], f32), vol["W"].shape)
    for v, share in ((np.nan, 0.01), (1.0, 0.01), (-1.0, 0.01), (-0.0, 0.01)):
        vol["T"][rng.random(vol["T"].shape) < share] = v
    for v, share in ((0.0, 0.02), (np.nextafter(f32(1), f32(0)), 0.02), (np.nan, 0.01)):
        vol["W"][rng.random(vol["W"].shape) < share] = v
    if vol["C"] is not None:
        vol["C"][:] = rng.integers(0, 256, vol["C"].shape)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    disp = []
    for k in range(n):
        Z = 1.3 + 0.02 * np.sin(xx / 5.0 + k) + 0.003 * yy + rng.uniform(-0.01, 0.01, (h, w))
        d = (f32(CAM["fx"]) * f32(CAM["baseline"]) / Z - CAM["doffs"]).astype(f32)
        for v, share in ((np.nan, 0.05), (-0.0, 0.03), (np.inf, 0.02), (3e9, 0.02)):
            d[rng.random((h, w)) < share] = v
        disp.append(d)
    motions = np.stack([pose(rng.uniform(-0.005, 0.005, 3), rng.uniform(-0.02, 0.02, 3)) for _ in range(n)])
    frames = rng.integers(0, 256, (n, h, w, ch) if ch == 3 else (n, h, w)).astype(np.uint8)
    return vol, np.stack(disp), motions, frames


def same(a, b, what):
    if a is None and b is None:
        return
    ab, bb = np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8)
    assert ab.shape == bb.shape and (ab == bb).all(), "%s differs" % what


def canon(a):
    # a NaN planted in T keeps its payload on the host but leaves a push as the device's NaN: compare NaN as NaN
    return np.where(np.isnan(a), f32(np.nan), a) if a is not None and a.dtype == f32 else a


def check(ctx, got, vol, exp, what):
    same(got[0], exp[0], what + " poses")
    for k in preprocess.FUSE_TRACK_STATS_DTYPE.names:
        same(got[1][k], exp[1][k], what + " stats " + k)
    v = ctx.fuse_volume()
    for k in ("T", "W", "C"):
        same(canon(v[k]), canon(vol[k]), "%s volume %s" % (what, k))


def load(ctx, p, vol):
    ctx.fuse_begin(p)
    ctx.fuse_set_volume(vol["T"], vol["W"], vol["C"])


@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("ch,color", [(1, 0), (1, 1), (3, 0), (3, 1)])
def test_device_equals_the_restatement(ch, color, mem, api):
    import torch

    h, w, mf = 45, 61, 4
    prm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=ch, nop=2)
    ctx = context(api, prm, h, w, mf)
    p = vparams(color=color)
    for case, (n, damping, step, motions_on, integrate) in enumerate(((1, 0.0, 1, True, 1), (mf + 1, 0.5, 3, True, 1),
                                                                      (mf + 1, 0.0, 2, False, 0))):
        vol, disp, motions, frames = scene(100 * ch + 10 * color + case, n, h, w, ch, p)
        tp = dict(TP, damping=damping, step=step, integrate=integrate, max_depth=1.33 if case == 2 else np.inf)
        prev = pose((0.01, -0.02, 0.005), (0.02, -0.01, 0.03))
        mot = motions if motions_on else None
        fr = frames if color and integrate else None
        load(ctx, p, vol)
        if mem == "host":
            got = ctx.fuse_track(disp, mot, prev, CAM, tp, width_org=w, height_org=h, frames=fr)
        else:
            dd, df = torch.from_numpy(disp).cuda(), torch.from_numpy(frames).cuda()
            got = ctx.fuse_track(dd.data_ptr(), mot, prev, CAM, tp, width_org=w, height_org=h, n=n,
                                 frames=df.data_ptr() if fr is not None else None, memkind=api.MEM_DEVICE)
        exp = preprocess.fuse_track(vol, p, tp, disp, mot, prev, CAM, fr)
        check(ctx, got, vol, exp, "case %d" % case)
        assert (exp[1]["rounds"] > 0).any(), exp[1]
    ctx.close()


def test_properties_on_the_device(api):
    h, w, n = 45, 61, 4
    prm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=3, nop=2)
    ctx = context(api, prm, h, w, n)
    p = vparams()
    vol, disp, motions, frames = scene(7, n, h, w, 3, p)
    prev = pose((0.01, 0.0, 0.0), (0.02, 0.0, 0.0))
    load(ctx, p, vol)
    whole = ctx.fuse_track(disp, motions, prev, CAM, TP, width_org=w, height_org=h, frames=frames)
    vw = ctx.fuse_volume()
    load(ctx, p, vol)
    P = prev
    for k in range(n):
        pk, sk = ctx.fuse_track(disp[k:k + 1], motions[k:k + 1], P, CAM, TP, width_org=w, height_org=h,
                                frames=frames[k:k + 1])
        same(pk[0], whole[0][k], "one of n: pose %d" % k)
        same(sk, whole[1][k:k + 1], "one of n: stats %d" % k)
        P = pk[0]
    v1 = ctx.fuse_volume()
    load(ctx, p, vol)
    P = prev
    for k in range(n):
        pk, sk = ctx.fuse_track(disp[k:k + 1], motions[k:k + 1], P, CAM, dict(TP, integrate=0), width_org=w,
                                height_org=h)
        same(pk[0], whole[0][k], "align then push: pose %d" % k)
        ctx.fuse_push(disp[k:k + 1], pk, CAM, width_org=w, height_org=h, frames=frames[k:k + 1])
        P = pk[0]
    v2 = ctx.fuse_volume()
    for k in ("T", "W", "C"):
        same(v1[k], vw[k], "one of n: volume " + k)
        same(v2[k], vw[k], "align then push: volume " + k)
    exp = preprocess.fuse_track(vol, p, TP, disp, motions, prev, CAM, frames)
    check(ctx, whole, vol, exp, "whole")
    ctx.close()


def test_argument_errors_leave_the_volume_and_outputs(api):
    h, w, n = 45, 61, 2
    prm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=1, nop=2)
    ctx = context(api, prm, h, w, 1)
    L = api.lib()
    nan, inf = float("nan"), float("inf")
    p = vparams()
    vol, disp, motions, frames = scene(4, n, h, w, 1, p)
    prev = pose()
    cam = api.StereoCamera(*[CAM[k] for k in preprocess.STEREO_CAMERA_FIELDS])
    poses = np.full((n, 12), 7.0)
    stats = (api.FuseTrackStats * n)()

    def call(n=n, d=disp, stride=h * w, M=motions, P=prev, c=cam, tp=TP, fr=frames, fs=h * w, out=poses, st=stats,
             ww=w, mk=0):
        q = None if tp is None else ctypes.byref(api.FuseTrackParams(*[tp[k] for k in preprocess.FUSE_TRACK_PARAM_FIELDS]))
        return L.ofdis_fuse_track(ctx._h, n, api._ptr(d), stride, api._ptr(M), api._ptr(P),
                                  None if c is None else ctypes.byref(c), q, api._ptr(fr), fs, api._ptr(out), st,
                                  ww, h, mk)

    assert call() == -1, "no live volume"
    load(ctx, p, vol)
    before = ctx.fuse_volume()
    bad_cam = [api.StereoCamera(*[dict(CAM, **kv)[k] for k in preprocess.STEREO_CAMERA_FIELDS])
               for kv in (dict(fx=0.0), dict(fy=inf), dict(baseline=-1.0), dict(cx=nan), dict(doffs=inf))]
    badm, badp = motions.copy(), prev.copy()
    badm[1, 2, 3], badp[0, 1] = nan, inf
    errs = [call(n=0), call(n=3), call(d=None), call(P=None), call(c=None), call(tp=None), call(out=None),
            call(st=None), call(stride=h * w - 1), call(fr=None), call(fs=h * w - 1), call(M=badm), call(P=badp),
            call(ww=w + 64), call(ww=w - 16), call(d=2, mk=1)] + [call(c=c) for c in bad_cam]
    for kv in (dict(step=0), dict(rounds=-1), dict(rounds=33), dict(min_weight=nan), dict(max_depth=0.0),
               dict(max_depth=nan), dict(huber=0.0), dict(huber=inf), dict(damping=-1.0), dict(damping=inf),
               dict(min_corr=5), dict(max_shift=0.0), dict(max_shift=inf), dict(min_cos=1.5), dict(min_cos=nan),
               dict(eps=-1.0), dict(eps=nan), dict(integrate=2)):
        errs.append(call(tp=dict(TP, **kv)))
    assert all(e == -1 for e in errs), errs  # OFDIS_ERR_ARG
    after = ctx.fuse_volume()
    for k in ("T", "W", "C"):
        same(after[k], before[k], "after the errors: " + k)
    assert (poses == 7.0).all() and all(s.status == 0 and s.cost == 0.0 for s in stats)
    assert call(fr=None, tp=dict(TP, integrate=0)) == 0
    assert call(M=None) == 0
    ctx.close()


def test_launch_counts(api):
    h, w, mf = 45, 61, 4
    prm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=1, nop=2)
    ctx = context(api, prm, h, w, mf)
    p = vparams(color=0)
    vol, disp, motions, _ = scene(5, mf + 1, h, w, 1, p)
    load(ctx, p, vol)
    counts, exp = {}, {}
    for n, rounds, integrate, eps in ((1, 0, 0, 0.0), (1, 5, 1, 0.0), (mf + 1, 3, 1, 1e9), (mf + 1, 32, 0, 1e-3)):
        before = ctx.launch_count
        _, st = ctx.fuse_track(disp[:n], motions[:n], pose(), CAM, dict(TP, rounds=rounds, integrate=integrate,
                                                                        eps=eps), width_org=w, height_org=h)
        key = "n%d r%d i%d" % (n, rounds, integrate)
        counts[key], exp[key] = ctx.launch_count - before, n * (rounds + 1) + n * integrate
        if eps == 1e9:
            assert (st["rounds"] == 0).all(), st  # every frame stopped at its first evaluation, every launch counted
    assert counts == exp, counts
    ctx.close()


def stereo_disparities(api, clip, cam, h, w, n, prm, device=False):
    ctx = context(api, prm, h, w, 2 * n)
    fwd = np.stack([clip["left"], clip["right"]], 1)
    ctx.upload_frames_u8(0, 2 * n, np.ascontiguousarray(np.concatenate([fwd, fwd[:, ::-1]])), w, h)
    ctx.set_swapped_slots(n, 2 * n, 1)
    ctx.run(2 * n)
    return ctx


def test_disparities_of_a_stereo_context(api):
    """A stereo context writes its filtered disparities to device memory and tracks against a volume fused from them."""
    import torch

    h, w, n = 96, 160, 3
    cam = dict(fx=180.0, fy=176.5, cx=w / 2 - 0.25, cy=h / 2 + 0.5, baseline=0.54, doffs=0.25)
    rels = [pose((0.0, 0.01, 0.0), (0.03, 0.0, -0.4)), pose((0.004, -0.006, 0.002), (0.0, 0.01, -0.3))]
    clip = synth.rigid_stereo_clip(n - 1, h, w, 1, 21, cam, rels)
    prm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=1, nop=1)
    ctx = stereo_disparities(api, clip, cam, h, w, n, prm)
    d_disp = torch.full((n, h, w), 7.0, device="cuda")
    torch.cuda.synchronize()
    ctx.disparity_fullres(0, n, n, w, h, lr_check=1, outputs=("disp",), memkind=api.MEM_DEVICE,
                          out={"disp": d_disp.data_ptr()})
    p = dict(nx=60, ny=40, nz=70, origin=(-4.0, -2.0, 2.0), voxel=0.15, trunc=0.45, max_weight=64.0, color=1)
    ctx.fuse_begin(p)
    d_frames = torch.from_numpy(np.ascontiguousarray(clip["left"])).cuda()
    torch.cuda.synchronize()
    ctx.fuse_push(d_disp.data_ptr(), clip["abs"][:1], cam, width_org=w, height_org=h, frames=d_frames.data_ptr(),
                  memkind=api.MEM_DEVICE)
    rel = np.stack(rels)
    got = ctx.fuse_track(d_disp.data_ptr() + 4 * h * w, rel, clip["abs"][0], cam, dict(TP, huber=0.2), width_org=w,
                         height_org=h, n=n - 1, frames=d_frames.data_ptr() + h * w, memkind=api.MEM_DEVICE)
    maps = d_disp.cpu().numpy()
    vol = preprocess.fuse_integrate(preprocess.fuse_new_volume(p), p, maps[:1], clip["abs"][:1], cam,
                                    frames=clip["left"][:1])
    exp = preprocess.fuse_track(vol, p, dict(TP, huber=0.2), maps[1:], rel, clip["abs"][0], cam, clip["left"][1:])
    check(ctx, got, vol, exp, "stereo context")
    assert (exp[1]["n_corr"] > 1000).all(), exp[1]
    ctx.close()


KITTI = dict(fx=721.5, fy=721.5, cx=609.6, cy=172.9, baseline=0.54, doffs=0.0)
QP = dict(nx=160, ny=55, nz=280, origin=(-8.0, -3.0, 3.0), voxel=0.1, trunc=0.3, max_weight=64.0, color=0)
QT = dict(step=2, rounds=10, min_weight=1.0, max_depth=30.0, huber=0.2, damping=1.0, min_corr=100, max_shift=0.5,
          min_cos=math.cos(math.radians(5.0)), eps=1e-7, integrate=0)


def kitti_clip(api, n, seed):
    h, w = 375, 1242
    rels = [pose((0.0, math.radians(0.3 * (k % 3 - 1)), 0.0), (0.02 * (k % 2), 0.0, -0.5)) for k in range(n - 1)]
    clip = synth.rigid_stereo_clip(n - 1, h, w, 1, seed, KITTI, rels, block={"velocity": (0.0, 0.0, 0.0)})
    prm = params.operating_point(2, w, noc=1, nop=1)
    ctx = stereo_disparities(api, clip, KITTI, h, w, n, prm)
    disp = ctx.disparity_fullres(0, n, n, w, h, lr_check=1, outputs=("disp",))["disp"]
    return ctx, clip, disp, np.stack(rels), h, w


@pytest.mark.xfail(strict=True, reason="the operating-point-2 stereo disparities' errors, in the fused model and in the "
                   "tracked frame, keep the alignment off the bound; with exact disparities it is met (DESIGN 5.26)")
def test_quality_relocalisation_and_drift(api):
    """Bounds written before the first run.  Re-localisation: 8 frames fused at their true poses, frame 8 aligned from
    its true pose perturbed by 0.15 m and 1 degree falls to <= 25 % of both.  Drift: 16 frames whose true relative
    motions carry a systematic bias (translation x 1.05, 0.1 degree of yaw per pair), tracked with integration: the last
    frame's translation error is at most half that of the chained poses, and the depth rendered at frame 0 is no worse
    than with the chained poses (median)."""
    n = 16
    ctx, clip, disp, rels, h, w = kitti_clip(api, n, 2)
    G = clip["abs"]
    figures = {}
    # re-localisation
    ctx.fuse_begin(QP)
    ctx.fuse_push(disp[:8], G[:8], KITTI, width_org=w, height_org=h)
    rng = np.random.default_rng(11)
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    tdir = rng.normal(size=3)
    tdir /= np.linalg.norm(tdir)
    start = np.concatenate([synth.axis_angle(axis * math.radians(1.0)) @ G[8][:, :3], (G[8][:, 3] + 0.15 * tdir)[:, None]], 1)
    got, st = ctx.fuse_track(disp[8:9], None, start, KITTI, QT, width_org=w, height_org=h)
    t_err, r_err = preprocess.trajectory_errors(got, G[8:9])
    figures["reloc"] = dict(t=float(t_err[0]), r=float(r_err[0]), status=int(st[0]["status"]),
                            rounds=int(st[0]["rounds"]), n_corr=int(st[0]["n_corr"]))
    # drift
    biased = []
    for k in range(n - 1):
        R, t = rels[k][:, :3], rels[k][:, 3] * 1.05
        biased.append(np.concatenate([synth.axis_angle((0.0, math.radians(0.1), 0.0)) @ R, t[:, None]], 1))
    biased = np.stack(biased)
    chained = preprocess.chain_poses(biased)
    ctx.fuse_begin(QP)
    ctx.fuse_push(disp[:1], G[:1], KITTI, width_org=w, height_org=h)
    tracked, st = ctx.fuse_track(disp[1:], biased, G[0], KITTI, dict(QT, integrate=1), width_org=w, height_org=h)
    tracked = np.concatenate([G[:1], tracked])
    fb = f32(f32(KITTI["fx"]) * f32(KITTI["baseline"]))
    true = fb / (clip["disp"][0] + f32(KITTI["doffs"]))
    depth_t = ctx.fuse_render(G[:1], KITTI, z_near=3.0, z_far=30.0, step=0.05, width_org=w, height_org=h)[0]
    ctx.fuse_begin(QP)
    ctx.fuse_push(disp, chained, KITTI, width_org=w, height_org=h)
    depth_c = ctx.fuse_render(G[:1], KITTI, z_near=3.0, z_far=30.0, step=0.05, width_org=w, height_org=h)[0]
    ctx.close()
    tt, rt = preprocess.trajectory_errors(tracked, G)
    tc, rc = preprocess.trajectory_errors(chained, G)
    both = np.isfinite(depth_t) & np.isfinite(depth_c)
    figures["drift"] = dict(t_tracked=float(tt[-1]), t_chained=float(tc[-1]), r_tracked=float(rt[-1]),
                            r_chained=float(rc[-1]), statuses=st["status"].tolist(), rounds=st["rounds"].tolist(),
                            depth_tracked=float(np.median(np.abs(depth_t[both] - true[both]))),
                            depth_chained=float(np.median(np.abs(depth_c[both] - true[both]))),
                            pixels=int(both.sum()))
    print(json.dumps(figures))
    assert figures["reloc"]["t"] <= 0.25 * 0.15 and figures["reloc"]["r"] <= 0.25 * 1.0, figures
    assert figures["drift"]["t_tracked"] <= 0.5 * figures["drift"]["t_chained"], figures
    assert figures["drift"]["depth_tracked"] <= figures["drift"]["depth_chained"], figures


@pytest.mark.xfail(strict=True, reason="the operating-point-2 stereo disparities' errors, in the fused model and in the "
                   "tracked frame, keep the alignment off the bound; with exact disparities it is met (DESIGN 5.26)")
def test_quality_end_to_end(api):
    """DIS flows -> egomotion_fullres -> fuse_track against the chained poses: reported, and tracking may be no worse
    than chaining by more than 10 % (last frame's translation error)."""
    n = 8
    h, w = 375, 1242
    rels = [pose((0.0, math.radians(0.3 * (k % 3 - 1)), 0.0), (0.02 * (k % 2), 0.0, -0.5)) for k in range(n - 1)]
    clip = synth.rigid_stereo_clip(n - 1, h, w, 1, 3, KITTI, rels, block={"velocity": (0.0, 0.0, 0.0)})
    sp = params.operating_point(2, w, noc=1, nop=1)
    sctx = stereo_disparities(api, clip, KITTI, h, w, n, sp)
    disp = sctx.disparity_fullres(0, n, n, w, h, lr_check=1, outputs=("disp",))["disp"]
    sctx.close()
    fp = params.operating_point(2, w, noc=1, nop=2)
    fctx = context(api, fp, h, w, n - 1)
    fctx.upload_sequence_u8(0, n - 1, np.ascontiguousarray(clip["left"]), w, h)
    fctx.run(n - 1)
    ep = dict(step=4, fb_check=0, alpha=0.01, beta=0.5, edge_diff=1.0, hypotheses=256, threshold=1.0, refine=5, seed=1)
    ego, est = fctx.egomotion_fullres(0, n - 1, disp[:-1], disp[1:], ep, camera=KITTI, width_org=w, height_org=h)[:2]
    chained = preprocess.chain_poses(ego)
    fctx.fuse_begin(QP)
    fctx.fuse_push(disp[:1], chained[:1], KITTI, width_org=w, height_org=h)
    tracked, st = fctx.fuse_track(disp[1:], ego, chained[0], KITTI, dict(QT, integrate=1), width_org=w, height_org=h)
    fctx.close()
    tracked = np.concatenate([chained[:1], tracked])
    tt, rt = preprocess.trajectory_errors(tracked, clip["abs"])
    tc, rc = preprocess.trajectory_errors(chained, clip["abs"])
    figures = dict(t_tracked=tt.tolist(), t_chained=tc.tolist(), r_tracked=rt.tolist(), r_chained=rc.tolist(),
                   statuses=st["status"].tolist(), ego_status=est["status"].tolist())
    print(json.dumps(figures))
    assert tt[-1] <= 1.1 * tc[-1] + 1e-3, figures
