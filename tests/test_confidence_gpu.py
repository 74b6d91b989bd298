"""ofdis_confidence_fullres: conf and terms equal preprocess.confidence bit for bit (gray and RGB, flow and stereo,
usefbcon 0 and 1, divisible and odd sizes, r = 1, 2 and 7, with and without the partner slots, the two-way upload with
its swapped slots, host and device outputs on a caller stream in graph mode, planted level flows with NaN, +-inf and
huge values); e equals ofdis_consistency_fullres's err; the launch count does not depend on n; argument errors leave the
outputs untouched.  ofdis_fuse_push_weighted and ofdis_fuse_track_weighted: all-ones weights give the unweighted
volume, poses and stats bit for bit, other weights the restatement, with the unweighted launch counts.  Quality: the
sparsification curve of conf on synth.layered_stereo and the KITTI-sized clip, and the weighted re-localisation."""
import ctypes
import json
import math

import numpy as np
import pytest

from of_dis_b200 import params, preprocess, synth

pytestmark = pytest.mark.gpu

f32 = np.float32
SMALL = "3 1 8 8 0.05 0.95 0 8 0.4 %d 1 0 1 10 10 5 1 3 1.6 0"
CP = dict(radius=2, s_fb=1.0, s_tex=100.0, min_count=5)


@pytest.fixture(scope="module")
def api():
    from of_dis_b200 import api as _api

    _api.lib()
    return _api


def context(api, prm, h, w, max_frames, stream=None):
    scf = 1 << prm.sc_f
    W, H = (w + scf - 1) // scf * scf, (h + scf - 1) // scf * scf
    return api.Context(prm, W, H, prm.p_samp_s, max_frames, stream=stream)


def bits_equal(got, exp, what):
    g, e = np.ascontiguousarray(got, f32).view(np.uint32), np.ascontiguousarray(exp, f32).view(np.uint32)
    assert g.shape == e.shape, (what, g.shape, e.shape)
    bad = g != e
    assert not bad.any(), "%s: %d of %d values differ, first at %s" % (what, int(bad.sum()), bad.size,
                                                                      np.argwhere(bad)[0].tolist())


def full(ctx, f0, f1, h, w, nop):
    out = np.empty((f1 - f0, h, w, nop), f32)
    ctx.get_flow_fullres(f0, f1, out, w, h)
    ctx.sync()
    return out


def bidir(api, nop, ch, fb, h, w, n, seed):
    """A context holding the two-way upload of an n+1-frame clip: slot k (frames k, k+1), slot n+k swapped."""
    prm = params.from_cli_numbers((SMALL % fb).split(), noc=ch, nop=nop)
    frames = synth.synthetic_sequence(n + 1, h, w, ch, seed=seed, amp=3.0, stereo=(nop == 1))
    ctx = context(api, prm, h, w, 2 * n)
    ctx.upload_sequence_bidir_u8(0, n, frames, w, h)
    ctx.run(2 * n)
    return ctx, prm, frames


def expected(frames0, frames1, F, B, p):
    out = [preprocess.confidence(frames0[k], frames1[k], F[k], None if B is None else B[k], p) for k in range(len(F))]
    return np.stack([c for c, _ in out]), np.stack([t for _, t in out])


@pytest.mark.parametrize("fb", [0, 1])
@pytest.mark.parametrize("nop,ch", [(2, 1), (2, 3), (1, 1), (1, 3)])
def test_device_equals_the_restatement(nop, ch, fb, api):
    h, w, n = 45, 77, 3  # the padding's crop and partial tiles on both axes
    ctx, prm, frames = bidir(api, nop, ch, fb, h, w, n, 10 * nop + ch + fb)
    F = full(ctx, 0, 2 * n, h, w, nop)
    for r in (1, 2, 7):
        p = dict(CP, radius=r, min_count=min(CP["min_count"], (2 * r + 1) ** 2))
        # forward slots against their backward partners, the swapped slots against the forward ones, and no partner
        for f0, b0, i0, i1 in ((0, n, frames[:-1], frames[1:]), (n, 0, frames[1:], frames[:-1]),
                               (0, -1, frames[:-1], frames[1:])):
            conf, terms = ctx.confidence_fullres(f0, f0 + n, b0, i0, i1, p, w, h, with_terms=True)
            ec, et = expected(i0, i1, F[f0:f0 + n], None if b0 < 0 else F[b0:b0 + n], p)
            what = "r%d f0 %d b0 %d" % (r, f0, b0)
            bits_equal(conf, ec, what + " conf")
            bits_equal(terms, et, what + " terms")
            assert (conf > 0).mean() > 0.2, what
    # e is ofdis_consistency_fullres's err, bit for bit
    _, terms = ctx.confidence_fullres(0, n, n, frames[:-1], frames[1:], CP, w, h, with_conf=False, with_terms=True)
    _, err = ctx.consistency_fullres(0, n, n, w, h, with_err=True)
    bits_equal(terms[..., 1], err, "e against consistency err")
    ctx.close()


def test_stereo_pairs_and_planted_level_flows(api):
    """upload_frames_u8 pairs of a stereo context, both slots' level flows planted with NaN, +-inf, -0 and 3e9."""
    h, w, n = 64, 96, 2
    prm = params.from_cli_numbers((SMALL % 0).split(), noc=1, nop=1)
    left, right, gt, _ = synth.layered_stereo(h, w, 1, seed=3)
    pairs = np.stack([np.stack([left, right]), np.stack([right, left])])
    ctx = context(api, prm, h, w, 2 * n)
    ctx.upload_frames_u8(0, n, np.ascontiguousarray(pairs), w, h)
    ctx.set_swapped_slots(1, 2, 1)
    ctx.run(n)
    rng = np.random.default_rng(5)
    for slot in (0, 1):
        lv = ctx.get_flow(slot, prm.sc_l)
        for v, share in ((np.nan, 0.05), (np.inf, 0.03), (-np.inf, 0.03), (-0.0, 0.05), (3e9, 0.03), (-3e9, 0.03)):
            lv[rng.random(lv.shape) < share] = v
        ctx.set_flow(slot, prm.sc_l, lv)
    F = full(ctx, 0, n, h, w, 1)
    i0, i1 = pairs[:, 0], pairs[:, 1]
    for b0 in (1, -1):
        conf, terms = ctx.confidence_fullres(0, 1, b0, i0[:1], i1[:1], CP, w, h, with_terms=True)
        ec, et = expected(i0[:1], i1[:1], F[:1], None if b0 < 0 else F[1:2], CP)
        bits_equal(conf, ec, "planted conf b0 %d" % b0)
        # a NaN partner flow makes e a NaN of arithmetic, whose payload the device and numpy choose differently
        bits_equal(np.where(np.isnan(terms), f32(np.nan), terms), np.where(np.isnan(et), f32(np.nan), et),
                   "planted terms b0 %d" % b0)
        assert b0 < 0 or np.isinf(terms[..., 1]).any()
    ctx.close()


def test_outputs_on_a_caller_stream_in_graph_mode(api):
    """Device and host outputs of a context on a caller's stream with graph mode on."""
    import torch

    h, w, n = 40, 56, 2
    stream = torch.cuda.Stream()
    prm = params.from_cli_numbers((SMALL % 1).split(), noc=3, nop=2)
    frames = synth.synthetic_sequence(n + 1, h, w, 3, seed=8, amp=3.0)
    ctx = context(api, prm, h, w, 2 * n, stream=stream.cuda_stream)
    ctx.set_graph_mode(True)
    ctx.upload_sequence_bidir_u8(0, n, frames, w, h)
    ctx.run(2 * n)
    F = full(ctx, 0, 2 * n, h, w, 2)
    d_frames = torch.from_numpy(frames).cuda()
    conf = torch.full((n, h, w), 7.0, device="cuda")
    terms = torch.full((n, h, w, 3), 7.0, device="cuda")
    torch.cuda.synchronize()
    hwc = h * w * 3
    ctx.confidence_fullres(0, n, n, d_frames.data_ptr(), d_frames.data_ptr() + hwc, CP, w, h, with_terms=True,
                           memkind=api.MEM_DEVICE, conf=conf.data_ptr(), terms=terms.data_ptr(), frame_stride=hwc)
    stream.synchronize()
    ec, et = expected(frames[:-1], frames[1:], F[:n], F[n:], CP)
    bits_equal(conf.cpu().numpy(), ec, "device conf")
    bits_equal(terms.cpu().numpy(), et, "device terms")
    hc, ht = ctx.confidence_fullres(0, n, n, frames[:-1], frames[1:], CP, w, h, with_terms=True)
    bits_equal(hc, ec, "host conf")
    bits_equal(ht, et, "host terms")
    ctx.close()


def test_launch_count_and_argument_errors(api):
    h, w, n = 40, 56, 4
    ctx, prm, frames = bidir(api, 2, 1, 0, h, w, n, 4)
    for k in (1, n):
        before = ctx.launch_count
        ctx.confidence_fullres(0, k, n, frames[:k], frames[1:k + 1], CP, w, h)
        assert ctx.launch_count - before == 1, k
    L = api.lib()
    conf = np.full((n, h, w), 7.0, f32)
    terms = np.full((n, h, w, 3), 7.0, f32)

    def call(f0=0, f1=n, b0=n, p=CP, a=frames, b=frames[1:], fs=h * w, c=conf, t=terms, ww=w, mk=0):
        q = None if p is None else ctypes.byref(api.ConfParams(*[p[k] for k in preprocess.CONF_PARAM_FIELDS]))
        return L.ofdis_confidence_fullres(ctx._h, f0, f1, b0, q, api._ptr(a), api._ptr(b), fs, api._ptr(c),
                                          api._ptr(t), ww, h, mk)

    errs = [call(f0=-1), call(f1=2 * n + 1), call(f0=2, f1=2), call(b0=n + 1), call(p=None), call(a=None), call(b=None),
            call(fs=h * w - 1), call(c=None, t=None), call(ww=w + 64), call(ww=w - 16), call(c=2, mk=1),
            call(c=None, t=6, mk=1)]
    for kv in (dict(radius=0), dict(radius=8), dict(s_fb=0.0), dict(s_fb=float("inf")), dict(s_fb=float("nan")),
               dict(s_tex=-1.0), dict(s_tex=float("inf")), dict(min_count=0), dict(radius=1, min_count=10)):
        errs.append(call(p=dict(CP, **kv)))
    assert all(e == -1 for e in errs), errs  # OFDIS_ERR_ARG
    assert (conf == 7.0).all() and (terms == 7.0).all()
    assert call(b0=-1) == 0 and call(t=None) == 0 and call(c=None) == 0
    ctx.close()


# ---- weighted fusion and tracking ---------------------------------------------------------------------------------
CAM = dict(fx=40.0, fy=38.5, cx=15.25, cy=11.5, baseline=0.5, doffs=0.25)
TP = dict(step=1, rounds=6, min_weight=1.0, max_depth=float("inf"), huber=0.3, damping=0.0, min_corr=6,
          max_shift=0.5, min_cos=0.99, eps=0.0, integrate=1)
VP = dict(nx=37, ny=23, nz=41, origin=(-1.9, -0.9, -0.35), voxel=0.07, trunc=0.2, max_weight=6.0, color=1)


def pose(w=(0, 0, 0), t=(0, 0, 0)):
    return np.concatenate([synth.axis_angle(np.asarray(w, np.float64)), np.asarray(t, np.float64).reshape(3, 1)], 1)


def scene(seed, n, h, w, ch):
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
        d = (f32(CAM["fx"]) * f32(CAM["baseline"]) / Z - CAM["doffs"]).astype(f32)
        d[rng.random((h, w)) < 0.05] = np.nan
        disp.append(d)
    motions = np.stack([pose(rng.uniform(-0.005, 0.005, 3), rng.uniform(-0.02, 0.02, 3)) for _ in range(n)])
    frames = rng.integers(0, 256, (n, h, w, ch) if ch == 3 else (n, h, w)).astype(np.uint8)
    return vol, np.stack(disp), motions, frames


def special_weights(rng, shape):
    wts = rng.uniform(0.05, 2.0, shape).astype(f32)
    for v, share in ((0.0, 0.05), (-0.0, 0.05), (np.nan, 0.05), (-1.0, 0.05), (-np.inf, 0.01), (np.inf, 0.01),
                     (3e9, 0.02), (1e-30, 0.02)):
        wts[rng.random(shape) < share] = v
    return wts


def volume_equal(ctx, vol, what):
    v = ctx.fuse_volume()
    for k in ("T", "W", "C"):
        a, b = v[k], vol[k]
        if a is not None and a.dtype == f32:  # a NaN leaves the device as the device's NaN: compare NaN as NaN
            a, b = np.where(np.isnan(a), f32(np.nan), a), np.where(np.isnan(b), f32(np.nan), b)
        assert np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8)), \
            "%s: volume %s" % (what, k)


@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("ch", [1, 3])
def test_weighted_push_and_track(ch, mem, api):
    import torch

    h, w, n = 45, 61, 3
    prm = params.from_cli_numbers((SMALL % 0).split(), noc=ch, nop=2)
    ctx = context(api, prm, h, w, n)
    vol, disp, motions, frames = scene(ch, n, h, w, ch)
    poses = np.stack([pose((0.01 * k, 0, 0), (0.02 * k, 0, 0)) for k in range(n)])
    prev = pose((0.01, -0.02, 0.005), (0.02, -0.01, 0.03))
    rng = np.random.default_rng(ch)
    ones = np.ones(disp.shape, f32)

    def dev(a):
        t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
        torch.cuda.synchronize()
        return t

    def push(wts):
        if mem == "host":
            ctx.fuse_push(disp, poses, CAM, width_org=w, height_org=h, frames=frames, weights=wts)
        else:
            keep = [dev(disp), dev(frames)] + ([] if wts is None else [dev(wts)])
            ctx.fuse_push(keep[0].data_ptr(), poses, CAM, width_org=w, height_org=h, frames=keep[1].data_ptr(),
                          weights=None if wts is None else keep[2].data_ptr(), memkind=api.MEM_DEVICE)
            torch.cuda.synchronize()

    def track(wts):
        if mem == "host":
            return ctx.fuse_track(disp, motions, prev, CAM, TP, width_org=w, height_org=h, frames=frames, weights=wts)
        keep = [dev(disp), dev(frames)] + ([] if wts is None else [dev(wts)])
        return ctx.fuse_track(keep[0].data_ptr(), motions, prev, CAM, TP, width_org=w, height_org=h, n=n,
                              frames=keep[1].data_ptr(), weights=None if wts is None else keep[2].data_ptr(),
                              memkind=api.MEM_DEVICE)

    # all-ones weights: the unweighted push and track, bit for bit, with the same launches
    for name, call in (("push", push), ("track", track)):
        ctx.fuse_begin(VP)
        ctx.fuse_set_volume(vol["T"], vol["W"], vol["C"])
        before = ctx.launch_count
        a = call(None)
        launches = ctx.launch_count - before
        va = ctx.fuse_volume()
        ctx.fuse_set_volume(vol["T"], vol["W"], vol["C"])
        before = ctx.launch_count
        b = call(ones)
        assert ctx.launch_count - before == launches, name
        volume_equal(ctx, va, name + " ones")
        if name == "track":
            assert np.array_equal(a[0].view(np.uint64), b[0].view(np.uint64)) and \
                np.array_equal(a[1].view(np.uint8), b[1].view(np.uint8)), "track ones"
    # random and special weights: the restatement
    wts = special_weights(rng, disp.shape)
    exp = {k: (None if v is None else v.copy()) for k, v in vol.items()}
    preprocess.fuse_integrate(exp, VP, disp, poses, CAM, frames=frames, weights=wts)
    ctx.fuse_set_volume(vol["T"], vol["W"], vol["C"])
    push(wts)
    volume_equal(ctx, exp, "weighted push")
    exp = {k: (None if v is None else v.copy()) for k, v in vol.items()}
    ep, es = preprocess.fuse_track(exp, VP, TP, disp, motions, prev, CAM, frames, weights=wts)
    ctx.fuse_set_volume(vol["T"], vol["W"], vol["C"])
    gp, gs = track(wts)
    assert np.array_equal(gp.view(np.uint64), ep.view(np.uint64)), "weighted track poses"
    assert np.array_equal(gs.view(np.uint8), es.view(np.uint8)), "weighted track stats"
    volume_equal(ctx, exp, "weighted track")
    assert (es["rounds"] > 0).any()
    ctx.close()


def test_weighted_argument_errors_leave_the_volume(api):
    h, w, n = 45, 61, 2
    prm = params.from_cli_numbers((SMALL % 0).split(), noc=1, nop=2)
    ctx = context(api, prm, h, w, n)
    L = api.lib()
    vol, disp, motions, frames = scene(9, n, h, w, 1)
    wts = np.ones(disp.shape, f32)
    cam = ctypes.byref(api.StereoCamera(*[CAM[k] for k in preprocess.STEREO_CAMERA_FIELDS]))
    poses = np.stack([pose() for _ in range(n)])
    out = np.full((n, 12), 7.0)
    stats = (api.FuseTrackStats * n)()
    tp = ctypes.byref(api.FuseTrackParams(*[TP[k] for k in preprocess.FUSE_TRACK_PARAM_FIELDS]))

    def push(wt=wts, ws=h * w, mk=0):
        return L.ofdis_fuse_push_weighted(ctx._h, n, api._ptr(disp), h * w, api._ptr(poses), cam, float("inf"),
                                          api._ptr(frames), h * w, api._ptr(wt), ws, w, h, mk)

    def track(wt=wts, ws=h * w, mk=0):
        return L.ofdis_fuse_track_weighted(ctx._h, n, api._ptr(disp), h * w, api._ptr(motions), api._ptr(poses[0]),
                                           cam, tp, api._ptr(frames), h * w, api._ptr(wt), ws, api._ptr(out), stats, w,
                                           h, mk)

    assert push() == -1 and track() == -1, "no live volume"
    ctx.fuse_begin(VP)
    ctx.fuse_set_volume(vol["T"], vol["W"], vol["C"])
    errs = [push(wt=None), push(ws=h * w - 1), track(wt=None), track(ws=h * w - 1), push(wt=6, mk=1), track(wt=6, mk=1)]
    assert all(e == -1 for e in errs), errs
    volume_equal(ctx, vol, "after the errors")
    assert (out == 7.0).all()
    assert push() == 0 and track() == 0
    ctx.close()


# ---- quality --------------------------------------------------------------------------------------------------------
FRACTIONS = (1.0, 0.9, 0.8, 0.7, 0.6, 0.5, 0.4, 0.3)


def sparsification(err, score, rng=None):
    """Mean error of the most confident x % of the pixels for x in FRACTIONS: ranked by score (descending, ties in
    pixel order), or in a random order when score is None."""
    order = rng.permutation(err.size) if score is None else np.argsort(-score, kind="stable")
    e = err[order]
    return [float(e[:max(1, int(round(x * e.size)))].mean()) for x in FRACTIONS]


def stereo_quality(api, left, right, gt, h, w, prm):
    """conf, e and |d - gt| of a stereo context's left disparities over the pixels with known ground truth."""
    n = len(left)
    ctx = context(api, prm, h, w, 2 * n)
    fwd = np.stack([left, right], 1)
    ctx.upload_frames_u8(0, 2 * n, np.ascontiguousarray(np.concatenate([fwd, fwd[:, ::-1]])), w, h)
    ctx.set_swapped_slots(n, 2 * n, 1)
    ctx.run(2 * n)
    F = full(ctx, 0, n, h, w, 1)[..., 0]
    conf, terms = ctx.confidence_fullres(0, n, n, np.ascontiguousarray(left), np.ascontiguousarray(right), CP, w, h,
                                         with_terms=True)
    ctx.close()
    known = np.isfinite(gt) & (gt > 0)
    err = np.abs(-F - gt)[known]
    return err, conf[known], -terms[..., 1][known]


def curves(err, conf, neg_e):
    rng = np.random.default_rng(0)
    out = dict(conf=sparsification(err, conf), e=sparsification(err, neg_e), random=sparsification(err, None, rng))
    out["area"] = {k: float(np.trapezoid(v[::-1], FRACTIONS[::-1])) for k, v in out.items() if k != "area"}
    d1 = lambda s: [float((err[np.argsort(-s, kind="stable")][:int(round(x * err.size))] > 3.0).mean())
                    for x in FRACTIONS]
    out["d1_conf"], out["d1_e"] = d1(conf), d1(neg_e)
    return out


def test_quality_sparsification(api):
    """Bounds from the feature's statement, written before the first run: on synth.layered_stereo and on the
    KITTI-sized clip, conf's sparsification curve lies below the random order's at every fraction below 100 %, and
    its area is below that of e alone."""
    h, w = 120, 200
    left, right, gt, _ = synth.layered_stereo(h, w, 1, seed=7)
    figures = {"layered": curves(*stereo_quality(api, left[None], right[None], gt[None], h, w,
                                                 params.from_cli_numbers((SMALL % 0).split(), noc=1, nop=1)))}
    KITTI = dict(fx=721.5, fy=721.5, cx=609.6, cy=172.9, baseline=0.54, doffs=0.0)
    h, w, n = 375, 1242, 4
    rels = [pose((0.0, math.radians(0.3 * (k % 3 - 1)), 0.0), (0.02 * (k % 2), 0.0, -0.5)) for k in range(n - 1)]
    clip = synth.rigid_stereo_clip(n - 1, h, w, 1, 2, KITTI, rels, block={"velocity": (0.0, 0.0, 0.0)})
    figures["kitti"] = curves(*stereo_quality(api, clip["left"], clip["right"], clip["disp"], h, w,
                                              params.operating_point(2, w, noc=1, nop=1)))
    print(json.dumps(figures))
    for name, c in figures.items():
        assert all(a < b for a, b in zip(c["conf"][1:], c["random"][1:])), (name, c)
        assert c["area"]["conf"] < c["area"]["e"], (name, c["area"])


@pytest.mark.xfail(strict=True, reason="conf weighting brings the re-localisation from 0.219 m and 1.77 degrees to "
                   "0.18 m and 1.4 degrees, still off DESIGN 5.26's bound (DESIGN 5.27)")
def test_quality_weighted_relocalisation(api):
    """DESIGN 5.26's re-localisation with conf-weighted push and track, against its bounds unchanged: 8 frames of the
    KITTI-sized clip fused at their true poses, frame 8 aligned from its true pose perturbed by 0.15 m and 1 degree
    falls to <= 25 % of both.  The figures of a few radii and conf thresholds are printed beside the asserted one."""
    KITTI = dict(fx=721.5, fy=721.5, cx=609.6, cy=172.9, baseline=0.54, doffs=0.0)
    QP = dict(nx=160, ny=55, nz=280, origin=(-8.0, -3.0, 3.0), voxel=0.1, trunc=0.3, max_weight=64.0, color=0)
    QT = dict(step=2, rounds=10, min_weight=1.0, max_depth=30.0, huber=0.2, damping=1.0, min_corr=100,
              max_shift=0.5, min_cos=math.cos(math.radians(5.0)), eps=1e-7, integrate=0)
    h, w, n = 375, 1242, 9
    rels = [pose((0.0, math.radians(0.3 * (k % 3 - 1)), 0.0), (0.02 * (k % 2), 0.0, -0.5)) for k in range(n - 1)]
    clip = synth.rigid_stereo_clip(n - 1, h, w, 1, 2, KITTI, rels, block={"velocity": (0.0, 0.0, 0.0)})
    prm = params.operating_point(2, w, noc=1, nop=1)
    ctx = context(api, prm, h, w, 2 * n)
    fwd = np.stack([clip["left"], clip["right"]], 1)
    ctx.upload_frames_u8(0, 2 * n, np.ascontiguousarray(np.concatenate([fwd, fwd[:, ::-1]])), w, h)
    ctx.set_swapped_slots(n, 2 * n, 1)
    ctx.run(2 * n)
    disp = ctx.disparity_fullres(0, n, n, w, h, lr_check=1, outputs=("disp",))["disp"]
    G = clip["abs"]
    rng = np.random.default_rng(11)
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    tdir = rng.normal(size=3)
    tdir /= np.linalg.norm(tdir)
    start = np.concatenate([synth.axis_angle(axis * math.radians(1.0)) @ G[8][:, :3],
                            (G[8][:, 3] + 0.15 * tdir)[:, None]], 1)
    left, right = np.ascontiguousarray(clip["left"]), np.ascontiguousarray(clip["right"])
    figures = {}
    for r in (2, 4, 7):
        conf, _ = ctx.confidence_fullres(0, n, n, left, right, dict(CP, radius=r, min_count=(2 * r + 1) ** 2 // 2),
                                         w, h)
        for thr in (0.0, 0.1, 0.3):
            wts = np.where(conf > thr, conf, f32(0)).astype(f32)
            ctx.fuse_begin(dict(QP, max_weight=64.0))
            ctx.fuse_push(disp[:8], G[:8], KITTI, width_org=w, height_org=h, weights=wts[:8])
            got, st = ctx.fuse_track(disp[8:9], None, start, KITTI, dict(QT, min_weight=0.5), width_org=w,
                                     height_org=h, weights=wts[8:9])
            t_err, r_err = preprocess.trajectory_errors(got, G[8:9])
            figures["r%d thr%.1f" % (r, thr)] = dict(t=float(t_err[0]), r=float(r_err[0]),
                                                      status=int(st[0]["status"]), n_corr=int(st[0]["n_corr"]))
    ctx.close()
    print(json.dumps(figures))
    main = figures["r2 thr0.0"]
    assert main["t"] <= 0.25 * 0.15 and main["r"] <= 0.25 * 1.0, figures


@pytest.mark.parametrize("binary", ["run_OF_INT", "run_DE_INT"])
@pytest.mark.parametrize("extra", [[], ["--bidirectional"]], ids=["one-way", "two-way"])
def test_batch_command_confidence(binary, extra, tmp_path):
    """run_*_batch --confidence 2: every <stem>_conf.pfm equals preprocess.confidence (the restatement of
    Context.confidence_fullres) of the pair's frames and the flows the command wrote, the forward-backward term with
    --bidirectional; the CONF line is the maps' mean; every other file keeps its bytes."""
    import subprocess

    from of_dis_b200 import build

    bindir = build.build_host()
    h, w = 61, 90
    stereo = binary.startswith("run_DE")
    ext = ".pfm" if stereo else ".flo"
    if stereo:
        views = [synth.layered_stereo(h, w, 1, seed=s)[:2] for s in (1, 2)]
        for k, (l, r) in enumerate(views):
            preprocess.write_pgm(str(tmp_path / ("l%d.pgm" % k)), l)
            preprocess.write_pgm(str(tmp_path / ("r%d.pgm" % k)), r)
        pairs = [(views[k][0], views[k][1]) for k in range(2)]
        lines = ["l%d.pgm r%d.pgm out%d%s\n" % (k, k, k, ext) for k in range(2)]
    else:
        frames = synth.synthetic_sequence(3, h, w, 1, seed=4, amp=3.0)
        for k in range(3):
            preprocess.write_pgm(str(tmp_path / ("f%d.pgm" % k)), frames[k])
        pairs = [(frames[k], frames[k + 1]) for k in range(2)]
        lines = ["f%d.pgm f%d.pgm out%d%s\n" % (k, k + 1, k, ext) for k in range(2)]
    out = {}
    for name, flags in (("plain", []), ("conf", ["--confidence", "2"])):
        d = tmp_path / name
        d.mkdir()
        (d / "list.txt").write_text("".join(lines))
        for q in tmp_path.glob("*.pgm"):
            (d / q.name).write_bytes(q.read_bytes())
        r = subprocess.run([str(bindir) + "/" + binary + "_batch", "list.txt"] + extra + flags, capture_output=True,
                           text=True, cwd=str(d))
        assert r.returncode == 0, r.stderr
        out[name] = r.stdout
    plain, conf = tmp_path / "plain", tmp_path / "conf"
    made = sorted(q.name for q in conf.iterdir() if q.name.endswith("_conf.pfm"))
    assert made == ["out0_conf.pfm", "out1_conf.pfm"], made
    for q in plain.iterdir():
        assert (conf / q.name).read_bytes() == q.read_bytes(), q.name
    assert sorted(q.name for q in conf.iterdir()) == sorted([q.name for q in plain.iterdir()] + made)
    p = dict(radius=2, s_fb=1.0, s_tex=100.0, min_count=25 // 2)
    read = preprocess.read_pfm if stereo else preprocess.read_flo
    maps = []
    for k in range(2):
        F = read(str(conf / ("out%d%s" % (k, ext))))
        B = read(str(conf / ("out%d_bw%s" % (k, ext)))) if extra else None
        exp, _ = preprocess.confidence(pairs[k][0], pairs[k][1], F, B, p)
        got = -preprocess.read_pfm(str(conf / ("out%d_conf.pfm" % k)))[..., 0]
        bits_equal(got, exp, "pair %d" % k)
        maps.append(exp)
    line = [ln.split() for ln in out["conf"].splitlines() if ln.startswith("CONF")]
    mean = float(np.mean(np.stack(maps), dtype=np.float64))
    assert len(line) == 1 and line[0][:3] == ["CONF", "pairs", "2"] and abs(float(line[0][4]) - mean) <= 1e-7, line
    assert not any(ln.startswith("CONF") for ln in out["plain"].splitlines())


@pytest.mark.xfail(strict=True, reason="conf weighting brings the tracked drift from 0.88 m to 0.67 m, still above the "
                   "0.39 m of chaining (DESIGN 5.27)")
def test_quality_weighted_drift(api):
    """DESIGN 5.26's drift case with conf-weighted push and track, against its bounds unchanged: 16 frames of the
    KITTI-sized clip whose true relative motions carry a systematic bias (translation x 1.05, 0.1 degree of yaw per
    pair), tracked with integration: the last frame's translation error is at most half that of the chained poses, and
    the depth rendered at frame 0 is no worse than with the chained poses (median)."""
    KITTI = dict(fx=721.5, fy=721.5, cx=609.6, cy=172.9, baseline=0.54, doffs=0.0)
    QP = dict(nx=160, ny=55, nz=280, origin=(-8.0, -3.0, 3.0), voxel=0.1, trunc=0.3, max_weight=64.0, color=0)
    QT = dict(step=2, rounds=10, min_weight=0.5, max_depth=30.0, huber=0.2, damping=1.0, min_corr=100,
              max_shift=0.5, min_cos=math.cos(math.radians(5.0)), eps=1e-7, integrate=1)
    h, w, n = 375, 1242, 16
    rels = [pose((0.0, math.radians(0.3 * (k % 3 - 1)), 0.0), (0.02 * (k % 2), 0.0, -0.5)) for k in range(n - 1)]
    clip = synth.rigid_stereo_clip(n - 1, h, w, 1, 2, KITTI, rels, block={"velocity": (0.0, 0.0, 0.0)})
    prm = params.operating_point(2, w, noc=1, nop=1)
    ctx = context(api, prm, h, w, 2 * n)
    fwd = np.stack([clip["left"], clip["right"]], 1)
    ctx.upload_frames_u8(0, 2 * n, np.ascontiguousarray(np.concatenate([fwd, fwd[:, ::-1]])), w, h)
    ctx.set_swapped_slots(n, 2 * n, 1)
    ctx.run(2 * n)
    disp = ctx.disparity_fullres(0, n, n, w, h, lr_check=1, outputs=("disp",))["disp"]
    conf, _ = ctx.confidence_fullres(0, n, n, np.ascontiguousarray(clip["left"]), np.ascontiguousarray(clip["right"]),
                                     CP, w, h)
    G = clip["abs"]
    biased = []
    for k in range(n - 1):
        R, t = np.asarray(rels[k])[:, :3], np.asarray(rels[k])[:, 3] * 1.05
        biased.append(np.concatenate([synth.axis_angle((0.0, math.radians(0.1), 0.0)) @ R, t[:, None]], 1))
    biased = np.stack(biased)
    chained = preprocess.chain_poses(biased)
    ctx.fuse_begin(QP)
    ctx.fuse_push(disp[:1], G[:1], KITTI, width_org=w, height_org=h, weights=conf[:1])
    tracked, st = ctx.fuse_track(disp[1:], biased, G[0], KITTI, QT, width_org=w, height_org=h, weights=conf[1:])
    tracked = np.concatenate([G[:1], tracked])
    fb = f32(f32(KITTI["fx"]) * f32(KITTI["baseline"]))
    true = fb / (clip["disp"][0] + f32(KITTI["doffs"]))
    depth_t = ctx.fuse_render(G[:1], KITTI, z_near=3.0, z_far=30.0, step=0.05, width_org=w, height_org=h,
                              min_weight=0.5)[0]
    ctx.fuse_begin(QP)
    ctx.fuse_push(disp, chained, KITTI, width_org=w, height_org=h, weights=conf)
    depth_c = ctx.fuse_render(G[:1], KITTI, z_near=3.0, z_far=30.0, step=0.05, width_org=w, height_org=h,
                              min_weight=0.5)[0]
    ctx.close()
    tt, rt = preprocess.trajectory_errors(tracked, G)
    tc, rc = preprocess.trajectory_errors(chained, G)
    both = np.isfinite(depth_t) & np.isfinite(depth_c)
    figures = dict(t_tracked=float(tt[-1]), t_chained=float(tc[-1]), r_tracked=float(rt[-1]), r_chained=float(rc[-1]),
                   statuses=st["status"].tolist(), rounds=st["rounds"].tolist(),
                   depth_tracked=float(np.median(np.abs(depth_t[both] - true[both]))),
                   depth_chained=float(np.median(np.abs(depth_c[both] - true[both]))), pixels=int(both.sum()))
    print(json.dumps(figures))
    assert figures["t_tracked"] <= 0.5 * figures["t_chained"], figures
    assert figures["depth_tracked"] <= figures["depth_chained"], figures
