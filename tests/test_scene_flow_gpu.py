"""ofdis_scene_flow_fullres: every output byte and count must equal preprocess.scene_flow on the flows
ofdis_get_flow_fullres returns (gray and RGB, usefbcon 0 and 1, divisible and non-divisible sizes, host and device
memory, a chained clip's disparities, several classes); a stereo context's device disparities read across contexts on
one stream; every bad argument refused with the flows left as they were."""
import ctypes

import numpy as np
import pytest

from of_dis_b200 import params, preprocess, synth

pytestmark = pytest.mark.gpu

CAM = dict(fx=721.5, fy=707.0, cx=101.25, cy=60.5, baseline=0.54, doffs=0.25)
OUTS = ("disp1", "status", "motion")


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.fixture(scope="module")
def api():
    from of_dis_b200 import api as _api

    _api.lib()
    return _api


def prm_for(ch, fb, nop=2):
    return params.from_cli_numbers(("3 1 8 8 0.05 0.95 0 8 0.4 %d 1 0 1 10 10 5 1 3 1.6 0" % fb).split(),
                                   noc=ch, nop=nop)


def context(api, prm, h, w, max_frames, stream=None):
    scf = 1 << prm.sc_f
    W, H = (w + scf - 1) // scf * scf, (h + scf - 1) // scf * scf
    return api.Context(prm, W, H, prm.p_samp_s, max_frames, stream=stream)


def fullres(ctx, f0, f1, h, w):
    out = np.empty((f1 - f0, h, w, ctx.prm.nop), np.float32)
    ctx.get_flow_fullres(f0, f1, out, w, h)
    ctx.sync()
    return out


def clip_inputs(rng, flows, n, h, w):
    """n + 1 disparity maps (a chained clip) with unknown entries, ground truth near them and 3 classes + ignored."""
    maps = rng.uniform(0, 30, (n + 1, h, w)).astype(np.float32)
    maps[rng.random(maps.shape) < 0.05] = np.nan
    maps[rng.random(maps.shape) < 0.01] = -0.0
    d1w, _, _, _ = preprocess.scene_flow(flows, maps[:-1], maps[1:], 1.0)
    g0 = (maps[:-1] + rng.choice([0, 2, 4], maps[:-1].shape)).astype(np.float32)
    g1 = (np.nan_to_num(d1w, nan=10.0) + rng.choice([0, 1, 5], g0.shape)).astype(np.float32)
    gf = (flows + rng.choice([0.0, 0.5, 4.0], flows.shape)).astype(np.float32)
    for g in (g0, g1):
        g[rng.random(g.shape) < 0.05] = np.nan
    gf[rng.random(g0.shape) < 0.05] = np.nan
    cls = rng.integers(0, 4, g0.shape).astype(np.uint8)
    return maps, (g0, g1, gf), cls


def check(got, stats, exp, what):
    d1w, st, motion, est = exp
    assert (bits(got["disp1"]) == bits(d1w)).all(), what
    assert (got["status"] == st).all(), what
    assert (bits(got["motion"]) == bits(motion)).all(), what
    if est is not None:
        assert (stats == est).all(), (what, stats, est)


@pytest.mark.parametrize("size", [(128, 256), (121, 203)], ids=["div", "nondiv"])
@pytest.mark.parametrize("fb", [0, 1], ids=["fb0", "fb1"])
@pytest.mark.parametrize("ch", [1, 3])
def test_run_flows_equal_the_restatement(ch, fb, size, api):
    import torch

    h, w = size
    n = 3
    rng = np.random.default_rng(11 + ch + fb)
    frames = synth.synthetic_sequence(n + 1, h, w, ch, seed=21 + ch, amp=4.0)
    ctx = context(api, prm_for(ch, fb), h, w, n)
    ctx.upload_sequence_u8(0, n, frames, w, h)
    ctx.run(n)
    flows = fullres(ctx, 0, n, h, w)
    maps, gt, cls = clip_inputs(rng, flows, n, h, w)
    seen = set()
    for edge in (1.0, 0.0, np.inf):
        exp = preprocess.scene_flow(flows, maps[:-1], maps[1:], edge, CAM, gt, cls, 3)
        before = ctx.launch_count
        got, stats = ctx.scene_flow_fullres(0, n, maps[:-1], maps[1:], width_org=w, height_org=h, edge_diff=edge,
                                            camera=CAM, outputs=OUTS, gt=gt, classes=cls, nclasses=3)
        assert ctx.launch_count - before == 1
        check(got, stats, exp, "host edge %s" % edge)
        seen |= set(np.unique(got["status"]).tolist())
        # a sub-range, one class, without ground truth, and each output alone
        sub = preprocess.scene_flow(flows[1:], maps[1:-1], maps[2:], edge, CAM)
        for name in OUTS:
            part, st = ctx.scene_flow_fullres(1, n, np.ascontiguousarray(maps[1:-1]), np.ascontiguousarray(maps[2:]),
                                              width_org=w, height_org=h, edge_diff=edge,
                                              camera=CAM if name == "motion" else None, outputs=(name,))
            assert st is None
            ref = sub[OUTS.index(name)]
            assert (bits(part[name]) == bits(ref)).all() if name != "status" else (part[name] == ref).all()
        one = preprocess.scene_flow(flows, maps[:-1], maps[1:], edge, None, gt)[3]
        _, st1 = ctx.scene_flow_fullres(0, n, maps[:-1], maps[1:], width_org=w, height_org=h, edge_diff=edge,
                                        outputs=(), gt=gt)
        assert (st1 == one).all()
    assert seen >= {0, 1, 4}, seen
    # device memory: the chained clip as one array, read with disp_stride = one frame
    pix = h * w
    d_maps = torch.from_numpy(maps).cuda()
    d_gt = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in gt]
    d_cls = torch.from_numpy(cls).cuda()
    dev = {"disp1": torch.full((n, h, w), 7.0, device="cuda"),
           "status": torch.full((n, h, w), 9, dtype=torch.uint8, device="cuda"),
           "motion": torch.full((n, h, w, 3), 7.0, device="cuda")}
    torch.cuda.synchronize()
    exp = preprocess.scene_flow(flows, maps[:-1], maps[1:], 1.0, CAM, gt, cls, 3)
    _, stats = ctx.scene_flow_fullres(0, n, d_maps.data_ptr(), d_maps.data_ptr() + 4 * pix, width_org=w, height_org=h,
                                      camera=CAM, outputs=OUTS, gt=[a.data_ptr() for a in d_gt],
                                      classes=d_cls.data_ptr(), nclasses=3, memkind=api.MEM_DEVICE,
                                      out={k: v.data_ptr() for k, v in dev.items()}, disp_stride=pix)
    ctx.sync()
    check({k: v.cpu().numpy() for k, v in dev.items()}, stats, exp, "device")
    assert (bits(fullres(ctx, 0, n, h, w)) == bits(flows)).all(), "the flows must not change"
    ctx.close()


def test_disparities_of_a_stereo_context_on_the_same_stream(api):
    """A stereo context writes device disparities and point clouds; a flow context on the same stream reads them by
    address.  P0 of the motion is the stereo context's xyz bit for bit."""
    import torch

    h, w = 96, 160
    frames, truth = synth.layered_scene_flow(h, w, 1, seed=4, d_bg=6, d_fg=(16, 20), dx=4)
    stream = torch.cuda.Stream()
    sctx = context(api, prm_for(1, 0, nop=1), h, w, 2, stream=stream.cuda_stream)
    fctx = context(api, prm_for(1, 0), h, w, 1, stream=stream.cuda_stream)
    with torch.cuda.stream(stream):
        disp = torch.full((2, h, w), 7.0, device="cuda")
        xyz = torch.full((2, h, w, 3), 7.0, device="cuda")
        dev = {"disp1": torch.empty((1, h, w), device="cuda"),
               "status": torch.empty((1, h, w), dtype=torch.uint8, device="cuda"),
               "motion": torch.empty((1, h, w, 3), device="cuda")}
        sctx.upload_frames_u8(0, 2, np.ascontiguousarray(frames.reshape(2, 2, h, w)), w, h)
        sctx.run(2)
        sctx.disparity_fullres(0, 2, 0, w, h, camera=CAM, outputs=("disp", "xyz"), memkind=api.MEM_DEVICE,
                               out={"disp": disp.data_ptr(), "xyz": xyz.data_ptr()})
        fctx.upload_frames_u8(0, 1, np.ascontiguousarray(frames[[0, 2]][None]), w, h)
        fctx.run(1)
        fctx.scene_flow_fullres(0, 1, disp.data_ptr(), disp.data_ptr() + 4 * h * w, width_org=w, height_org=h,
                                camera=CAM, outputs=OUTS, memkind=api.MEM_DEVICE,
                                out={k: v.data_ptr() for k, v in dev.items()})
    stream.synchronize()
    flows = fullres(fctx, 0, 1, h, w)
    d = disp.cpu().numpy()
    exp = preprocess.scene_flow(flows, d[:1], d[1:], 1.0, CAM)
    got = {k: v.cpu().numpy() for k, v in dev.items()}
    check(got, None, exp, "cross-context")
    # motion = P1 - P0 with P0 the stereo context's xyz
    f32 = np.float32
    c = {k: f32(v) for k, v in CAM.items()}
    F = flows[0]
    xs = np.arange(w, dtype=f32)[None, :] + F[..., 0]
    ys = np.arange(h, dtype=f32)[:, None] + F[..., 1]
    d1 = got["disp1"][0]
    ok = (got["status"][0] == 0) & (d[0] + c["doffs"] > 0) & (d1 + c["doffs"] > 0)
    with np.errstate(all="ignore"):
        Z1 = f32(c["fx"] * c["baseline"]) / (d1 + c["doffs"])
        P1 = np.stack([((xs - c["cx"]) * Z1) / c["fx"], ((ys - c["cy"]) * Z1) / c["fy"], Z1], -1)
        m = (P1 - xyz.cpu().numpy()[0]).astype(f32)
    assert ok.sum() > h * w // 2
    assert (bits(got["motion"][0][ok]) == bits(m[ok])).all()
    sctx.close()
    fctx.close()


def test_bad_arguments_are_refused(api):
    import torch

    h, w, n = 64, 96, 2
    ctx = context(api, prm_for(1, 0), h, w, n)
    frames = synth.synthetic_sequence(n + 1, h, w, 1, seed=3, amp=3.0)
    ctx.upload_sequence_u8(0, n, frames, w, h)
    ctx.run(n)
    flows = fullres(ctx, 0, n, h, w)
    L = api.lib()
    pix = h * w
    d = torch.zeros((n + 1) * pix + 1, device="cuda")
    out = torch.zeros(3 * n * pix + 1, device="cuda")
    st = torch.zeros(n * pix, dtype=torch.uint8, device="cuda")
    cam = api.StereoCamera(*[CAM[k] for k in preprocess.STEREO_CAMERA_FIELDS])
    a, o = d.data_ptr(), out.data_ptr()
    gt = api.SfGt(a, a, a)
    stats = np.zeros((n, 16), preprocess.SF_STATS_DTYPE)
    S = stats.ctypes.data

    def call(f0=0, f1=n, d0=a, d1=a + 4 * pix, stride=pix, edge=1.0, c=ctypes.byref(cam), dw=o, s=st.data_ptr(),
             m=None, g=None, cls=None, ncls=1, sp=None, ww=w, hh=h, mem=1):
        return L.ofdis_scene_flow_fullres(ctx._h, f0, f1, d0, d1, stride, edge, c, dw, s, m, g, cls, ncls, sp, ww, hh, mem)

    assert call() == 0
    bad = [dict(f1=n + 1), dict(f0=1, f1=1), dict(f0=-1), dict(d0=None), dict(d1=None), dict(stride=pix - 1),
           dict(edge=float("nan")), dict(edge=-1.0), dict(dw=None, s=None), dict(g=ctypes.byref(gt)), dict(sp=S),
           dict(g=ctypes.byref(api.SfGt(a, None, a)), sp=S), dict(ncls=0), dict(ncls=17, g=ctypes.byref(gt), sp=S),
           dict(ncls=2, g=ctypes.byref(gt), sp=S), dict(m=o, c=None), dict(d0=a + 2), dict(dw=o + 1),
           dict(m=o + 2), dict(ww=w + 16), dict(hh=h - 17),
           dict(m=o, c=ctypes.byref(api.StereoCamera(0.0, 1.0, 0.0, 0.0, 1.0, 0.0))),
           dict(m=o, c=ctypes.byref(api.StereoCamera(1.0, 1.0, float("inf"), 0.0, 1.0, 0.0)))]
    for kw in bad:
        assert call(**kw) == -1, kw
    # a stereo context
    sctx = context(api, prm_for(1, 0, nop=1), h, w, 1)
    assert L.ofdis_scene_flow_fullres(sctx._h, 0, 1, a, a, pix, 1.0, None, o, None, None, None, None, 1, None, w, h,
                                      1) == -1
    sctx.close()
    assert (bits(fullres(ctx, 0, n, h, w)) == bits(flows)).all(), "the flows must not change"
    ctx.close()


def _read_pfm3(path):
    with open(path, "rb") as f:
        data = f.read()
    parts = data.split(b"\n", 3)
    assert parts[0] == b"PF" and float(parts[2]) < 0
    w, h = (int(x) for x in parts[1].split())
    return np.frombuffer(parts[3], "<f4").reshape(h, w, 3)[::-1]


def test_batch_command_on_a_kitti_layout_scene(tmp_path):
    """run_DE_INT_batch writes the disparities at t and t+1, run_OF_INT_batch --scene-flow reads them: the written
    disparities, motion and SFEVAL counts equal the restatement on the written flow."""
    import subprocess

    from of_dis_b200 import build

    bindir = build.build_host()
    h, w = 72, 120
    frames, truth = synth.layered_scene_flow(h, w, 1, seed=6, d_bg=6, d_fg=(16, 20), dx=4)
    for name, img in zip(("l0", "r0", "l1", "r1"), frames):
        preprocess.write_pgm(str(tmp_path / (name + ".pgm")), img)
    preprocess.write_kitti_png(str(tmp_path / "g0.png"), preprocess.encode_kitti(-truth["disp0"][..., None]))
    preprocess.write_kitti_png(str(tmp_path / "g1.png"), preprocess.encode_kitti(-truth["disp1"][..., None]))
    preprocess.write_kitti_png(str(tmp_path / "gf.png"), preprocess.encode_kitti(truth["flow"]))
    (tmp_path / "stereo.txt").write_text("l0.pgm r0.pgm d0.pfm\nl1.pgm r1.pgm d1.pfm\n")
    (tmp_path / "disps.txt").write_text("d0.pfm d1.pfm\n")
    (tmp_path / "gts.txt").write_text("g0.png g1.png gf.png\n")
    r = subprocess.run([str(bindir) + "/run_DE_INT_batch", "stereo.txt"], capture_output=True, text=True,
                       cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
    cam = ",".join(repr(float(CAM[k])) for k in preprocess.STEREO_CAMERA_FIELDS)
    d0 = -preprocess.read_pfm(str(tmp_path / "d0.pfm"))[..., 0]
    d1 = -preprocess.read_pfm(str(tmp_path / "d1.pfm"))[..., 0]
    gt = tuple(preprocess.kitti_to_flow(preprocess.read_kitti_png(str(tmp_path / f)), nop)
               for f, nop in (("g0.png", 1), ("g1.png", 1), ("gf.png", 2)))
    gt = (-gt[0][..., 0], -gt[1][..., 0], gt[2])
    for out, extra in (("out.flo", []), ("out.png", ["--kitti"])):
        (tmp_path / "flow.txt").write_text("l0.pgm l1.pgm %s\n" % out)
        r = subprocess.run([str(bindir) + "/run_OF_INT_batch", "flow.txt", "--scene-flow", "disps.txt", "--camera", cam,
                            "--gt-scene-flow", "gts.txt"] + extra, capture_output=True, text=True, cwd=str(tmp_path))
        assert r.returncode == 0, r.stderr
        if out == "out.flo":
            F = preprocess.read_flo(str(tmp_path / "out.flo"))
            d1w, _, motion, stats = preprocess.scene_flow(F, d0, d1, 1.0, CAM, gt)
            got = -preprocess.read_pfm(str(tmp_path / "out_disp1.pfm"))[..., 0]
            assert (bits(got) == bits(d1w)).all()
            assert (bits(_read_pfm3(str(tmp_path / "out_sceneflow.pfm"))) == bits(motion)).all()
        else:
            enc = preprocess.read_kitti_png(str(tmp_path / "out_disp1.png"))
            assert (enc == preprocess.encode_kitti(-d1w[..., None])).all()
        lines = [ln.split() for ln in r.stdout.splitlines() if ln.startswith("SFEVAL")]
        assert len(lines) == 2 and lines[0][1] == out and lines[1][1] == "(1", lines
        for ln in lines:
            vals = ln[ln.index("d1"):]
            for i, key in enumerate(("d1", "d2", "fl", "sf")):
                assert vals[4 * i] == key
                assert int(vals[4 * i + 1]) == stats["out_" + key] and int(vals[4 * i + 2]) == stats["n_" + key], ln
    assert stats["n_sf"] > h * w // 2
