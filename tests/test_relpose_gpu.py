"""ofdis_relpose_fullres: pose, stats, epipolar masks, Sampson distances and depths must equal preprocess.relpose of
the flows ofdis_get_flow_fullres returns, bit for bit (gray and RGB, usefbcon 0 and 1, fb_check on and off, divisible
and odd sizes, n = 1 and n = max_frames, host and device memory on a caller stream, planted special flows, an
all-invalid pair); one call against per-pair calls; a fixed launch count; every argument error; the grow-only
workspace; and on the KITTI-sized synthetic clip the fit must find the camera's rotation and direction of travel."""
import ctypes
import math

import numpy as np
import pytest
from scipy import ndimage

from of_dis_b200 import params, preprocess, synth

pytestmark = pytest.mark.gpu

SMALL = "3 %d 8 8 0.05 0.95 0 8 0.4 %d 1 0 1 10 10 5 1 3 1.6 0"
OUTS = ("mask", "sampson", "depth")


@pytest.fixture(scope="module")
def api():
    from of_dis_b200 import api as _api

    _api.lib()
    return _api


def context(api, prm, h, w, max_frames, stream=None):
    scf = 1 << prm.sc_f
    W, H = (w + scf - 1) // scf * scf, (h + scf - 1) // scf * scf
    return api.Context(prm, W, H, prm.p_samp_s, max_frames, stream=stream)


def fullres(ctx, f0, f1, h, w):
    out = np.empty((f1 - f0, h, w, 2), np.float32)
    ctx.get_flow_fullres(f0, f1, out, w, h)
    ctx.sync()
    return out


def motion(w=(0.0, 0.0, 0.0), t=(0.0, 0.0, 0.0)):
    return np.concatenate([synth.axis_angle(w), np.asarray(t, np.float64).reshape(3, 1)], 1)


def small_clip(n, h, w, ch, seed):
    cam = dict(fx=180.0, fy=176.5, cx=w / 2 - 0.25, cy=h / 2 + 0.5, baseline=0.54, doffs=0.25)
    rels = [motion((0.0, 0.01, 0.0), (0.03, 0.0, -0.5)), motion((0.004, -0.006, 0.002), (0.0, 0.01, -0.3)),
            motion((0.0, 0.0, 0.0), (0.05, 0.0, -0.6))][:n]
    return synth.rigid_stereo_clip(n, h, w, ch, seed, cam, rels), cam


def rp(cam, **kw):
    p = dict(fx=cam["fx"], fy=cam["fy"], cx=cam["cx"], cy=cam["cy"], step=4, fb_check=0, alpha=0.01, beta=0.5,
             hypotheses=128, threshold=1.0, refine=5, min_parallax=0.25, seed=3)
    p.update(kw)
    return p


def same(got, exp, what):
    for name, g, e in zip(("pose", "stats") + OUTS, got, exp):
        if g is None and e is None:
            continue
        gb, eb = np.ascontiguousarray(g).view(np.uint8), np.ascontiguousarray(e).view(np.uint8)
        if gb.shape != eb.shape or (gb != eb).any():
            raise AssertionError("%s %s differ: got %s expected %s" % (what, name, g if g.size < 40 else g.shape,
                                                                        e if e.size < 40 else e.shape))


def call(ctx, f0, f1, p, w, h, b0=None, outputs=OUTS):
    pose, stats, outs = ctx.relpose_fullres(f0, f1, p, width_org=w, height_org=h, b0=b0, outputs=outputs)
    return (pose, stats) + tuple(outs.get(k) for k in OUTS)


@pytest.mark.parametrize("size", [(96, 160), (91, 151)], ids=["div", "odd"])
@pytest.mark.parametrize("fb", [0, 1], ids=["fb0", "fb1"])
@pytest.mark.parametrize("ch", [1, 3])
def test_run_flows_equal_the_restatement(ch, fb, size, api):
    h, w = size
    n = 3
    clip, cam = small_clip(n, h, w, ch, seed=7 + ch)
    ctx = context(api, params.from_cli_numbers((SMALL % (1, fb)).split(), noc=ch, nop=2), h, w, 2 * n)
    ctx.upload_sequence_bidir_u8(0, n, clip["left"], w, h)
    ctx.run(2 * n)
    flows = fullres(ctx, 0, 2 * n, h, w)
    refits = 0
    for fbc, step in ((0, 4), (1, 4), (1, 1)):
        p = rp(cam, fb_check=fbc, step=step, hypotheses=64 if step == 1 else 128)
        exp = preprocess.relpose(flows[:n], flows[n:] if fbc else None, p)
        before = ctx.launch_count
        got = call(ctx, 0, n, p, w, h, b0=n if fbc else None)
        assert ctx.launch_count - before == 6
        same(got, exp, "fb_check %d step %d" % (fbc, step))
        assert (got[1]["best_hypothesis"] >= 0).all(), got[1]
        refits += int(got[1]["refits"].sum())
        # n = 1 at f0 != 0
        sub = preprocess.relpose(flows[1:2], flows[n + 1:n + 2] if fbc else None, p)
        before = ctx.launch_count
        same(call(ctx, 1, 2, p, w, h, b0=n + 1 if fbc else None), sub, "n = 1, fb_check %d" % fbc)
        assert ctx.launch_count - before == 6
    assert refits > 0
    # n = max_frames: the backward slots are flows too
    p = rp(cam)
    before = ctx.launch_count
    same(call(ctx, 0, 2 * n, p, w, h), preprocess.relpose(flows, None, p), "n = max_frames")
    assert ctx.launch_count - before == 6
    for f0, f1 in ((0, 1), (0, 2 * n)):
        before = ctx.launch_count
        call(ctx, f0, f1, p, w, h, outputs=())
        assert ctx.launch_count - before == 5
    before = ctx.launch_count
    got = call(ctx, 0, n, p, w, h, outputs=())
    assert ctx.launch_count - before == 5, "no per-pixel output: five launches, whatever the number of pairs"
    same(got[:2], preprocess.relpose(flows[:n], None, p)[:2], "pose only")
    # one call equals per-pair calls
    for k in range(n):
        one = call(ctx, k, k + 1, p, w, h)
        same(one, tuple(None if g is None else g[k:k + 1] for g in got[:2]) + one[2:], "pair %d" % k)
    ctx.close()


def test_device_memory_on_a_caller_stream(api):
    import torch

    h, w, n = 61, 90, 2
    prm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=3, nop=2)
    clip, cam = small_clip(n, h, w, 3, seed=37)
    stream = torch.cuda.Stream()
    ctx = context(api, prm, h, w, 2 * n, stream=stream.cuda_stream)
    ctx.set_graph_mode(True)
    for _ in range(2):  # capture, then replay
        ctx.upload_sequence_bidir_u8(0, n, clip["left"], w, h)
        ctx.run(2 * n)
    flows = fullres(ctx, 0, 2 * n, h, w)
    p = rp(cam, fb_check=1, step=2)
    exp = preprocess.relpose(flows[:n], flows[n:], p)
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        dm = torch.full((n, h, w), 9, dtype=torch.uint8, device="cuda")
        ds = torch.full((n, h, w), 7.0, device="cuda")
        dd = torch.full((n, h, w), 7.0, device="cuda")
        pose, stats, _ = ctx.relpose_fullres(0, n, p, width_org=w, height_org=h, b0=n, outputs=OUTS,
                                             out=dict(mask=dm.data_ptr(), sampson=ds.data_ptr(), depth=dd.data_ptr()),
                                             memkind=api.MEM_DEVICE)
    stream.synchronize()
    same((pose, stats, dm.cpu().numpy(), ds.cpu().numpy(), dd.cpu().numpy()), exp, "device")
    same(call(ctx, 0, n, p, w, h, b0=n), exp, "host")
    ctx.close()


def test_special_level_flows(api):
    """Level flows set at sc_l = 0: a rigid flow with NaN, +-inf and 3e9 planted fits; an all-invalid pair has status
    1; a zero flow is restated bit for bit too."""
    h, w = 48, 64
    clip, cam = small_clip(1, h, w, 1, seed=5)
    prm = params.from_cli_numbers("3 0 8 8 0.05 0.95 0 8 0.4 0 1 0 0 10 10 5 1 3 1.6 0".split(), noc=1, nop=2)
    ctx = context(api, prm, h, w, 3)
    a = clip["flow"][0].astype(np.float32).copy()
    a[::3, ::5] = np.nan
    a[1::7, ::2, 0] = np.inf
    a[2::5, 1::3, 1] = -np.inf
    a[3::4, 3::4, 0] = 3e9
    flows = [a, np.full((h, w, 2), np.nan, np.float32), np.zeros((h, w, 2), np.float32)]
    for k, f in enumerate(flows):
        ctx.set_flow(k, 0, f)
    full = fullres(ctx, 0, 3, h, w)
    assert (full.view(np.uint32) == np.stack(flows).view(np.uint32)).all()
    p = rp(cam, step=1, hypotheses=256)
    got = call(ctx, 0, 3, p, w, h)
    same(got, preprocess.relpose(full, None, p), "special")
    assert got[1]["status"].tolist()[:2] == [0, 1], got[1]
    assert set(np.unique(got[2][0]).tolist()) <= {0, 1, 2} and (got[2][0] == 0).any()
    assert np.isnan(got[0][1]).all()
    ctx.close()


def test_argument_errors(api):
    h, w, n = 61, 90, 2
    prm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=1, nop=2)
    clip, cam = small_clip(n, h, w, 1, seed=43)
    ctx = context(api, prm, h, w, 2 * n)
    ctx.upload_sequence_bidir_u8(0, n, clip["left"], w, h)
    ctx.run(2 * n)
    flows = fullres(ctx, 0, 2 * n, h, w)
    L = api.lib()
    pose = np.empty((2 * n, 12))
    stats = np.zeros(2 * n, preprocess.MOTION_STATS_DTYPE)
    good = rp(cam)

    def rc(f0=0, f1=n, b0=-1, p=None, ps=True, st=True, kind=0, ww=w, hh=h, **kw):
        q = dict(good)
        q.update(kw)
        prm_ = api.RelposeParams(*[q[k] for k in preprocess.RELPOSE_PARAM_FIELDS])
        return L.ofdis_relpose_fullres(ctx._h, f0, f1, b0, ctypes.byref(prm_) if p is None else None,
                                       api._ptr(pose) if ps else None, api._ptr(stats) if st else None, None, None,
                                       None, ww, hh, kind)

    assert rc() == 0
    bad = [dict(f0=-1), dict(f1=2 * n + 1), dict(f0=1, f1=1), dict(fb_check=1, b0=-1), dict(fb_check=1, b0=n + 1),
           dict(fb_check=2), dict(step=0), dict(alpha=-1.0), dict(beta=math.inf), dict(fx=0.0), dict(fy=-1.0),
           dict(fx=math.inf), dict(cx=math.nan), dict(cy=math.inf), dict(hypotheses=0), dict(hypotheses=65537),
           dict(threshold=0.0), dict(threshold=math.nan), dict(refine=-1), dict(refine=17),
           dict(min_parallax=-0.5), dict(min_parallax=math.inf), dict(p=0), dict(ps=False), dict(st=False),
           dict(ww=w + 64), dict(hh=0)]
    for kw in bad:
        assert rc(**kw) == -1, kw
    # misaligned device outputs
    import torch

    buf = torch.zeros(n * h * w + 4, device="cuda")
    prm_ = api.RelposeParams(*[good[k] for k in preprocess.RELPOSE_PARAM_FIELDS])
    for which in (1, 2):
        ptrs = [None, None, None]
        ptrs[which] = buf.data_ptr() + 2
        assert L.ofdis_relpose_fullres(ctx._h, 0, n, -1, ctypes.byref(prm_), api._ptr(pose), api._ptr(stats),
                                       *ptrs, w, h, 1) == -1
    # more than 2^24 cells per pair: a 4096 x 4097 context at step 1
    big = api.Context(params.from_cli_numbers("0 0 8 8 0.05 0.95 0 8 0.4 0 1 0 0 10 10 5 1 3 1.6 0".split(), noc=1,
                                               nop=2), 4096, 4097, 8, 1)
    p1 = api.RelposeParams(*[dict(good, step=1)[k] for k in preprocess.RELPOSE_PARAM_FIELDS])
    assert L.ofdis_relpose_fullres(big._h, 0, 1, -1, ctypes.byref(p1), api._ptr(pose), api._ptr(stats), None, None,
                                   None, 4096, 4097, 0) == -1
    big.close()
    # a stereo context
    sprm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=1, nop=1)
    sctx = context(api, sprm, h, w, 1)
    assert L.ofdis_relpose_fullres(sctx._h, 0, 1, -1, ctypes.byref(prm_), api._ptr(pose), api._ptr(stats), None,
                                   None, None, w, h, 0) == -1
    sctx.close()
    # the flows are left as they were
    assert (fullres(ctx, 0, 2 * n, h, w).view(np.uint32) == flows.view(np.uint32)).all()
    ctx.close()


def test_grow_only_workspace(api):
    """A small call, a large one (more cells and hypotheses), the small one again: each equals the same call on a
    fresh context."""
    h, w, n = 61, 90, 2
    prm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=1, nop=2)
    clip, cam = small_clip(n, h, w, 1, seed=11)

    def run(ctx):
        ctx.upload_sequence_bidir_u8(0, n, clip["left"], w, h)
        ctx.run(2 * n)

    small = rp(cam, step=6, hypotheses=32)
    large = rp(cam, step=1, hypotheses=600)
    ctx = context(api, prm, h, w, 2 * n)
    run(ctx)
    seq = [call(ctx, 0, n, q, w, h) for q in (small, large, small)]
    for q, got in zip((small, large, small), seq):
        fresh = context(api, prm, h, w, 2 * n)
        run(fresh)
        same(got, call(fresh, 0, n, q, w, h), "grow-only step %d" % q["step"])
        fresh.close()
    ctx.close()


@pytest.fixture(scope="module")
def kitti_figures(api):
    """synth.rigid_stereo_clip at KITTI's size and camera, left frames only, DIS flows at operating point 2 with the
    two-way upload and fb_check (tools/relpose_prestudy.py gives the same figures on the CPU): per pair the status, the rotation and translation-direction errors in degrees, the
    share of the moving box's eroded interior at mask 1 and the AbsRel of the median-scaled depth on the mask-0
    background."""
    h, w, n = 375, 1242, 3
    cam = dict(fx=721.5, fy=721.5, cx=609.6, cy=172.9, baseline=0.54, doffs=0.0)
    rels = [motion((0.0, math.radians(0.5), 0.0), (0.0, 0.0, -0.9)),
            motion((math.radians(0.3), math.radians(-0.8), 0.0), (0.1, 0.0, -0.6)),
            motion((0.0, math.radians(1.0), 0.0), (0.0, 0.0, -0.3))]
    clip = synth.rigid_stereo_clip(n, h, w, 1, 2, cam, rels)
    prm = params.operating_point(2, w, noc=1)
    ctx = context(api, prm, h, w, 2 * n)
    ctx.upload_sequence_bidir_u8(0, n, clip["left"], w, h)
    ctx.run(2 * n)
    p = rp(cam, step=4, fb_check=1, hypotheses=1024, refine=5, min_parallax=0.5, seed=0)
    pose, stats, outs = ctx.relpose_fullres(0, n, p, width_org=w, height_org=h, b0=n, outputs=OUTS)
    ctx.close()
    r_err, t_err = preprocess.relpose_errors(pose, clip["poses"])
    fb = np.float32(np.float32(cam["fx"]) * np.float32(cam["baseline"]))
    figs = []
    for k in range(n):
        box = clip["box"][k]
        interior = ndimage.binary_erosion(box, iterations=8)
        back = ~ndimage.binary_dilation(box, iterations=8)
        true_depth = fb / clip["disp"][k].astype(np.float64)
        d = outs["depth"][k].astype(np.float64)
        sel = back & (outs["mask"][k] == 0) & np.isfinite(d) & np.isfinite(true_depth)
        scale = np.median(true_depth[sel]) / np.median(d[sel])
        figs.append(dict(status=int(stats["status"][k]), r_err=float(r_err[k]), t_err=float(t_err[k]),
                         moving=float((outs["mask"][k][interior] == 1).mean()),
                         absrel=float(np.mean(np.abs(d[sel] * scale - true_depth[sel]) / true_depth[sel]))))
        print("pair %d: status %d, r_err %.4f deg, t_dir_err %.3f deg, box at mask 1 %.3f, AbsRel %.4f"
              % ((k,) + tuple(figs[k][key] for key in ("status", "r_err", "t_err", "moving", "absrel"))))
    return figs


def test_camera_motion_of_a_synthetic_clip(kitti_figures):
    """The first two pairs: status 0, the rotation within 0.1 degrees, the direction of travel within 3 degrees, at
    least 90 % of the moving box's eroded interior at mask 1; the first pair's depth within AbsRel 0.10."""
    for k, f in enumerate(kitti_figures[:2]):
        assert f["status"] == 0, (k, f)
        assert f["r_err"] <= 0.1 and f["t_err"] <= 3.0, (k, f)
        assert f["moving"] >= 0.9, (k, f)
    assert kitti_figures[0]["absrel"] <= 0.10, kitti_figures[0]


@pytest.mark.xfail(strict=True, reason="the second pair's direction of travel is 2.9 degrees off with DIS flows, and "
                   "its median-scaled depth misses AbsRel 0.10 (0.136; DESIGN 5.28)")
def test_depth_of_the_second_pair(kitti_figures):
    assert kitti_figures[1]["absrel"] <= 0.10, kitti_figures[1]


@pytest.mark.xfail(strict=True, reason="the third pair (0.3 m forward, 1 degree of yaw) has the least parallax; with "
                   "DIS flows its fit lands 1.5 degrees and 141 degrees off, against 0.009 and 0.58 degrees with the "
                   "exact flow (DESIGN 5.28)")
def test_camera_motion_of_the_third_pair(kitti_figures):
    f = kitti_figures[2]
    assert f["status"] == 0 and f["r_err"] <= 0.1 and f["t_err"] <= 3.0 and f["moving"] >= 0.9, f
    assert f["absrel"] <= 0.10, f


def test_stationary_pairs_have_status_3(api):
    """Identical frames and a pure rotation of a static scene at KITTI's size: status 3 (too little parallax)."""
    h, w = 375, 1242
    cam = dict(fx=721.5, fy=721.5, cx=609.6, cy=172.9, baseline=0.54, doffs=0.0)
    clip = synth.rigid_stereo_clip(1, h, w, 1, 2, cam, [motion((0.0, math.radians(1.0), 0.0))],
                                   block=dict(velocity=(0.0, 0.0, 0.0)))
    prm = params.operating_point(2, w, noc=1)
    p = rp(cam, step=4, fb_check=1, hypotheses=1024, refine=5, min_parallax=0.5, seed=0)
    st = []
    for frames in (np.stack([clip["left"][0], clip["left"][0]]), clip["left"]):
        ctx = context(api, prm, h, w, 2)
        ctx.upload_sequence_bidir_u8(0, 1, frames, w, h)
        ctx.run(2)
        st.append(int(ctx.relpose_fullres(0, 1, p, width_org=w, height_org=h, b0=1)[1]["status"][0]))
        ctx.close()
    assert st == [3, 3], st


def _read_pgm(path):
    with open(path, "rb") as f:
        data = f.read()
    parts = data.split(b"\n", 3)
    assert parts[0] == b"P5"
    w, h = (int(x) for x in parts[1].split())
    return np.frombuffer(parts[3], np.uint8).reshape(h, w)


def test_batch_command_mono_odometry(tmp_path):
    """A chained clip of three pairs and an unrelated pair (two clips) through run_OF_INT_batch --bidirectional
    --mono-odometry --intrinsics --gt-poses: monodometry.txt, the epipolar masks and relative depths equal the
    restatement on the written flows pair for pair, the poses files chain the relative poses with the ground truth's
    step lengths, and MONOEVAL gives the errors of the pairs of status 0."""
    import subprocess

    from of_dis_b200 import build

    bindir = build.build_host()
    h, w, n = 91, 150, 3
    clip, cam = small_clip(n, h, w, 1, seed=31)
    for k in range(n + 1):
        preprocess.write_pgm(str(tmp_path / ("f%d.pgm" % k)), clip["left"][k])
    pairs = [(k, k + 1) for k in range(n)] + [(2, 0)]  # the last pair starts a clip of its own
    (tmp_path / "list.txt").write_text("".join("f%d.pgm f%d.pgm out%d.flo\n" % (a, b, j)
                                               for j, (a, b) in enumerate(pairs)))
    gt_abs = preprocess.chain_poses(clip["poses"])
    preprocess.write_kitti_poses(str(tmp_path / "gt0.txt"), gt_abs)
    preprocess.write_kitti_poses(str(tmp_path / "gt1.txt"), gt_abs[:2])
    (tmp_path / "gts.txt").write_text("gt0.txt gt1.txt\n")
    (tmp_path / "mono").mkdir()
    K = [np.float32(cam[k]) for k in ("fx", "fy", "cx", "cy")]
    r = subprocess.run([str(bindir) + "/run_OF_INT_batch", "list.txt", "--bidirectional", "--mono-odometry", "mono",
                        "--intrinsics", ",".join(repr(float(v)) for v in K), "--gt-poses", "gts.txt"],
                       capture_output=True, text=True, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
    p = dict(fx=K[0], fy=K[1], cx=K[2], cy=K[3], step=8, fb_check=1, alpha=0.01, beta=0.5, hypotheses=1024,
             threshold=1.0, refine=5, min_parallax=0.5, seed=0)
    lines = [ln.split() for ln in (tmp_path / "mono" / "monodometry.txt").read_text().splitlines()]
    assert len(lines) == len(pairs)
    rels, st0 = {0: [], 1: []}, []
    for j, (a, b) in enumerate(pairs):
        F = preprocess.read_flo(str(tmp_path / ("out%d.flo" % j)))
        B = preprocess.read_flo(str(tmp_path / ("out%d_bw.flo" % j)))
        pose, stats, mask, _, depth = preprocess.relpose(F[None], B[None], p)
        clip_id, frame = (0, j) if j < n else (1, 0)
        assert [int(v) for v in lines[j][:3]] == [clip_id, frame, stats[0]["status"]], (j, lines[j])
        got = np.array([float(v) for v in lines[j][3:]])
        assert (got.view(np.uint64) == pose[0].ravel().view(np.uint64)).all(), j
        rels[clip_id].append(got.reshape(3, 4))
        st0.append(stats[0]["status"] == 0)
        assert (_read_pgm(str(tmp_path / ("out%d_epimask.pgm" % j))) == np.array([0, 255, 128], np.uint8)[mask[0]]).all()
        dr = -preprocess.read_pfm(str(tmp_path / ("out%d_depthrel.pfm" % j)))[..., 0]  # the body as _depth.pfm's
        assert np.array_equal(dr.view(np.uint32), depth[0].view(np.uint32)), j
    for c, gt in ((0, gt_abs), (1, gt_abs[:2])):
        poses = preprocess.read_kitti_poses(str(tmp_path / "mono" / ("poses_%04d.txt" % c)))
        steps = np.linalg.norm(gt[1:len(rels[c]) + 1, :, 3] - gt[:len(rels[c]), :, 3], axis=1)
        assert poses.shape == (len(rels[c]) + 1, 3, 4)
        assert np.allclose(poses, preprocess.chain_poses(np.stack(rels[c]), steps), rtol=0, atol=1e-12,
                           equal_nan=True)
    ev = [ln.split() for ln in r.stdout.splitlines() if ln.startswith("MONOEVAL")]
    assert len(ev) == sum(st0) + 1 and ev[-1][1] == "(%d" % sum(st0), ev
    errs = []
    for c, gt in ((0, gt_abs), (1, gt_abs[:2])):
        gt_rel = np.stack([np.linalg.inv(preprocess._pose44(gt[k + 1])) @ preprocess._pose44(gt[k])
                           for k in range(len(rels[c]))])[:, :3]
        errs += list(zip(*preprocess.relpose_errors(np.stack(rels[c]), gt_rel)))
    errs = [e for e, ok in zip(errs, st0) if ok]
    for line, (re, te) in zip(ev[:-1], errs):
        assert np.isclose(float(line[3]), re, rtol=1e-6, atol=1e-6), (line, re)
        assert np.isclose(float(line[4]), te, rtol=1e-6, atol=1e-6), (line, te)
