"""ofdis_global_motion_fullres: models, stats, masks, residuals and registered bytes must equal
preprocess.global_motion of the flows ofdis_get_flow_fullres returns, bit for bit, across the three models, gray and
RGB, usefbcon 0 and 1, fb_check on and off with the two-way upload and with pairs plus swapped copies, padded and
unpadded sizes, steps 1 and 8, f0 != 0 and b0 != f1, one call against per-pair calls, host and device memory on a
caller stream in graph mode, special level flows and every argument error; and the fit must find the camera motion of
synth.global_motion_clip."""
import ctypes
import json

import numpy as np
import pytest
from scipy import ndimage

from of_dis_b200 import params, preprocess, synth

pytestmark = pytest.mark.gpu

MODELS = ("similarity", "affine", "homography")
SMALL = "3 %d 8 8 0.05 0.95 0 8 0.4 %d 1 0 1 10 10 5 1 3 1.6 0"


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


def mp(model, **kw):
    p = dict(model=model, step=8, fb_check=0, alpha=0.01, beta=0.5, hypotheses=128, threshold=1.0, refine=3, seed=11)
    p.update(kw)
    return p


def outputs(n, h, w, noc):
    frame = (h, w) + ((noc,) if noc > 1 else ())
    return dict(mask=np.full((n, h, w), 7, np.uint8), residual=np.full((n, h, w, 2), 7.0, np.float32),
                registered=np.full((n,) + frame, 7, np.uint8))


def same(got, exp, what):
    for name, g, e in zip(("models", "stats", "mask", "residual", "registered"), got, exp):
        if g is None and e is None:
            continue
        gb, eb = np.ascontiguousarray(g).view(np.uint8), np.ascontiguousarray(e).view(np.uint8)
        if gb.shape != eb.shape or (gb != eb).any():
            raise AssertionError("%s %s differ: got %s expected %s" % (what, name, g if g.size < 40 else g.shape,
                                                                        e if e.size < 40 else e.shape))


def call(ctx, f0, f1, p, w, h, b0=None, i1=None, outs=None):
    o = outs or {}
    models, stats = ctx.global_motion_fullres(f0, f1, p, width_org=w, height_org=h, b0=b0, i1=i1, **o)
    return models, stats, o.get("mask"), o.get("residual"), o.get("registered")


def expected(flows, f0, f1, b0, i1, p, outs=True):
    e = preprocess.global_motion(flows[f0:f1], None if b0 is None else flows[b0:b0 + f1 - f0], i1, p)
    return e if outs else (e[0], e[1], None, None, None)


@pytest.mark.parametrize("size", [(64, 96), (61, 90)], ids=["div", "nondiv"])
@pytest.mark.parametrize("fb", [0, 1], ids=["fb0", "fb1"])
@pytest.mark.parametrize("ch", [1, 3])
def test_run_flows_equal_the_restatement(ch, fb, size, api):
    h, w = size
    n = 3
    prm = params.from_cli_numbers((SMALL % (1, fb)).split(), noc=ch, nop=2)
    clip = synth.synthetic_sequence(n + 1, h, w, ch, seed=31 + ch, amp=3.0)
    ctx = context(api, prm, h, w, 2 * n)
    ctx.upload_sequence_bidir_u8(0, n, clip, w, h)
    ctx.run(2 * n)
    flows = fullres(ctx, 0, 2 * n, h, w)
    statuses = set()
    for model in MODELS:
        # forward slots against their backward partners, a sub-range at f0 != 0, the backward slots against the forward
        for f0, f1, b0, i1 in ((0, n, n, clip[1:]), (1, 3, n + 1, clip[2:4]), (n, 2 * n, 0, clip[:-1])):
            for fbc, step in ((0, 8), (1, 8), (1, 1)):
                p = mp(model, fb_check=fbc, step=step, hypotheses=64 if step == 1 else 128)
                exp = expected(flows, f0, f1, b0 if fbc else None, i1, p)
                before = ctx.launch_count
                got = call(ctx, f0, f1, p, w, h, b0 if fbc else None, i1, outputs(f1 - f0, h, w, ch))
                assert ctx.launch_count - before == 6
                same(got, exp, "%s slots %d..%d fb_check %d step %d" % (model, f0, f1, fbc, step))
                statuses |= set(got[1]["status"].tolist())
                if step == 1:
                    assert (got[1]["n_corr"] > 4096).all(), "more than one score tile"
        before = ctx.launch_count
        got = call(ctx, 0, 2 * n, mp(model), w, h)
        assert ctx.launch_count - before == 5, "no per-pixel output: five launches, whatever the number of pairs"
        same(got, expected(flows, 0, 2 * n, None, None, mp(model), outs=False), "%s models only" % model)
    assert statuses == {0}
    assert (fullres(ctx, 0, 2 * n, h, w).view(np.uint32) == flows.view(np.uint32)).all(), "the flows must not change"
    ctx.close()


@pytest.mark.parametrize("ch", [1, 3])
def test_pairs_with_swapped_copies_and_slot_independence(ch, api):
    """The pair upload of the forward pairs and their swapped copies; one call over every pair gives what one call
    per pair gives."""
    h, w, n = 61, 90, 3
    prm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=ch, nop=2)
    clip = synth.synthetic_sequence(n + 1, h, w, ch, seed=41, amp=3.0)
    fwd = np.stack([clip[:-1], clip[1:]], axis=1)
    bwd = np.stack([clip[1:], clip[:-1]], axis=1)
    pairs = np.ascontiguousarray(np.concatenate([fwd, bwd]))
    ctx = context(api, prm, h, w, 2 * n)
    ctx.upload_frames_u8(0, 2 * n, pairs, w, h)
    ctx.run(2 * n)
    flows = fullres(ctx, 0, 2 * n, h, w)
    for model in MODELS:
        p = mp(model, fb_check=1)
        whole = call(ctx, 0, 2 * n, p, w, h, b0=0, i1=pairs[:, 1], outs=outputs(2 * n, h, w, ch))
        # b0 = 0 pairs slot k with slot k: forward against forward, only the consistent stay
        same(whole, expected(flows, 0, 2 * n, 0, pairs[:, 1], p), "%s b0 = f0" % model)
        whole = call(ctx, 0, n, p, w, h, b0=n, i1=pairs[:n, 1], outs=outputs(n, h, w, ch))
        same(whole, expected(flows, 0, n, n, pairs[:n, 1], p), "%s pairs + swapped" % model)
        for k in range(n):
            one = call(ctx, k, k + 1, p, w, h, b0=n + k, i1=pairs[k:k + 1, 1], outs=outputs(1, h, w, ch))
            same(one, tuple(a[k:k + 1] for a in whole), "%s pair %d alone" % (model, k))
    ctx.close()


def test_device_memory_on_a_caller_stream_in_graph_mode(api):
    import torch

    h, w, n = 61, 90, 2
    prm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=3, nop=2)
    clip = synth.synthetic_sequence(n + 1, h, w, 3, seed=37, amp=3.0)
    stream = torch.cuda.Stream()
    ctx = context(api, prm, h, w, 2 * n, stream=stream.cuda_stream)
    ctx.set_graph_mode(True)
    for _ in range(2):  # capture, then replay
        ctx.upload_sequence_bidir_u8(0, n, clip, w, h)
        ctx.run(2 * n)
    flows = fullres(ctx, 0, 2 * n, h, w)
    dclip = torch.from_numpy(clip).cuda()
    torch.cuda.synchronize()
    for model in MODELS:
        p = mp(model, fb_check=1)
        exp = expected(flows, 0, n, n, clip[1:], p)
        with torch.cuda.stream(stream):
            dm = torch.full((n, h, w), 9, dtype=torch.uint8, device="cuda")
            dr = torch.full((n, h, w, 2), 7.0, device="cuda")
            dg = torch.full((n, h, w, 3), 9, dtype=torch.uint8, device="cuda")
            models, stats = ctx.global_motion_fullres(0, n, p, width_org=w, height_org=h, b0=n,
                                                      i1=dclip[1:].data_ptr(), mask=dm.data_ptr(),
                                                      residual=dr.data_ptr(), registered=dg.data_ptr(),
                                                      memkind=api.MEM_DEVICE)
        stream.synchronize()
        same((models, stats, dm.cpu().numpy(), dr.cpu().numpy(), dg.cpu().numpy()), exp, "device %s" % model)
        same(call(ctx, 0, n, p, w, h, b0=n, i1=clip[1:], outs=outputs(n, h, w, 3)), exp, "host %s" % model)
    ctx.close()


def test_special_level_flows(api):
    """Level flows set at sc_l = 0: NaN, +-inf and values beyond 1e9 are unknown; a pair without correspondences has
    status 1 and a pair of one valid cell too; a constant shift is found exactly."""
    h, w = 40, 56
    prm = params.from_cli_numbers("3 0 8 8 0.05 0.95 0 8 0.4 0 1 0 0 10 10 5 1 3 1.6 0".split(), noc=1, nop=2)
    ctx = context(api, prm, h, w, 4)
    rng = np.random.default_rng(5)
    base = np.zeros((h, w, 2), np.float32)
    base[..., 0], base[..., 1] = 1.25, -0.5
    a = base + rng.normal(0, 0.1, base.shape).astype(np.float32)
    a[::3, ::5] = np.nan
    a[1::7, ::2, 0] = np.inf
    a[2::5, 1::3, 1] = -np.inf
    a[3::4, 3::4, 0] = 2e9
    a[10:20, 10:20] = [4.0, 3.0]
    flows = [a, np.full((h, w, 2), np.nan, np.float32), np.full((h, w, 2), 1e10, np.float32), base]
    flows[2][5, 5] = [0.5, 0.5]  # one valid cell (the seed pixel of cell (2, 2))
    for k, f in enumerate(flows):
        ctx.set_flow(k, 0, f)
    full = fullres(ctx, 0, 4, h, w)
    assert (full.view(np.uint32) == np.stack(flows).view(np.uint32)).all()
    i1 = rng.integers(0, 256, (4, h, w), dtype=np.uint8)
    for model in MODELS:
        p = mp(model, step=2)
        got = call(ctx, 0, 4, p, w, h, i1=i1, outs=outputs(4, h, w, 1))
        same(got, expected(full, 0, 4, None, i1, p), "special %s" % model)
        assert got[1]["status"].tolist() == [0, 1, 1, 0]
        assert set(np.unique(got[2][0]).tolist()) == {0, 1, 2}
    ctx.close()


def test_argument_errors(api):
    h, w, n = 61, 90, 2
    prm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=1, nop=2)
    clip = synth.synthetic_sequence(n + 1, h, w, 1, seed=43, amp=3.0)
    ctx = context(api, prm, h, w, 2 * n)
    ctx.upload_sequence_bidir_u8(0, n, clip, w, h)
    ctx.run(2 * n)
    L = api.lib()
    models = np.empty((n, 9))
    stats = np.empty(n, preprocess.MOTION_STATS_DTYPE)
    i1 = np.ascontiguousarray(clip[1:])
    reg = np.empty((n, h, w), np.uint8)

    def rc(f0=0, f1=n, b0=n, p=None, i1p=i1.ctypes.data, stride=h * w, m=models, s=stats, mask=None, res=None,
           regp=None, ww=w, hh=h, memkind=api.MEM_HOST, **kw):
        q = mp("affine", fb_check=1)
        q.update(kw)
        prm_ = api.MotionParams(*[preprocess.motion_params(q)[k] for k in preprocess.MOTION_PARAM_FIELDS]) \
            if p is None else p
        return L.ofdis_global_motion_fullres(ctx._h, f0, f1, b0, ctypes.byref(prm_) if prm_ is not False else None,
                                             api._ptr(i1p), stride, api._ptr(m), api._ptr(s), api._ptr(mask),
                                             api._ptr(res), api._ptr(regp), ww, hh, memkind)

    assert rc() == 0
    bad = [dict(f0=-1), dict(f1=2 * n + 1), dict(f0=1, f1=1), dict(b0=-1), dict(b0=n + 1), dict(p=False),
           dict(model=0), dict(model=4), dict(step=0), dict(fb_check=2), dict(alpha=-1.0), dict(alpha=float("inf")),
           dict(beta=float("nan")), dict(hypotheses=0), dict(hypotheses=65537), dict(threshold=0.0),
           dict(threshold=float("inf")), dict(refine=-1), dict(refine=17), dict(m=None), dict(s=None),
           dict(regp=reg.ctypes.data, i1p=None), dict(regp=reg.ctypes.data, stride=h * w - 1),
           dict(res=1, memkind=api.MEM_DEVICE), dict(step=1, ww=w + 64, hh=h), dict(ww=w - 16)]
    for b in bad:
        assert rc(**b) == -1, b  # OFDIS_ERR_ARG
    assert rc(b0=n + 1, fb_check=0) == 0, "b0 is read with fb_check only"
    # more than 2^24 cells per pair: a 4096 x 4097 context at step 1
    big = api.Context(params.from_cli_numbers("0 0 8 8 0.05 0.95 0 8 0.4 0 1 0 0 10 10 5 1 3 1.6 0".split(), noc=1,
                                               nop=2), 4096, 4097, 8, 1)
    p1 = api.MotionParams(*[preprocess.motion_params(mp("affine", step=1))[k] for k in preprocess.MOTION_PARAM_FIELDS])
    assert L.ofdis_global_motion_fullres(big._h, 0, 1, 0, ctypes.byref(p1), None, 0, api._ptr(models),
                                         api._ptr(stats), None, None, None, 4096, 4097, 0) == -1
    big.close()
    # a stereo context
    sprm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=1, nop=1)
    sctx = context(api, sprm, h, w, 2)
    p2 = api.MotionParams(*[preprocess.motion_params(mp("affine"))[k] for k in preprocess.MOTION_PARAM_FIELDS])
    assert L.ofdis_global_motion_fullres(sctx._h, 0, 1, 0, ctypes.byref(p2), None, 0, api._ptr(models),
                                         api._ptr(stats), None, None, None, w, h, 0) == -1
    sctx.close()
    ctx.close()


def test_camera_motion_of_a_synthetic_clip(api):
    """synth.global_motion_clip: rotation 0.5 deg, zoom 1.01 and a 3 px shift, and a rectangle of about 15 % of the
    frame that moves on its own, at operating point 2 with the two-way upload and fb_check."""
    h, w, n = 218, 512, 2
    H = synth.similarity_about_centre(h, w, 0.5, 1.01, (3.0, 0.0))
    figures = {}
    for ch in (1, 3):
        clip, models, rect = synth.global_motion_clip(n, h, w, ch, seed=9, H=H)
        prm = params.operating_point(2, w, noc=ch)
        ctx = context(api, prm, h, w, 2 * n)
        ctx.upload_sequence_bidir_u8(0, n, clip, w, h)
        ctx.run(2 * n)
        p = mp("homography", fb_check=1, hypotheses=1024)
        mask = np.empty((n, h, w), np.uint8)
        got, stats = ctx.global_motion_fullres(0, n, p, width_org=w, height_org=h, b0=n, mask=mask)
        ctx.close()
        y, x = np.mgrid[0:h, 0:w].astype(np.float64)

        def pts(A):
            q = A[2, 0] * x + A[2, 1] * y + A[2, 2]
            return np.stack([(A[0, 0] * x + A[0, 1] * y + A[0, 2]) / q, (A[1, 0] * x + A[1, 1] * y + A[1, 2]) / q], -1)

        for k in range(n):
            dist = float(np.linalg.norm(pts(got[k]) - pts(H), axis=-1).mean())
            interior = ndimage.binary_erosion(rect[k], iterations=8)
            moving = float((mask[k][interior] == 1).mean())
            back = ~ndimage.binary_dilation(rect[k], iterations=8)
            still = float((mask[k][back] == 0).mean())
            figures["ch%d_pair%d" % (ch, k)] = dict(reprojection_px=dist, rect_moving=moving, background_still=still,
                                                    status=int(stats[k]["status"]), inliers=int(stats[k]["n_inliers"]),
                                                    corr=int(stats[k]["n_corr"]))
    print(json.dumps(figures, indent=1))
    # The fit lands 0.10-0.11 px (mean over the frame) from the true motion on an H100: DIS at operating point 2
    # computes the flow two levels below full resolution and upsamples it bilinearly, which biases the flow near the
    # frame's border and the rectangle's edges by about that much (DESIGN.md section 5.18), so the bound is 0.15 px.
    for k, f in figures.items():
        assert f["status"] == 0, (k, f)
        assert f["reprojection_px"] < 0.15, (k, f)
        assert f["rect_moving"] >= 0.9, (k, f)
        assert f["background_still"] >= 0.95, (k, f)


def test_lists_longer_than_two_score_tiles(api):
    """At step 1 on 128 x 160 frames every pair has more than 8192 correspondences, so the score kernel refills each of
    its two 4096-entry buffers at least once."""
    h, w, n = 128, 160, 2
    prm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=1, nop=2)
    clip = synth.synthetic_sequence(n + 1, h, w, 1, seed=53, amp=3.0)
    ctx = context(api, prm, h, w, 2 * n)
    ctx.upload_sequence_bidir_u8(0, n, clip, w, h)
    ctx.run(2 * n)
    flows = fullres(ctx, 0, 2 * n, h, w)
    for model in MODELS:
        for fbc in (0, 1):
            p = mp(model, step=1, fb_check=fbc, hypotheses=96)
            got = call(ctx, 0, n, p, w, h, b0=n if fbc else None, i1=clip[1:], outs=outputs(n, h, w, 1))
            same(got, expected(flows, 0, n, n if fbc else None, clip[1:], p), "%s fb_check %d" % (model, fbc))
            assert (got[1]["n_corr"] > 2 * 4096).all(), got[1]
    ctx.close()


@pytest.mark.parametrize("extra", [["--bidirectional"], ["--kitti"]], ids=["flo-bidirectional", "kitti"])
@pytest.mark.parametrize("ch", [1, 3])
def test_batch_command_global_motion(tmp_path, ch, extra, api):
    """A chain of three pairs (the sequence upload) and two unrelated ones (pairs, with --bidirectional plus their
    swapped copies) in batches of three.  --global-motion homography PATH writes PATH lines, <stem>_residual<ext>,
    <stem>_moving.pgm and <stem>_registered.png equal to the Python call on the same flows; every other output keeps
    its bytes."""
    import os
    import subprocess

    from test_interpolate_gpu import _read_png8, _write_png

    from of_dis_b200 import build

    bindir = build.build_host()
    exe = os.path.join(bindir, ("run_OF_INT" if ch == 1 else "run_OF_RGB") + "_batch")
    bidir = "--bidirectional" in extra
    kitti = "--kitti" in extra
    h, w = 150, 250
    clip = synth.global_motion_clip(3, h, w, ch, seed=96, H=synth.similarity_about_centre(h, w, 0.5, 1.01, (3, 0)))[0]
    other = synth.synthetic_sequence(3, h, w, ch, seed=97, amp=3.0)
    paths, imgs = {}, {}
    for name, fr in (("a", clip), ("b", other)):
        for t, img in enumerate(fr):
            paths[name, t] = str(tmp_path / ("%s%d.png" % (name, t)))
            imgs[name, t] = img
            _write_png(paths[name, t], img)
    pairs = [("a", 0), ("a", 1), ("a", 2), ("b", 1), ("b", 0)]
    outs = {}
    oext = "png" if kitti else "flo"
    gm_path = str(tmp_path / "motion.txt")
    for tag in ("plain", "gm"):
        outs[tag] = [str(tmp_path / ("%s%d.%s" % (tag, k, oext))) for k in range(len(pairs))]
        lst = tmp_path / ("%s.txt" % tag)
        lst.write_text("".join("%s %s %s\n" % (paths[nm, t], paths[nm, t + 1], outs[tag][k])
                               for k, (nm, t) in enumerate(pairs)))
        opts = extra + (["--global-motion", "homography", gm_path] if tag == "gm" else [])
        r = subprocess.run([exe, str(lst), "--batch", "3"] + opts + ["2"], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
    with_suffix = lambda p, s, e=None: os.path.splitext(p)[0] + s + (e or os.path.splitext(p)[1])  # noqa: E731
    prm = params.operating_point(2, w, noc=ch)
    bgr = (lambda a: a[..., ::-1]) if ch == 3 else (lambda a: a)  # the decoder holds BGR
    p = mp("homography", step=8, fb_check=int(bidir), hypotheses=1024, threshold=1.0, refine=3, seed=0)
    lines = open(gm_path).read().splitlines()
    assert len(lines) == len(pairs)
    pgm = {0: 0, 1: 255, 2: 128}
    for b0, b1, layout in ((0, 3, "sequence"), (3, 5, "pairs")):
        n = b1 - b0
        i0 = np.ascontiguousarray(np.stack([bgr(imgs[pairs[k]]) for k in range(b0, b1)]))
        i1 = np.ascontiguousarray(np.stack([bgr(imgs[pairs[k][0], pairs[k][1] + 1]) for k in range(b0, b1)]))
        ctx = context(api, prm, h, w, 2 * n)
        if layout == "sequence":
            ctx.upload_sequence_bidir_u8(0, n, np.concatenate([i0, i1[-1:]]), w, h)
        else:
            pr = np.ascontiguousarray(np.stack([i0, i1], 1))
            ctx.upload_frames_u8(0, 2 * n, np.ascontiguousarray(np.concatenate([pr, pr[:, ::-1]])), w, h)
        ctx.run(2 * n)
        o = outputs(n, h, w, ch)
        models, stats = ctx.global_motion_fullres(0, n, p, width_org=w, height_org=h, b0=n if bidir else None, i1=i1,
                                                  **o)
        ctx.close()
        for k in range(b0, b1):
            q = k - b0
            want = " ".join([os.path.splitext(outs["gm"][k])[0]] + ["%.17g" % v for v in models[q].reshape(-1)] +
                            ["%d" % stats[q][f] for f in ("status", "n_corr", "n_inliers")])
            assert lines[k] == want, (lines[k], want)
            res = o["residual"][q]
            f = with_suffix(outs["gm"][k], "_residual")
            if kitti:
                assert np.array_equal(preprocess.read_kitti_png(f), preprocess.encode_kitti(res)), k
            else:
                assert (preprocess.read_flo(f).view(np.uint32) == res.view(np.uint32)).all(), k
            mv = open(with_suffix(outs["gm"][k], "_moving", ".pgm"), "rb").read()
            assert mv == b"P5\n%d %d\n255\n" % (w, h) + np.vectorize(pgm.get)(o["mask"][q]).astype(np.uint8).tobytes()
            reg = _read_png8(with_suffix(outs["gm"][k], "_registered", ".png"))
            assert np.array_equal(reg, bgr(o["registered"][q])), k
        assert (stats["status"] == 0).all(), stats
    for k in range(len(pairs)):
        for suffix in [""] + (["_bw", "_occ"] if bidir else []):
            e = ".pgm" if suffix == "_occ" else None
            assert open(with_suffix(outs["plain"][k], suffix, e), "rb").read() == \
                open(with_suffix(outs["gm"][k], suffix, e), "rb").read(), (k, suffix)
        for suffix, e in (("_residual", None), ("_moving", ".pgm"), ("_registered", ".png")):
            assert not os.path.exists(with_suffix(outs["plain"][k], suffix, e))
