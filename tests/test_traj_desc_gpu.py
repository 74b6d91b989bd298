"""Trajectory descriptors on the device: ofdis_traj_begin / ofdis_traj_advance / ofdis_traj_stats_get.  Every record,
descriptor float, count and counter must be BITWISE what preprocess.traj_descriptors gives on
ofdis_get_flow_fullres's flows of the same slots, and the tracks bitwise those of ofdis_track_advance."""
import ctypes
import json

import numpy as np
import pytest
from scipy import ndimage

from of_dis_b200 import params, preprocess, synth

pytestmark = pytest.mark.gpu

f32 = np.float32
SMALL = "3 %d 8 8 0.05 0.95 0 8 0.4 %d 1 0 1 10 10 5 1 3 1.6 0"
SHORT = dict(preprocess.TRAJ_DEFAULTS, L=4, nt=2, N=16, ns=4, min_disp=0.5)


def track_params(**kw):
    p = dict(capacity=4000, spacing=6, alpha=0.01, beta=0.5, mb_alpha=0.01, mb_beta=0.002, min_eig=25.0)
    p.update(kw)
    return p


def same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def assert_result(got, exp, name):
    """got: (lists, records, desc, n_desc) of Context.traj_advance; exp the same of TrajStream.advance."""
    assert len(got[0]) == len(exp[0]), name
    for k, (g, e) in enumerate(zip(got[0], exp[0])):
        assert same(g, e), "%s: list %d differs" % (name, k)
    assert np.array_equal(got[3], exp[3]), (name, got[3], exp[3])
    assert same(got[1], exp[1]), "%s: records differ" % name
    assert same(got[2], exp[2]), "%s: descriptors differ" % name


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


def two_way_context(api, layout, ch, fb, h, w, n, seed):
    """Slots 1 .. n hold the forward pairs of a clip and n+1 .. 2n their backward partners (slots 0 and 2n+1 hold
    unrelated pairs).  Returns (ctx, clip, the frames as traj_advance takes image2 of slot 1 + k, all flows)."""
    prm = params.from_cli_numbers((SMALL % (1, fb)).split(), noc=ch, nop=2)
    clip = synth.synthetic_sequence(n + 1, h, w, ch, seed=seed, amp=3.0)
    other = synth.synthetic_sequence(2, h, w, ch, seed=seed + 1, amp=3.0)
    ctx = context(api, prm, h, w, 2 * n + 2)
    ctx.upload_frames_u8(0, 1, np.ascontiguousarray(other[None]), w, h)
    if layout == "sequence":
        ctx.upload_sequence_bidir_u8(1, n, clip, w, h)
        image2 = clip[1:]
    else:  # the pairs, then their swapped copies, as the batch command uploads them
        pairs = np.ascontiguousarray(np.stack([clip[:-1], clip[1:]], 1))
        ctx.upload_frames_u8(1, n + 1, pairs, w, h)
        ctx.upload_frames_u8(n + 1, 2 * n + 1, np.ascontiguousarray(pairs[:, ::-1]), w, h)
        ctx.set_swapped_slots(n + 1, 2 * n + 1, 1)
        image2 = pairs[:, 1]
    ctx.upload_frames_u8(2 * n + 1, 2 * n + 2, np.ascontiguousarray(other[::-1][None]), w, h)
    ctx.run(2 * n + 2)
    return ctx, clip, image2, fullres(ctx, 0, 2 * n + 2, h, w)


def make_models(kind, n, h, w, rng):
    if kind == "none":
        return None
    m = np.stack([synth.similarity_about_centre(h, w, rng.normal(0, 0.3), 1 + rng.normal(0, 0.003),
                                                tuple(rng.normal(0, 1.5, 2))).reshape(9) for _ in range(n)])
    if kind == "nan":
        m[::2] = np.nan
        m[1::4, 8] = 0.0
    return m


CASES = [  # ch, layout, fb, size, models, traj params
    (1, "sequence", 0, (128, 256), "none", "default"),
    (3, "pairs", 1, (121, 203), "fitted", "default"),
    (1, "pairs", 0, (121, 203), "nan", "short"),
    (3, "sequence", 1, (128, 256), "fitted", "short"),
    (1, "sequence", 1, (121, 203), "fitted", "default"),
    (3, "pairs", 0, (128, 256), "none", "short"),
]


@pytest.mark.parametrize("ch,layout,fb,size,models,tp", CASES,
                         ids=["-".join(map(str, c[:3])) + "-%dx%d-%s-%s" % (c[3] + c[4:]) for c in CASES])
def test_descriptors_equal_the_restatement(ch, layout, fb, size, models, tp, api):
    """Host memory; the whole clip in one call (f0 = 1, b0 = f1), then the same clip in three calls; the tracks are
    track_advance's, and the flows of every slot stay as they were."""
    h, w = size
    p = preprocess.TRAJ_DEFAULTS if tp == "default" else SHORT
    n = 2 * p["L"] + 2
    ctx, clip, image2, flows = two_way_context(api, layout, ch, fb, h, w, n, seed=31)
    tpp = track_params()
    M = make_models(models, n, h, w, np.random.default_rng(5))
    F, B = flows[1:n + 1], flows[n + 1:2 * n + 1]
    s = preprocess.TrajStream(tpp, p)
    first = s.begin(clip[0])
    exp = s.advance(clip[1:], F, B, M)
    assert exp[1].size > 0 and int(exp[3].sum()) == exp[1].size
    got0 = ctx.traj_begin(tpp, p, clip[0], w, h)
    assert same(got0, first)
    before = ctx.launch_count
    got = ctx.traj_advance(1, n + 1, n + 1, image2, w, h, models=M)
    assert ctx.launch_count - before == 10 * n
    assert_result(got, exp, "one call")
    assert ctx.traj_stats() == s.tstats
    assert ctx.track_stats() == s.track_stats()
    assert got[2].shape[1] == preprocess.traj_dim(p)
    # the tracks are the plain tracker's
    tl = [ctx.track_begin(tpp, clip[0], w, h)] + ctx.track_advance(1, n + 1, n + 1, image2, w, h)
    for a, b in zip(tl, [first] + got[0]):
        assert same(a, b)
    # three calls
    ctx.traj_begin(tpp, p, clip[0], w, h)
    cuts = [0, 1, p["L"] + 1, n]
    parts = [ctx.traj_advance(1 + a, 1 + b, n + 1 + a, image2[a:b], w, h, models=None if M is None else M[a:b])
             for a, b in zip(cuts[:-1], cuts[1:])]
    joined = (sum((q[0] for q in parts), []), np.concatenate([q[1] for q in parts]),
              np.concatenate([q[2] for q in parts]), np.concatenate([q[3] for q in parts]))
    assert_result(joined, exp, "three calls")
    assert ctx.traj_stats() == s.tstats
    assert np.array_equal(fullres(ctx, 0, 2 * n + 2, h, w).view(np.uint32), flows.view(np.uint32))
    ctx.close()


@pytest.mark.parametrize("layout", ["sequence", "pairs"])
def test_device_memory_on_a_caller_stream(layout, api):
    import torch

    h, w, n, ch = 121, 203, 6, 3
    p = SHORT
    stream = torch.cuda.Stream()
    prm = params.from_cli_numbers((SMALL % (0, 0)).split(), noc=ch, nop=2)
    clip = synth.synthetic_sequence(n + 1, h, w, ch, seed=41, amp=3.0)
    ctx = context(api, prm, h, w, 2 * n, stream=stream.cuda_stream)
    hwc = h * w * ch
    if layout == "sequence":
        dev = torch.from_numpy(clip.reshape(-1)).cuda()
        ctx.upload_sequence_bidir_u8(0, n, clip, w, h)
        p1, stride = dev.data_ptr() + hwc, hwc
    else:
        pairs = np.ascontiguousarray(np.stack([clip[:-1], clip[1:]], 1))
        dev = torch.from_numpy(pairs.reshape(-1)).cuda()
        ctx.upload_frames_u8(0, n, pairs, w, h)
        ctx.upload_frames_u8(n, 2 * n, np.ascontiguousarray(pairs[:, ::-1]), w, h)
        ctx.set_swapped_slots(n, 2 * n, 1)
        p1, stride = dev.data_ptr() + hwc, 2 * hwc
    ctx.run(2 * n)
    flows = fullres(ctx, 0, 2 * n, h, w)
    tpp = track_params(capacity=3000)
    M = make_models("fitted", n, h, w, np.random.default_rng(6))
    s = preprocess.TrajStream(tpp, p)
    s.begin(clip[0])
    exp = s.advance(clip[1:], flows[:n], flows[n:], M)
    cap = tpp["capacity"]
    bound, dim = preprocess.traj_bound(cap, n, p["L"]), preprocess.traj_dim(p)
    pts = torch.full((n * cap * 3,), -7, dtype=torch.int32, device="cuda")
    rec = torch.full((bound * 7,), -7, dtype=torch.int32, device="cuda")
    desc = torch.full((bound * dim,), -7.0, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    ctx.traj_begin(tpp, p, dev.data_ptr(), w, h, memkind=api.MEM_DEVICE, points=pts.data_ptr())
    counts, n_desc = ctx.traj_advance(0, n, n, p1, w, h, models=M, frame_stride=stride, memkind=api.MEM_DEVICE,
                                      points=pts.data_ptr(), records=rec.data_ptr(), desc=desc.data_ptr())
    stream.synchronize()
    allp = pts.cpu().numpy().view(preprocess.TRACK_POINT_DTYPE)
    total = int(n_desc.sum())
    got = ([allp[k * cap:k * cap + counts[k]] for k in range(n)],
           rec.cpu().numpy().view(preprocess.TRAJ_RECORD_DTYPE)[:total],
           desc.cpu().numpy().reshape(bound, dim)[:total], n_desc)
    assert total > 0
    assert_result(got, exp, "device")
    assert ctx.traj_stats() == s.tstats
    ctx.close()


def test_graph_mode_and_a_run_between_calls(api):
    h, w, n = 128, 256, 10
    ctx, clip, image2, flows = two_way_context(api, "sequence", 1, 0, h, w, n, seed=51)
    ctx.set_graph_mode(True)
    ctx.run(2 * n + 2)
    ctx.run(2 * n + 2)  # a replay
    tpp, p = track_params(), SHORT
    s = preprocess.TrajStream(tpp, p)
    s.begin(clip[0])
    exp = s.advance(clip[1:], flows[1:n + 1], flows[n + 1:2 * n + 1])
    for _ in range(2):
        ctx.traj_begin(tpp, p, clip[0], w, h)
        assert_result(ctx.traj_advance(1, n + 1, n + 1, image2, w, h), exp, "graph mode")
    ctx.traj_begin(tpp, p, clip[0], w, h)
    a = ctx.traj_advance(1, 4, n + 1, image2[:3], w, h)
    ctx.run(2 * n + 2)
    b = ctx.traj_advance(4, n + 1, n + 4, image2[3:], w, h)
    joined = (a[0] + b[0], np.concatenate([a[1], b[1]]), np.concatenate([a[2], b[2]]), np.concatenate([a[3], b[3]]))
    assert_result(joined, exp, "across a run")
    ctx.close()


@pytest.mark.parametrize("sc_l", [0, 1])
def test_extreme_level_flows_and_capacity_overflow(sc_l, api):
    """Level flows set directly: NaN, +-inf, values beyond 1e9; then a capacity that drops seeds."""
    h, w, n = 96, 160, 9
    prm = params.from_cli_numbers((SMALL % (sc_l, 0)).split(), noc=1, nop=2)
    ctx = context(api, prm, h, w, 2 * n)
    hl, wl = h >> sc_l, w >> sc_l
    rng = np.random.default_rng(61)
    for k in range(n):
        F = (rng.normal(0, 0.7, (hl, wl, 2)) + np.array([1.2, -0.6])).astype(f32)
        m = rng.random((hl, wl))
        F[m < 0.01, 0] = np.nan
        F[(m >= 0.01) & (m < 0.02), 1] = np.inf
        F[(m >= 0.02) & (m < 0.03), 0] = -np.inf
        F[(m >= 0.03) & (m < 0.04), 1] = 3e9
        B = -F + rng.normal(0, 0.05, F.shape).astype(f32)
        ctx.set_flow(k, sc_l, F)
        ctx.set_flow(n + k, sc_l, B)
    flows = fullres(ctx, 0, 2 * n, h, w)
    clip = synth.synthetic_sequence(n + 1, h, w, 1, seed=62)
    M = make_models("nan", n, h, w, rng)
    for cap in (5000, 60):
        tpp = track_params(capacity=cap, spacing=3, min_eig=4.0, alpha=0.5, beta=2.0, mb_alpha=1.0, mb_beta=5.0)
        s = preprocess.TrajStream(tpp, SHORT)
        s.begin(clip[0])
        exp = s.advance(clip[1:], flows[:n], flows[n:], M)
        ctx.traj_begin(tpp, SHORT, clip[0], w, h)
        assert_result(ctx.traj_advance(0, n, n, clip[1:], w, h, models=M), exp, "capacity %d" % cap)
        assert ctx.traj_stats() == s.tstats and ctx.track_stats() == s.track_stats()
        assert s.tstats["emitted"] > 0
        if cap == 60:
            assert s.stats["dropped"] > 0
    ctx.close()


def test_bad_arguments(api):
    import torch

    h, w, n = 128, 256, 2
    prm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=1, nop=2)
    ctx = context(api, prm, h, w, 2 * n)
    clip = synth.synthetic_sequence(n + 1, h, w, 1, seed=71)
    ctx.upload_sequence_bidir_u8(0, n, clip, w, h)
    ctx.run(2 * n)
    L = api.lib()
    tpp, good = track_params(), dict(SHORT)
    cap = tpp["capacity"]
    bound = preprocess.traj_bound(cap, n, good["L"])
    pts = np.zeros(n * cap, preprocess.TRACK_POINT_DTYPE)
    rec = np.zeros(bound, preprocess.TRAJ_RECORD_DTYPE)
    desc = np.zeros((bound, preprocess.traj_dim(good)), f32)
    dev = torch.zeros((1 << 20,), dtype=torch.int32, device="cuda")
    counts, n_desc = np.zeros(n, np.int32), np.zeros(n, np.int32)
    count = ctypes.c_int(0)
    frame = clip.ctypes.data_as(ctypes.c_void_p)
    tp = api.TrackParams(*[tpp[k] for k in preprocess.TRACK_PARAM_FIELDS])
    P = api._ptr

    def begin(ctx_=ctx, **kw):
        q = api.TrajParams(*[dict(good, **kw)[k] for k in preprocess.TRAJ_PARAM_FIELDS])
        return L.ofdis_traj_begin(ctx_._h, ctypes.byref(tp), ctypes.byref(q), frame, P(pts), ctypes.byref(count), w, h,
                                  api.MEM_HOST)

    def advance(f0=0, f1=n, b0=n, fr=ctypes.c_void_p(clip.ctypes.data + h * w), stride=h * w, pt=P(pts),
                cnt=P(counts), r=P(rec), d=P(desc), nd=P(n_desc), mem=api.MEM_HOST):
        return L.ofdis_traj_advance(ctx._h, f0, f1, b0, fr, stride, None, pt, cnt, r, d, nd, w, h, mem)

    def stats_ok():
        return L.ofdis_traj_stats_get(ctx._h, ctypes.byref(api.TrajStats())) == 0

    assert advance() == -1 and not stats_ok()
    nan, inf = float("nan"), float("inf")
    bad = [dict(L=0), dict(L=65), dict(nt=0), dict(L=5, nt=2), dict(ns=0), dict(ns=5), dict(N=0), dict(N=18, ns=4),
           dict(N=w + 8, ns=1), dict(N=h + 4), dict(min_flow=nan), dict(eps=0.0), dict(eps=inf), dict(min_disp=-1.0),
           dict(min_disp=nan), dict(min_var=inf), dict(max_var=nan), dict(max_dis=-inf)]
    before = ctx.launch_count
    for kw in bad:
        assert begin(**kw) == -1, kw
    assert L.ofdis_traj_begin(ctx._h, ctypes.byref(tp), None, frame, P(pts), ctypes.byref(count), w, h, 0) == -1
    assert ctx.launch_count == before
    assert begin() == 0 and stats_ok()
    bad_adv = [dict(f0=-1), dict(f1=2 * n + 1), dict(f0=1, f1=1), dict(b0=n + 1), dict(fr=None), dict(pt=None),
               dict(cnt=None), dict(r=None), dict(d=None), dict(nd=None), dict(stride=h * w - 1),
               dict(fr=ctypes.c_void_p(dev.data_ptr()), pt=ctypes.c_void_p(dev.data_ptr()),
                    r=ctypes.c_void_p(dev.data_ptr() + 2), d=ctypes.c_void_p(dev.data_ptr()), mem=api.MEM_DEVICE),
               dict(fr=ctypes.c_void_p(dev.data_ptr()), pt=ctypes.c_void_p(dev.data_ptr()),
                    r=ctypes.c_void_p(dev.data_ptr()), d=ctypes.c_void_p(dev.data_ptr() + 1), mem=api.MEM_DEVICE)]
    before = ctx.launch_count
    for kw in bad_adv:
        assert advance(**kw) == -1, kw
    assert ctx.launch_count == before and stats_ok()
    assert L.ofdis_traj_stats_get(ctx._h, None) == -1
    # a refused call leaves the stage as it was
    flows = fullres(ctx, 0, 2 * n, h, w)
    s = preprocess.TrajStream(tpp, good)
    s.begin(clip[0])
    exp = s.advance(clip[1:], flows[:n], flows[n:])
    assert advance() == 0
    assert np.array_equal(n_desc, exp[3]) and ctx.traj_stats() == s.tstats
    # track_begin and track_advance end the stage
    ctx.track_begin(tpp, clip[0], w, h)
    assert advance() == -1 and not stats_ok()
    assert begin() == 0
    ctx.track_advance(0, 1, n, clip[1:2], w, h)
    assert advance() == -1 and not stats_ok()
    ctx.close()
    # a stereo context
    sctx = context(api, params.from_cli_numbers((SMALL % (1, 0)).split(), noc=1, nop=1), h, w, 2)
    assert begin(sctx) == -1
    sctx.close()


def test_a_refused_begin_keeps_the_live_stage(api):
    """A traj_begin the library refuses leaves the previous stage live, and Context.traj_advance keeps sizing its host
    outputs by that stage's parameters."""
    h, w, n = 128, 256, 10
    ctx, clip, image2, flows = two_way_context(api, "sequence", 1, 0, h, w, n, seed=57)
    tpp, p = track_params(), SHORT
    s = preprocess.TrajStream(tpp, p)
    s.begin(clip[0])
    exp = s.advance(clip[1:], flows[1:n + 1], flows[n + 1:2 * n + 1])
    ctx.traj_begin(tpp, p, clip[0], w, h)
    a = ctx.traj_advance(1, 4, n + 1, image2[:3], w, h)
    with pytest.raises(api.OfdisError):
        ctx.traj_begin(track_params(capacity=9000), dict(preprocess.TRAJ_DEFAULTS, eps=0.0), clip[0], w, h)
    b = ctx.traj_advance(4, n + 1, n + 4, image2[3:], w, h)
    joined = (a[0] + b[0], np.concatenate([a[1], b[1]]), np.concatenate([a[2], b[2]]), np.concatenate([a[3], b[3]]))
    assert_result(joined, exp, "after a refused begin")
    assert exp[1].size > 0 and b[2].shape[1] == preprocess.traj_dim(p)
    ctx.close()


def test_end_to_end_on_a_camera_motion_clip(api):
    """DIS flows at operating point 2 and fitted homographies on synth.global_motion_clip (a camera similarity and a
    rectangle that moves on its own) over 2L + 1 frames: the restatement's bits, and the descriptors' purpose --
    compensated, the background's segments are dropped as camera motion and the rectangle's are emitted."""
    h, w = 218, 512
    L = preprocess.TRAJ_DEFAULTS["L"]
    n = 2 * L + 1
    H = synth.similarity_about_centre(h, w, 0.3, 1.003, (1.5, 0.5))
    figures = {}
    for ch in (1, 3):
        clip, _, rect = synth.global_motion_clip(n, h, w, ch, seed=9, H=H)
        prm = params.operating_point(2, w, noc=ch)
        ctx = context(api, prm, h, w, 2 * n)
        ctx.upload_sequence_bidir_u8(0, n, clip, w, h)
        ctx.run(2 * n)
        mp = dict(model=3, step=8, fb_check=1, alpha=0.01, beta=0.5, hypotheses=1024, threshold=1.0, refine=3, seed=11)
        models, stats = ctx.global_motion_fullres(0, n, mp, width_org=w, height_org=h, b0=n)
        assert (stats["status"] == 0).all()
        flows = fullres(ctx, 0, 2 * n, h, w)
        tpp = track_params(capacity=20000, spacing=8)
        for comp in (True, False):
            M = models.reshape(n, 9) if comp else None
            s = preprocess.TrajStream(tpp, preprocess.TRAJ_DEFAULTS)
            s.begin(clip[0])
            exp = s.advance(clip[1:], flows[:n], flows[n:], M)
            ctx.traj_begin(tpp, preprocess.TRAJ_DEFAULTS, clip[0], w, h)
            got = ctx.traj_advance(0, n, n, clip[1:], w, h, models=M)
            assert_result(got, exp, "ch %d comp %s" % (ch, comp))
            recs = got[1]
            # a segment belongs to the rectangle or the background by its mean position in its middle frame
            fg = bg = 0
            for r in recs:
                t = min(int(r["start"]) + L // 2, n - 1)
                inner = ndimage.binary_erosion(rect[t], iterations=16)
                back = ~ndimage.binary_dilation(rect[t], iterations=16)
                x, y = min(int(round(float(r["mean_x"]))), w - 1), min(int(round(float(r["mean_y"]))), h - 1)
                fg += bool(inner[y, x])
                bg += bool(back[y, x])
            figures["ch%d_%s" % (ch, "comp" if comp else "raw")] = dict(ctx.traj_stats(), segments=int(recs.size),
                                                                         rect_segments=fg, background_segments=bg)
        ctx.close()
    print(json.dumps(figures, indent=1))
    # Measured on an H100: compensated, 27 (gray) and 16 (RGB) of the 2368 and 2348 background segments remain (1.1 %
    # and 0.7 %), and all 294 and 289 rectangle segments are emitted with and without models.  Asserted with margins:
    # at most 5 % of the background, at least 90 % of the rectangle.
    for ch in (1, 3):
        comp, raw = figures["ch%d_comp" % ch], figures["ch%d_raw" % ch]
        assert raw["background_segments"] > 0.5 * raw["segments"], raw
        assert comp["background_segments"] <= 0.05 * raw["background_segments"], (comp, raw)
        assert comp["rect_segments"] >= 0.9 * raw["rect_segments"] > 0, (comp, raw)


# ---- batch front-end --------------------------------------------------------------------------------------------
def _read_desc(path):
    lines = open(path).read().splitlines()
    assert lines[0] == "# clip id start mean_x mean_y sd_x sd_y length d0 .. d425"
    out = {}
    for ln in lines[1:]:
        f = ln.split()
        assert len(f) == 8 + 426, len(f)
        rec = np.zeros(1, preprocess.TRAJ_RECORD_DTYPE)
        rec["id"], rec["start"] = int(f[1]), int(f[2])
        for k, v in zip(("mean_x", "mean_y", "sd_x", "sd_y", "length"), f[3:8]):
            rec[k] = f32(float(v))
        r, d = out.setdefault(int(f[0]), ([], []))
        r.append(rec)
        d.append(np.array([f32(float(v)) for v in f[8:]], f32))
    return {c: (np.concatenate(r), np.stack(d)) for c, (r, d) in out.items()}


@pytest.mark.parametrize("exe,ch,gm", [("run_OF_INT", 1, False), ("run_OF_RGB", 3, True)],
                         ids=["gray", "rgb-global-motion"])
def test_batch_command_descriptors(tmp_path, exe, ch, gm, api):
    """A 17-frame clip (16 pairs, split by batches of 5) and a one-pair clip.  --descriptors writes the Python call's
    records and descriptors clip for clip (with the --global-motion models when given); --tracks and every other output
    keep their bytes."""
    import os
    import subprocess

    from of_dis_b200 import build

    from test_traj_desc import _write_png

    bindir = build.build_host()
    h, w = 96, 160
    clip = synth.global_motion_clip(16, h, w, ch, seed=98, H=synth.similarity_about_centre(h, w, 0.2, 1.0, (1.2, 0.4)))[0]
    other = synth.synthetic_sequence(2, h, w, ch, seed=99, amp=3.0)
    paths, imgs = {}, {}
    for name, fr in (("a", clip), ("b", other)):
        for t, img in enumerate(fr):
            paths[name, t] = str(tmp_path / ("%s%d.png" % (name, t)))
            imgs[name, t] = img
            _write_png(paths[name, t], img)
    pairs = [("a", t) for t in range(16)] + [("b", 0)]
    clips = [list(range(16)), [16]]
    gm_opt = ["--global-motion", "homography"] if gm else []
    outs, logs = {}, {}
    for tag in ("plain", "desc"):
        outs[tag] = [str(tmp_path / ("%s%d.flo" % (tag, k))) for k in range(len(pairs))]
        lst = tmp_path / ("%s.txt" % tag)
        lst.write_text("".join("%s %s %s\n" % (paths[nm, t], paths[nm, t + 1], outs[tag][k])
                               for k, (nm, t) in enumerate(pairs)))
        opts = ["--tracks", str(tmp_path / ("tracks_%s.txt" % tag))]
        opts += (gm_opt + [str(tmp_path / ("gm_%s.txt" % tag))]) if gm else []
        opts += ["--descriptors", str(tmp_path / "desc.txt")] if tag == "desc" else []
        r = subprocess.run([os.path.join(bindir, exe + "_batch"), str(lst), "--batch", "5"] + opts + ["2"],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        logs[tag] = r.stdout
    got = _read_desc(str(tmp_path / "desc.txt"))
    prm = params.operating_point(2, w, noc=ch, nop=2)
    bgr = (lambda a: a[..., ::-1]) if ch == 3 else (lambda a: a)  # the decoder holds BGR
    tp = dict(capacity=4 * ((w + 7) // 8) * ((h + 7) // 8), spacing=8, alpha=0.01, beta=0.5, mb_alpha=0.01,
              mb_beta=0.002, min_eig=25.0)
    total = dict.fromkeys(preprocess.TRAJ_STATS_FIELDS, 0)
    for c, ks in enumerate(clips):
        fr = [bgr(imgs[pairs[ks[0]]])] + [bgr(imgs[pairs[k][0], pairs[k][1] + 1]) for k in ks]
        fr = np.ascontiguousarray(np.stack(fr))
        n = len(ks)
        ctx = context(api, prm, h, w, 2 * n)
        ctx.upload_sequence_bidir_u8(0, n, fr, w, h)
        ctx.run(2 * n)
        M = None
        if gm:
            mp = dict(model=3, step=8, fb_check=0, alpha=0.01, beta=0.5, hypotheses=1024, threshold=1.0, refine=3,
                      seed=0)
            M = ctx.global_motion_fullres(0, n, mp, width_org=w, height_org=h, b0=n)[0].reshape(n, 9)
        ctx.traj_begin(tp, preprocess.TRAJ_DEFAULTS, fr[0], w, h)
        _, recs, desc, _ = ctx.traj_advance(0, n, n, fr[1:], w, h, models=M)
        st = ctx.traj_stats()
        ctx.close()
        for k in total:
            total[k] += st[k]
        g = got.get(c, (np.zeros(0, preprocess.TRAJ_RECORD_DTYPE), np.zeros((0, 426), f32)))
        assert same(g[0], recs), (c, g[0].size, recs.size)
        assert same(g[1], desc), c
    assert total["emitted"] > 0
    line = [ln for ln in logs["desc"].splitlines() if ln.startswith("DESCRIPTORS")]
    assert line == ["DESCRIPTORS clips 2 emitted %d static %d erratic %d jump %d camera %d"
                    % tuple(total[k] for k in preprocess.TRAJ_STATS_FIELDS)], logs["desc"]
    # the tracks, the models and every per-pair output keep their bytes
    assert open(tmp_path / "tracks_plain.txt", "rb").read() == open(tmp_path / "tracks_desc.txt", "rb").read()
    assert [ln for ln in logs["plain"].splitlines() if ln.startswith("TRACKS")] == \
        [ln for ln in logs["desc"].splitlines() if ln.startswith("TRACKS")]
    with_suffix = lambda q, s, e=None: os.path.splitext(q)[0] + s + (e or os.path.splitext(q)[1])  # noqa: E731
    if gm:
        a = open(tmp_path / "gm_plain.txt").read().replace(str(tmp_path / "plain"), "")
        b = open(tmp_path / "gm_desc.txt").read().replace(str(tmp_path / "desc"), "")
        assert a == b
    for k in range(len(pairs)):
        others = [("", None)] + ([("_residual", None), ("_moving", ".pgm"), ("_registered", ".png")] if gm else [])
        for suffix, e in others:
            assert open(with_suffix(outs["plain"][k], suffix, e), "rb").read() == \
                open(with_suffix(outs["desc"][k], suffix, e), "rb").read(), (k, suffix)
