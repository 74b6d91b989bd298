"""Dense point tracking on the device: ofdis_track_begin / ofdis_track_advance / ofdis_track_stats_get.  Every record,
count and counter must be BITWISE what preprocess.track_points gives on ofdis_get_flow_fullres's flows of the same
slots; the batch command's --tracks file must be the Python call's tracks and leave every other output as it is."""
import ctypes
import os
import struct
import subprocess
import zlib

import numpy as np
import pytest

from of_dis_b200 import params, preprocess, synth

pytestmark = pytest.mark.gpu

f32 = np.float32
SMALL = "3 %d 8 8 0.05 0.95 0 8 0.4 %d 1 0 1 10 10 5 1 3 1.6 0"


def track_params(nop, **kw):
    p = dict(capacity=4000, spacing=4, alpha=0.01 if nop == 2 else 0.0, beta=0.5 if nop == 2 else 1.0, mb_alpha=0.01,
             mb_beta=0.002, min_eig=25.0)
    p.update(kw)
    return p


def assert_lists(got, exp, name):
    assert len(got) == len(exp), (name, len(got), len(exp))
    for k, (g, e) in enumerate(zip(got, exp)):
        assert g.dtype == preprocess.TRACK_POINT_DTYPE and g.shape == e.shape, (name, k, g.shape, e.shape)
        assert np.array_equal(g.view(np.uint8), e.view(np.uint8)), "%s: list %d differs" % (name, k)


@pytest.fixture(scope="module")
def api():
    from of_dis_b200 import api as _api

    _api.lib()
    return _api


def context(api, prm, h, w, max_frames, stream=None):
    scf = 1 << prm.sc_f
    W, H = (w + scf - 1) // scf * scf, (h + scf - 1) // scf * scf
    return api.Context(prm, W, H, prm.p_samp_s, max_frames, stream=stream)


def fullres(ctx, f0, f1, h, w, nop):
    out = np.empty((f1 - f0, h, w, nop), np.float32)
    ctx.get_flow_fullres(f0, f1, out, w, h)
    ctx.sync()
    return out


def two_way_context(api, layout, nop, ch, fb, h, w, n, seed, graph=False):
    """Slots 1 .. n hold the forward pairs of a clip and n+1 .. 2n their backward partners (slots 0 and 2n+1 hold
    unrelated pairs).  Returns (ctx, clip, the frames as track_advance takes image2 of slot 1 + k, all flows)."""
    prm = params.from_cli_numbers((SMALL % (1, fb)).split(), noc=ch, nop=nop)
    clip = synth.synthetic_sequence(n + 1, h, w, ch, seed=seed, amp=3.0, stereo=(nop == 1))
    other = synth.synthetic_sequence(2, h, w, ch, seed=seed + 1, amp=3.0, stereo=(nop == 1))
    ctx = context(api, prm, h, w, 2 * n + 2)
    if graph:
        ctx.set_graph_mode(True)
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
    return ctx, clip, image2, fullres(ctx, 0, 2 * n + 2, h, w, nop)


@pytest.mark.parametrize("layout", ["sequence", "pairs"])
@pytest.mark.parametrize("fb", [0, 1], ids=["fb0", "fb1"])
@pytest.mark.parametrize("size", [(128, 256), (121, 203)], ids=["div", "nondiv"])
@pytest.mark.parametrize("nop,ch", [(2, 1), (2, 3), (1, 1), (1, 3)])
def test_tracks_equal_the_restatement(nop, ch, size, fb, layout, api):
    """Host memory; the whole clip in one call (f0 = 1, b0 = f1), and from frame 1 in two calls (f0 = 2, b0 = n + 2);
    the flows of every slot stay as they were."""
    h, w = size
    n = 4
    ctx, clip, image2, flows = two_way_context(api, layout, nop, ch, fb, h, w, n, seed=31)
    p = track_params(nop)
    exp, est = preprocess.track_points(clip, flows[1:n + 1], flows[n + 1:2 * n + 1], p)
    assert est["seeded"] > 0 and est["alive"] > 0
    got = [ctx.track_begin(p, clip[0], w, h)]
    before = ctx.launch_count
    got += ctx.track_advance(1, n + 1, n + 1, image2, w, h)
    assert ctx.launch_count - before == 5 * n
    assert_lists(got, exp, "one call")
    assert ctx.track_stats() == est
    # from frame 1, split over two calls
    exp1, est1 = preprocess.track_points(clip[1:], flows[2:n + 1], flows[n + 2:2 * n + 1], p)
    got1 = [ctx.track_begin(p, clip[1], w, h)]
    got1 += ctx.track_advance(2, 3, n + 2, image2[1:2], w, h)
    got1 += ctx.track_advance(3, n + 1, n + 3, image2[2:], w, h)
    assert_lists(got1, exp1, "two calls")
    assert ctx.track_stats() == est1
    assert np.array_equal(fullres(ctx, 0, 2 * n + 2, h, w, nop).view(np.uint32), flows.view(np.uint32))
    ctx.close()


@pytest.mark.parametrize("layout", ["sequence", "pairs"])
@pytest.mark.parametrize("nop,ch", [(2, 3), (1, 1)])
def test_device_memory_on_a_caller_stream(nop, ch, layout, api):
    import torch

    h, w, n = 121, 203, 3
    stream = torch.cuda.Stream()
    prm = params.from_cli_numbers((SMALL % (0, 0)).split(), noc=ch, nop=nop)
    clip = synth.synthetic_sequence(n + 1, h, w, ch, seed=41, amp=3.0, stereo=(nop == 1))
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
    flows = fullres(ctx, 0, 2 * n, h, w, nop)
    p = track_params(nop, capacity=3000)
    exp, est = preprocess.track_points(clip, flows[:n], flows[n:], p)
    cap = p["capacity"]
    pts = torch.full((n * cap * 3,), -7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    c0 = ctx.track_begin(p, dev.data_ptr(), w, h, memkind=api.MEM_DEVICE, points=pts.data_ptr())
    stream.synchronize()
    got = [pts[:c0 * 3].cpu().numpy().view(preprocess.TRACK_POINT_DTYPE)]
    counts = ctx.track_advance(0, n, n, p1, w, h, frame_stride=stride, memkind=api.MEM_DEVICE, points=pts.data_ptr())
    stream.synchronize()
    allp = pts.cpu().numpy().view(preprocess.TRACK_POINT_DTYPE)
    got += [allp[k * cap:k * cap + counts[k]] for k in range(n)]
    assert_lists(got, exp, "device")
    assert ctx.track_stats() == est
    ctx.close()


def test_graph_mode_and_repeated_calls(api):
    """Runs replayed from a graph; a second begin resets the tracker and gives the same bits."""
    h, w, n = 128, 256, 3
    ctx, clip, image2, flows = two_way_context(api, "sequence", 2, 1, 0, h, w, n, seed=51, graph=True)
    ctx.run(2 * n + 2)  # a replay
    p = track_params(2)
    exp, est = preprocess.track_points(clip, flows[1:n + 1], flows[n + 1:2 * n + 1], p)
    for _ in range(2):
        got = [ctx.track_begin(p, clip[0], w, h)] + ctx.track_advance(1, n + 1, n + 1, image2, w, h)
        assert_lists(got, exp, "graph mode")
        assert ctx.track_stats() == est
    # the tracker survives a run
    ctx.track_begin(p, clip[0], w, h)
    ctx.track_advance(1, 2, n + 1, image2[:1], w, h)
    ctx.run(2 * n + 2)
    rest = ctx.track_advance(2, n + 1, n + 2, image2[1:], w, h)
    assert_lists(rest, exp[2:], "across a run")
    ctx.close()


@pytest.mark.parametrize("sc_l", [0, 1])
@pytest.mark.parametrize("nop", [2, 1])
def test_extreme_level_flows_and_capacity_overflow(sc_l, nop, api):
    """Level flows set directly: NaN, +-inf, values beyond 1e9 and out-of-frame moves; then a capacity that drops."""
    h, w, n = 96, 160, 2
    prm = params.from_cli_numbers((SMALL % (sc_l, 0)).split(), noc=1, nop=nop)
    ctx = context(api, prm, h, w, 2 * n)
    hl, wl = h >> sc_l, w >> sc_l
    rng = np.random.default_rng(61)
    for k in range(n):
        F = rng.normal(0, 1.5, (hl, wl, nop)).astype(f32)
        m = rng.random((hl, wl))
        F[m < 0.05, 0] = np.nan
        F[(m >= 0.05) & (m < 0.08), -1] = np.inf
        F[(m >= 0.08) & (m < 0.1), 0] = -np.inf
        F[(m >= 0.1) & (m < 0.12), 0] = 3e9
        F[(m >= 0.12) & (m < 0.2), 0] += w / 3
        B = -F + rng.normal(0, 0.3, F.shape).astype(f32)
        ctx.set_flow(k, sc_l, F)
        ctx.set_flow(n + k, sc_l, B)
    flows = fullres(ctx, 0, 2 * n, h, w, nop)
    clip = synth.synthetic_sequence(n + 1, h, w, 1, seed=62)
    for cap in (5000, 60):
        p = track_params(nop, capacity=cap, spacing=3, min_eig=4.0)
        exp, est = preprocess.track_points(clip, flows[:n], flows[n:], p)
        got = [ctx.track_begin(p, clip[0], w, h)] + ctx.track_advance(0, n, n, clip[1:], w, h)
        assert_lists(got, exp, "capacity %d" % cap)
        assert ctx.track_stats() == est
        assert min(est["ended_leaves"], est["ended_inconsistent"]) > 0
        if cap == 60:
            assert est["dropped"] > 0 and all(len(l) <= cap for l in got)
    assert np.array_equal(fullres(ctx, 0, 2 * n, h, w, nop).view(np.uint32), flows.view(np.uint32))
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
    hwc = h * w
    good = track_params(2)
    pts = np.zeros(n * good["capacity"], preprocess.TRACK_POINT_DTYPE)
    dev = torch.zeros((n * good["capacity"] * 3 + 1,), dtype=torch.int32, device="cuda")
    counts = np.zeros(n, np.int32)
    count = ctypes.c_int(0)
    frame = clip.ctypes.data_as(ctypes.c_void_p)
    pp = pts.ctypes.data_as(ctypes.c_void_p)

    def stats_ok():
        return L.ofdis_track_stats_get(ctx._h, ctypes.byref(api.TrackStats())) == 0

    def begin(fr=frame, pt=pp, cnt=ctypes.byref(count), ww=w, hh=h, mem=api.MEM_HOST, **kw):
        tp = api.TrackParams(*[dict(good, **kw)[k] for k in preprocess.TRACK_PARAM_FIELDS])
        return L.ofdis_track_begin(ctx._h, ctypes.byref(tp), fr, pt, cnt, ww, hh, mem)

    def advance(f0=0, f1=n, b0=n, fr=ctypes.c_void_p(clip.ctypes.data + hwc), stride=hwc, pt=pp,
                cnt=counts.ctypes.data_as(ctypes.c_void_p), ww=w, hh=h, mem=api.MEM_HOST):
        return L.ofdis_track_advance(ctx._h, f0, f1, b0, fr, stride, pt, cnt, ww, hh, mem)

    # before any begin
    assert advance() == -1
    assert not stats_ok()
    nan, inf = float("nan"), float("inf")
    bad_begin = [dict(capacity=0), dict(capacity=(1 << 24) + 1), dict(capacity=-5), dict(spacing=0), dict(spacing=-1),
                 dict(alpha=-1.0), dict(alpha=nan), dict(alpha=inf), dict(beta=-0.1), dict(beta=nan), dict(beta=inf),
                 dict(mb_alpha=-1.0), dict(mb_alpha=nan), dict(mb_alpha=inf), dict(mb_beta=-1.0), dict(mb_beta=nan),
                 dict(mb_beta=inf), dict(min_eig=nan), dict(fr=None), dict(pt=None), dict(cnt=None),
                 dict(ww=w + 8), dict(hh=h - 17), dict(ww=0),
                 dict(fr=ctypes.c_void_p(dev.data_ptr()), pt=ctypes.c_void_p(dev.data_ptr() + 2), mem=api.MEM_DEVICE)]
    before = ctx.launch_count
    for kw in bad_begin:
        assert begin(**kw) == -1, kw
    assert L.ofdis_track_begin(ctx._h, None, frame, pp, ctypes.byref(count), w, h, api.MEM_HOST) == -1
    assert ctx.launch_count == before
    assert begin() == 0 and count.value > 0
    bad_advance = [dict(f0=-1), dict(f1=2 * n + 1), dict(f0=1, f1=1), dict(b0=-1), dict(b0=n + 1), dict(fr=None),
                   dict(pt=None), dict(cnt=None), dict(stride=hwc - 1), dict(ww=w + 8), dict(hh=h - 17),
                   dict(ww=w - 8), dict(fr=ctypes.c_void_p(dev.data_ptr()), pt=ctypes.c_void_p(dev.data_ptr() + 2),
                                         mem=api.MEM_DEVICE)]
    before = ctx.launch_count
    for kw in bad_advance:
        assert advance(**kw) == -1, kw
    assert ctx.launch_count == before
    assert L.ofdis_track_stats_get(ctx._h, None) == -1
    # a refused call leaves the tracker as it was
    assert stats_ok()
    flows = fullres(ctx, 0, 2 * n, h, w, 2)
    exp, est = preprocess.track_points(clip, flows[:n], flows[n:], good)
    assert advance() == 0
    got = [pts[k * good["capacity"]:k * good["capacity"] + counts[k]].copy() for k in range(n)]
    assert_lists(got, exp[1:], "after the refused calls")
    assert ctx.track_stats() == est
    ctx.close()


# ---- batch front-end --------------------------------------------------------------------------------------------
def _write_png(path, img):
    h, w = img.shape[:2]
    ch = 1 if img.ndim == 2 else 3
    raw = b"".join(b"\0" + row.tobytes() for row in np.ascontiguousarray(img).reshape(h, w * ch))

    def chunk(t, d):
        return struct.pack(">I", len(d)) + t + d + struct.pack(">I", zlib.crc32(t + d) & 0xFFFFFFFF)

    with open(path, "wb") as f:
        f.write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 0 if ch == 1 else 2, 0, 0, 0)))
        f.write(chunk(b"IDAT", zlib.compress(raw)) + chunk(b"IEND", b""))


def _read_tracks(path):
    lines = open(path).read().splitlines()
    assert lines[0] == "# clip frame id x y"
    out = {}
    for ln in lines[1:]:
        c, fr, i, x, y = ln.split()
        out.setdefault((int(c), int(fr)), []).append((int(i), f32(float(x)), f32(float(y))))
    return {k: np.array(v, preprocess.TRACK_POINT_DTYPE) for k, v in out.items()}


@pytest.mark.parametrize("exe,nop,ch,extra", [("run_OF_INT", 2, 1, []), ("run_OF_RGB", 2, 3, ["--bidirectional"]),
                                              ("run_DE_INT", 1, 1, ["--color"]),
                                              ("run_DE_RGB", 1, 3, ["--interpolate", "0.5"])],
                         ids=["flow-gray", "flow-rgb-bidirectional", "stereo-gray-color", "stereo-rgb-interpolate"])
def test_batch_command_tracks(tmp_path, exe, nop, ch, extra, api):
    """Clip a (three pairs) split by batches of two, then two one-pair clips.  --tracks writes the Python call's tracks
    clip for clip; every other output keeps its bytes."""
    from of_dis_b200 import build

    bindir = build.build_host()
    ext = "flo" if nop == 2 else "pfm"
    h, w = 150, 250
    clip = synth.synthetic_sequence(4, h, w, ch, seed=96, amp=3.0, stereo=(nop == 1))
    other = synth.synthetic_sequence(3, h, w, ch, seed=97, amp=3.0, stereo=(nop == 1))
    paths, imgs = {}, {}
    for name, fr in (("a", clip), ("b", other)):
        for t, img in enumerate(fr):
            paths[name, t] = str(tmp_path / ("%s%d.png" % (name, t)))
            imgs[name, t] = img
            _write_png(paths[name, t], img)
    pairs = [("a", 0), ("a", 1), ("a", 2), ("b", 1), ("b", 0)]
    clips = [[0, 1, 2], [3], [4]]
    outs = {}
    logs = {}
    for tag in ("plain", "tracks"):
        outs[tag] = [str(tmp_path / ("%s%d.%s" % (tag, k, ext))) for k in range(len(pairs))]
        lst = tmp_path / ("%s.txt" % tag)
        lst.write_text("".join("%s %s %s\n" % (paths[nm, t], paths[nm, t + 1], outs[tag][k])
                               for k, (nm, t) in enumerate(pairs)))
        opts = extra + (["--tracks", str(tmp_path / "tracks.txt")] if tag == "tracks" else [])
        r = subprocess.run([os.path.join(bindir, exe + "_batch"), str(lst), "--batch", "2"] + opts + ["2"],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        logs[tag] = r.stdout
    got = _read_tracks(str(tmp_path / "tracks.txt"))
    prm = params.operating_point(2, w, noc=ch, nop=nop)
    bgr = (lambda a: a[..., ::-1]) if ch == 3 else (lambda a: a)  # the decoder holds BGR
    p = dict(capacity=4 * ((w + 7) // 8) * ((h + 7) // 8), spacing=8, alpha=0.01 if nop == 2 else 0.0,
             beta=0.5 if nop == 2 else 1.0, mb_alpha=0.01, mb_beta=0.002, min_eig=25.0)
    total = dict.fromkeys(preprocess.TRACK_STATS_FIELDS, 0)
    frames = 0
    for c, ks in enumerate(clips):
        fr = [bgr(imgs[pairs[ks[0]]])] + [bgr(imgs[pairs[k][0], pairs[k][1] + 1]) for k in ks]
        fr = np.ascontiguousarray(np.stack(fr))
        n = len(ks)
        ctx = context(api, prm, h, w, 2 * n)
        ctx.upload_sequence_bidir_u8(0, n, fr, w, h)
        ctx.run(2 * n)
        exp = [ctx.track_begin(p, fr[0], w, h)] + ctx.track_advance(0, n, n, fr[1:], w, h)
        st = ctx.track_stats()
        ctx.close()
        for k in total:
            total[k] += st[k]
        for t, e in enumerate(exp):
            g = got.get((c, t), np.empty(0, preprocess.TRACK_POINT_DTYPE))
            assert np.array_equal(g.view(np.uint8), e.view(np.uint8)), (c, t, g.shape, e.shape)
            frames += 1
    assert len(got) <= frames and total["seeded"] > 0
    line = [ln for ln in logs["tracks"].splitlines() if ln.startswith("TRACKS")]
    assert line == ["TRACKS clips 3 frames %d seeded %d leaves %d inconsistent %d boundary %d dropped %d"
                    % (frames, total["seeded"], total["ended_leaves"], total["ended_inconsistent"],
                       total["ended_boundary"], total["dropped"])], logs["tracks"]
    with_suffix = lambda q, s, e=None: os.path.splitext(q)[0] + s + (e or os.path.splitext(q)[1])  # noqa: E731
    bidir = "--bidirectional" in extra
    for k in range(len(pairs)):
        others = [""] + (["_bw", "_occ"] if bidir else []) + (["_color"] if "--color" in extra else []) + \
            (["_interp"] if "--interpolate" in extra else [])
        for suffix in others:
            e = ".pgm" if suffix == "_occ" else ".png" if suffix in ("_color", "_interp") else None
            a = open(with_suffix(outs["plain"][k], suffix, e), "rb").read()
            b = open(with_suffix(outs["tracks"][k], suffix, e), "rb").read()
            assert a == b, (k, suffix)
        if not bidir:
            assert not os.path.exists(with_suffix(outs["tracks"][k], "_bw"))
            assert not os.path.exists(with_suffix(outs["tracks"][k], "_occ", ".pgm"))


@pytest.mark.parametrize("args", [["--tracks"], ["--warm-start", "--tracks", "t.txt"]])
def test_batch_command_refuses(tmp_path, args):
    from of_dis_b200 import build

    bindir = build.build_host()
    lst = tmp_path / "list.txt"
    lst.write_text("")
    r = subprocess.run([os.path.join(bindir, "run_OF_INT_batch"), str(lst)] + args, capture_output=True, text=True,
                       cwd=str(tmp_path))
    assert r.returncode == 2, (args, r.stdout, r.stderr)
