"""Frame interpolation on the device: ofdis_interpolate_fullres.  Every output frame and every flow at time t must be
BITWISE what preprocess.interpolate_frames gives on ofdis_get_flow_fullres's flows of the same slots; the batch
command's --interpolate PNGs must be the Python call's frames and leave every other output as it is."""
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


def assert_same(got, exp, name):
    got, exp = np.asarray(got), np.asarray(exp)
    assert got.shape == exp.shape and got.dtype == exp.dtype, (name, got.shape, exp.shape, got.dtype, exp.dtype)
    a = got.view(np.uint32) if got.dtype == f32 else got
    b = exp.view(np.uint32) if exp.dtype == f32 else exp
    bad = a != b
    if bad.any():
        i = tuple(np.argwhere(bad)[0])
        raise AssertionError("%s: %d of %d values differ, first at %s: %r, expected %r"
                             % (name, int(bad.sum()), bad.size, i, got[i], exp[i]))


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


SMALL = "3 %d 8 8 0.05 0.95 0 8 0.4 %d 1 0 1 10 10 5 1 3 1.6 0"


def two_way_context(api, layout, nop, ch, sc_l, fb, h, w, n, seed, graph=False):
    """A context whose slots 1 .. n hold the forward pairs of a clip and n+1 .. 2n their backward partners (slots 0
    and 2n+1 hold unrelated pairs).  Returns (ctx, frames0, frames1, all slots' full-resolution flows)."""
    prm = params.from_cli_numbers((SMALL % (sc_l, fb)).split(), noc=ch, nop=nop)
    clip = synth.synthetic_sequence(n + 1, h, w, ch, seed=seed, amp=3.0, stereo=(nop == 1))
    other = synth.synthetic_sequence(2, h, w, ch, seed=seed + 1, amp=3.0, stereo=(nop == 1))
    ctx = context(api, prm, h, w, 2 * n + 2)
    if graph:
        ctx.set_graph_mode(True)
    ctx.upload_frames_u8(0, 1, np.ascontiguousarray(other[None]), w, h)
    if layout == "sequence":
        ctx.upload_sequence_bidir_u8(1, n, clip, w, h)
        frames0, frames1 = clip[:-1], clip[1:]
    else:  # the pairs, then their swapped copies, as the batch command uploads them
        pairs = np.ascontiguousarray(np.stack([clip[:-1], clip[1:]], 1))
        ctx.upload_frames_u8(1, n + 1, pairs, w, h)
        ctx.upload_frames_u8(n + 1, 2 * n + 1, np.ascontiguousarray(pairs[:, ::-1]), w, h)
        ctx.set_swapped_slots(1, n + 1, 0)
        ctx.set_swapped_slots(n + 1, 2 * n + 1, 1)
        frames0, frames1 = pairs[:, 0], pairs[:, 1]
    ctx.upload_frames_u8(2 * n + 1, 2 * n + 2, np.ascontiguousarray(other[::-1][None]), w, h)
    ctx.run(2 * n + 2)
    return ctx, frames0, frames1, fullres(ctx, 0, 2 * n + 2, h, w, nop)


@pytest.mark.parametrize("layout", ["sequence", "pairs"])
@pytest.mark.parametrize("fb", [0, 1], ids=["fb0", "fb1"])
@pytest.mark.parametrize("size", [(128, 256), (121, 203)], ids=["div", "nondiv"])
@pytest.mark.parametrize("nop,ch", [(2, 1), (2, 3), (1, 1), (1, 3)])
def test_interpolation_equals_the_restatement(nop, ch, size, fb, layout, api):
    """Host memory, f0 = 1 and b0 = n + 1, sub-ranges, two times; the flows of every slot stay as they were."""
    h, w = size
    n = 3
    ctx, frames0, frames1, flows = two_way_context(api, layout, nop, ch, 1, fb, h, w, n, seed=31)
    alpha, beta = 0.01 if nop == 2 else 0.0, 0.5 if nop == 2 else 1.0
    for t in (0.5, 0.3):
        exp_out, exp_ut = preprocess.interpolate_frames(frames0, frames1, flows[1:n + 1], flows[n + 1:2 * n + 1], t,
                                                        alpha, beta)
        before = ctx.launch_count
        out, ut = ctx.interpolate_fullres(1, n + 1, n + 1, frames0, frames1, t, w, h, with_flow=True)
        assert ctx.launch_count - before >= 6
        assert_same(out, exp_out, "out t=%g" % t)
        assert_same(ut, exp_ut, "flow_t t=%g" % t)
        assert len(np.unique(out)) > 16
        for k0, k1 in ((1, 3), (2, 3)):
            o, u = ctx.interpolate_fullres(1 + k0, 1 + k1, n + 1 + k0, frames0[k0:k1], frames1[k0:k1], t, w, h,
                                           with_flow=True)
            assert_same(o, exp_out[k0:k1], "out %d..%d" % (k0, k1))
            assert_same(u, exp_ut[k0:k1], "flow_t %d..%d" % (k0, k1))
    assert_same(fullres(ctx, 0, 2 * n + 2, h, w, nop), flows, "flows after the calls")
    ctx.close()


@pytest.mark.parametrize("layout", ["sequence", "pairs"])
@pytest.mark.parametrize("nop,ch", [(2, 3), (1, 1)])
def test_device_memory_on_a_caller_stream(nop, ch, layout, api):
    import torch

    h, w, n = 121, 203, 2
    stream = torch.cuda.Stream()
    prm = params.from_cli_numbers((SMALL % (0, 0)).split(), noc=ch, nop=nop)
    clip = synth.synthetic_sequence(n + 1, h, w, ch, seed=41, amp=3.0, stereo=(nop == 1))
    ctx = context(api, prm, h, w, 2 * n, stream=stream.cuda_stream)
    hwc = h * w * ch
    if layout == "sequence":
        dev = torch.from_numpy(clip.reshape(-1)).cuda()
        ctx.upload_sequence_bidir_u8(0, n, clip, w, h)
        p0, stride = dev.data_ptr(), hwc
        frames0, frames1 = clip[:-1], clip[1:]
    else:
        pairs = np.ascontiguousarray(np.stack([clip[:-1], clip[1:]], 1))
        dev = torch.from_numpy(pairs.reshape(-1)).cuda()
        ctx.upload_frames_u8(0, n, pairs, w, h)
        ctx.upload_frames_u8(n, 2 * n, np.ascontiguousarray(pairs[:, ::-1]), w, h)
        ctx.set_swapped_slots(n, 2 * n, 1)
        p0, stride = dev.data_ptr(), 2 * hwc
        frames0, frames1 = pairs[:, 0], pairs[:, 1]
    ctx.run(2 * n)
    flows = fullres(ctx, 0, 2 * n, h, w, nop)
    alpha, beta = (0.01, 0.5) if nop == 2 else (0.0, 1.0)
    exp_out, exp_ut = preprocess.interpolate_frames(frames0, frames1, flows[:n], flows[n:], 0.5, alpha, beta)
    out = torch.full((n, h, w, ch), 7, dtype=torch.uint8, device="cuda")
    ut = torch.full((n, h, w, nop), -3.0, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    r = ctx.interpolate_fullres(0, n, n, p0, p0 + hwc, 0.5, w, h, out=out.data_ptr(), flow_t=ut.data_ptr(),
                                memkind=api.MEM_DEVICE, frame_stride=stride)
    assert r == (out.data_ptr(), ut.data_ptr())
    stream.synchronize()
    assert_same(out.cpu().numpy().reshape(exp_out.shape), exp_out, "device out")
    assert_same(ut.cpu().numpy(), exp_ut, "device flow_t")
    # without flow_t
    out2 = torch.zeros_like(out)
    ctx.interpolate_fullres(0, n, n, p0, p0 + hwc, 0.5, w, h, out=out2.data_ptr(), memkind=api.MEM_DEVICE,
                            frame_stride=stride)
    stream.synchronize()
    assert torch.equal(out, out2)
    ctx.close()


def test_graph_mode_repeated_calls_and_two_contexts(api):
    """Runs replayed from a graph, two calls and two contexts give the same bits."""
    h, w, n = 128, 256, 3
    got = []
    for _ in range(2):
        ctx, frames0, frames1, flows = two_way_context(api, "sequence", 2, 1, 1, 0, h, w, n, seed=51, graph=True)
        ctx.run(2 * n + 2)  # a replay
        exp_out, exp_ut = preprocess.interpolate_frames(frames0, frames1, flows[1:n + 1], flows[n + 1:2 * n + 1],
                                                        0.5, 0.01, 0.5)
        for _ in range(2):
            out, ut = ctx.interpolate_fullres(1, n + 1, n + 1, frames0, frames1, 0.5, w, h, with_flow=True)
            assert_same(out, exp_out, "graph-mode out")
            assert_same(ut, exp_ut, "graph-mode flow_t")
            got.append(out)
        ctx.close()
    for g in got[1:]:
        assert_same(g, got[0], "same bits")


@pytest.mark.parametrize("sc_l", [0, 1])
def test_one_source_fills_the_frame_and_extreme_flows(sc_l, api):
    """Level flows set directly: slot 0 has one known pixel (every other NaN), so one splat fills the frame over about
    w + h rounds; slot 1 holds NaN, +-inf, huge and out-of-frame values; slot 2 is all NaN (u_t = 0)."""
    h, w = 128, 256
    prm = params.from_cli_numbers((SMALL % (sc_l, 0)).split(), noc=1, nop=2)
    ctx = context(api, prm, h, w, 6)
    hl, wl = h >> sc_l, w >> sc_l
    rng = np.random.default_rng(61)
    lv = [np.full((hl, wl, 2), np.nan, f32) for _ in range(6)]
    lv[0][0, 0] = (1.0, 0.5)  # full-resolution pixel (0, 0) is the only one whose upsampling taps no NaN
    lv[1] = rng.normal(0, 2, (hl, wl, 2)).astype(f32)
    m = rng.random((hl, wl))
    lv[1][m < 0.1, 0] = np.nan
    lv[1][(m >= 0.1) & (m < 0.15), 1] = np.inf
    lv[1][(m >= 0.15) & (m < 0.2), 0] = -np.inf
    lv[1][(m >= 0.2) & (m < 0.25), 0] = 3e9
    lv[1][(m >= 0.25) & (m < 0.3), 1] = 9e8
    lv[1][(m >= 0.3) & (m < 0.4), 0] += w
    lv[3] = np.zeros((hl, wl, 2), f32)
    lv[4] = -lv[1]
    for k in range(6):
        ctx.set_flow(k, sc_l, lv[k])
    flows = fullres(ctx, 0, 6, h, w, 2)
    frames = synth.synthetic_sequence(2, h, w, 1, seed=62)
    f0 = np.ascontiguousarray(np.stack([frames[0]] * 3))
    f1 = np.ascontiguousarray(np.stack([frames[1]] * 3))
    exp_out, exp_ut, rounds = preprocess.interpolate_frames(f0, f1, flows[:3], flows[3:], 0.5, 0.01, 0.5,
                                                            with_rounds=True)
    assert rounds > (w + h) // 2
    before = ctx.launch_count
    out, ut = ctx.interpolate_fullres(0, 3, 3, f0, f1, 0.5, w, h, with_flow=True)
    assert ctx.launch_count - before >= rounds
    assert_same(out, exp_out, "out")
    assert_same(ut, exp_ut, "flow_t")
    assert not ut[2].any()
    assert_same(fullres(ctx, 0, 6, h, w, 2), flows, "flows after the call")
    ctx.close()


def test_bad_arguments(api):
    import torch

    h, w, n = 128, 256, 2
    prm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=1, nop=2)
    ctx = context(api, prm, h, w, 2 * n)
    clip = synth.synthetic_sequence(n + 1, h, w, 1, seed=71)
    ctx.upload_sequence_bidir_u8(0, n, clip, w, h)
    ctx.run(2 * n)
    flows = fullres(ctx, 0, 2 * n, h, w, 2)
    out = np.zeros((n, h, w), np.uint8)
    ut = torch.zeros((n * h * w * 2 + 1,), dtype=torch.float32, device="cuda")
    L = api.lib()
    hwc = h * w
    p0 = clip.ctypes.data_as(ctypes.c_void_p)
    p1 = ctypes.c_void_p(clip.ctypes.data + hwc)
    po = out.ctypes.data_as(ctypes.c_void_p)

    def call(f0=0, f1=n, b0=n, i0=p0, i1=p1, stride=hwc, t=0.5, alpha=0.01, beta=0.5, o=po, fl=None, ww=w, hh=h,
             mem=api.MEM_HOST):
        return L.ofdis_interpolate_fullres(ctx._h, f0, f1, b0, i0, i1, stride, t, alpha, beta, o, fl, ww, hh, mem)

    bad = [dict(f0=-1), dict(f1=2 * n + 1), dict(f0=1, f1=1), dict(b0=-1), dict(b0=n + 1), dict(i0=None),
           dict(i1=None), dict(o=None), dict(t=0.0), dict(t=1.0), dict(t=-0.5), dict(t=float("nan")),
           dict(t=float("inf")), dict(stride=hwc - 1), dict(alpha=-1.0), dict(alpha=float("nan")),
           dict(alpha=float("inf")), dict(beta=-0.1), dict(beta=float("nan")), dict(beta=float("inf")),
           dict(ww=w + 8), dict(hh=h - 17), dict(ww=0),
           dict(o=ctypes.c_void_p(ut.data_ptr()), fl=ctypes.c_void_p(ut.data_ptr() + 2), mem=api.MEM_DEVICE,
                i0=ctypes.c_void_p(ut.data_ptr()), i1=ctypes.c_void_p(ut.data_ptr()))]
    before = ctx.launch_count
    for kw in bad:
        assert call(**kw) == -1, kw
    assert ctx.launch_count == before
    # the checks in Python: strides, shapes, dtypes
    with pytest.raises(ValueError):
        ctx.interpolate_fullres(0, n, n, clip[:-1], clip[1:].astype(np.int16), 0.5, w, h)
    with pytest.raises(api.OfdisError):
        ctx.interpolate_fullres(0, n, n, clip[:-1], clip[1:], 1.5, w, h)
    assert call() == 0
    ctx.sync()
    exp, _ = preprocess.interpolate_frames(clip[:-1], clip[1:], flows[:n], flows[n:], 0.5, 0.01, 0.5)
    assert_same(out, exp, "after the refused calls")
    assert_same(fullres(ctx, 0, 2 * n, h, w, 2), flows, "flows")
    ctx.close()


@pytest.mark.parametrize("ch", [1, 3])
def test_quality_on_a_synthetic_clip(ch, api):
    """Frames 0 and 2 of a synthetic clip interpolated at 0.5 are closer (RMS) to the held-out frame 1 than the plain
    blend and than frame 0 (tools/interp_e2e.py reports the numbers)."""
    h, w = 218, 512
    clip = synth.synthetic_sequence(3, h, w, ch, seed=81, amp=3.0)
    prm = params.operating_point(2, w, noc=ch)
    ctx = context(api, prm, h, w, 2)
    ends = np.ascontiguousarray(clip[::2])
    ctx.upload_sequence_bidir_u8(0, 1, ends, w, h)
    ctx.run(2)
    out, _ = ctx.interpolate_fullres(0, 1, 1, ends[:1], ends[1:], 0.5, w, h)
    ctx.close()
    ref = clip[1].astype(np.float64)
    rms = lambda a: float(np.sqrt(np.mean((np.asarray(a, np.float64) - ref) ** 2)))  # noqa: E731
    naive = 0.5 * clip[0].astype(np.float64) + 0.5 * clip[2].astype(np.float64)
    assert rms(out[0]) < rms(naive) and rms(out[0]) < rms(clip[0])


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


def _read_png8(path):
    """An 8-bit gray or RGB non-interlaced PNG (any row filter), checking every chunk's CRC."""
    b = open(path, "rb").read()
    assert b[:8] == b"\x89PNG\r\n\x1a\n", path
    pos, idat, hdr = 8, [], None
    while pos + 12 <= len(b):
        n, t = struct.unpack(">I", b[pos:pos + 4])[0], b[pos + 4:pos + 8]
        data = b[pos + 8:pos + 8 + n]
        assert struct.unpack(">I", b[pos + 8 + n:pos + 12 + n])[0] == zlib.crc32(t + data) & 0xFFFFFFFF, (path, t)
        if t == b"IHDR":
            hdr = struct.unpack(">IIBBBBB", data[:13])
        elif t == b"IDAT":
            idat.append(data)
        elif t == b"IEND":
            break
        pos += 12 + n
    w, h, depth, ctype, _, _, interlace = hdr
    assert depth == 8 and ctype in (0, 2) and interlace == 0, (path, hdr)
    ch = 3 if ctype == 2 else 1
    raw = np.frombuffer(zlib.decompress(b"".join(idat)), np.uint8).reshape(h, ch * w + 1)
    img = np.zeros((h, ch * w), np.uint8)
    up = np.zeros(ch * w, np.uint8)
    for y in range(h):
        img[y] = preprocess._unfilter(int(raw[y, 0]), raw[y, 1:], up, ch)
        up = img[y]
    return img.reshape(h, w, ch) if ch == 3 else img.reshape(h, w)


@pytest.mark.parametrize("exe,nop,ch,extra", [("run_OF_INT", 2, 1, []), ("run_OF_RGB", 2, 3, ["--bidirectional"]),
                                              ("run_DE_INT", 1, 1, ["--color"]),
                                              ("run_DE_RGB", 1, 3, ["--bidirectional", "--kitti"])],
                         ids=["flow-gray", "flow-rgb-bidirectional", "stereo-gray-color", "stereo-rgb-bidir-kitti"])
def test_batch_command_interpolate(tmp_path, exe, nop, ch, extra, api):
    """A chain of three pairs (two-way sequence upload) and two unrelated ones (pairs plus swapped copies) in batches of
    three.  --interpolate 0.5 writes <stem>_interp.png equal to the Python call on the same slots' flows; the flow,
    _bw, _occ and _color files keep their bytes, and no _bw / _occ appear without --bidirectional."""
    from of_dis_b200 import build

    bindir = build.build_host()
    ext = "flo" if nop == 2 else "pfm"
    bidir = "--bidirectional" in extra
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
    outs = {}
    oext = "png" if "--kitti" in extra else ext
    for tag in ("plain", "interp"):
        outs[tag] = [str(tmp_path / ("%s%d.%s" % (tag, k, oext))) for k in range(len(pairs))]
        lst = tmp_path / ("%s.txt" % tag)
        lst.write_text("".join("%s %s %s\n" % (paths[nm, t], paths[nm, t + 1], outs[tag][k])
                               for k, (nm, t) in enumerate(pairs)))
        opts = extra + (["--interpolate", "0.5"] if tag == "interp" else [])
        r = subprocess.run([os.path.join(bindir, exe + "_batch"), str(lst), "--batch", "3"] + opts + ["2"],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
    with_suffix = lambda p, s, e=None: os.path.splitext(p)[0] + s + (e or os.path.splitext(p)[1])  # noqa: E731
    # the Python call on the same slots: the batch command's parameters (operating point 2 from the CLI's "2")
    prm = params.operating_point(2, w, noc=ch, nop=nop)
    bgr = (lambda a: a[..., ::-1]) if ch == 3 else (lambda a: a)  # the decoder holds BGR
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
            ctx.set_swapped_slots(n, 2 * n, 1)
        ctx.run(2 * n)
        exp, _ = ctx.interpolate_fullres(0, n, n, i0, i1, 0.5, w, h)
        ctx.close()
        for k in range(b0, b1):
            got = _read_png8(with_suffix(outs["interp"][k], "_interp", ".png"))
            assert_same(got, bgr(exp[k - b0]), "pair %d" % k)
    for k in range(len(pairs)):
        assert not os.path.exists(with_suffix(outs["plain"][k], "_interp", ".png"))
        others = [""] + (["_bw", "_occ"] if bidir else []) + (["_color"] if "--color" in extra else []) + \
            (["_bw_color"] if "--color" in extra and bidir else [])
        for suffix in others:
            e = ".pgm" if suffix == "_occ" else ".png" if suffix.endswith("_color") else None
            a = open(with_suffix(outs["plain"][k], suffix, e), "rb").read()
            b = open(with_suffix(outs["interp"][k], suffix, e), "rb").read()
            assert a == b, (k, suffix)
        if not bidir:
            assert not os.path.exists(with_suffix(outs["interp"][k], "_bw"))
            assert not os.path.exists(with_suffix(outs["interp"][k], "_occ", ".pgm"))


@pytest.mark.parametrize("args", [["--interpolate", "0"], ["--interpolate", "1"], ["--interpolate", "nan"],
                                  ["--interpolate", "inf"], ["--interpolate", "0.5x"], ["--interpolate"],
                                  ["--warm-start", "--interpolate", "0.5"]])
def test_batch_command_refuses(tmp_path, args):
    from of_dis_b200 import build

    bindir = build.build_host()
    lst = tmp_path / "list.txt"
    lst.write_text("")
    r = subprocess.run([os.path.join(bindir, "run_OF_INT_batch"), str(lst)] + args, capture_output=True, text=True)
    assert r.returncode == 2, (args, r.stdout, r.stderr)
