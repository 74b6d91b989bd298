"""Color-coded full-resolution flows on the device: ofdis_flow_color_fullres.  Every image and scale must be BITWISE
what preprocess.flow_to_color / disp_to_color give on ofdis_get_flow_fullres's flow; the batch command's --color
PNGs decode to the restatement of the .flo / .pfm files the same run writes, and leave every other output as it is."""
import ctypes
import os
import re
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


def context(api, prm, h, w, max_frames):
    scf = 1 << prm.sc_f
    W, H = (w + scf - 1) // scf * scf, (h + scf - 1) // scf * scf
    return api.Context(prm, W, H, prm.p_samp_s, max_frames)


def fullres(ctx, f0, f1, h, w, nop):
    out = np.empty((f1 - f0, h, w, nop), np.float32)
    ctx.get_flow_fullres(f0, f1, out, w, h)
    ctx.sync()
    return out


def expected(flows, max_value=0.0, swapped=None):
    """The restatement of a batch of slots; `swapped` marks (stereo) per slot."""
    if flows.shape[-1] == 2:
        return preprocess.flow_to_color(flows, max_value)
    return preprocess.disp_to_color(flows, max_value, [False] * len(flows) if swapped is None else swapped)


def device_color(api, ctx, f0, f1, h, w, max_value):
    """The color call into caller-owned device tensors (uint8 images, float32 scales)."""
    import torch

    rgb = torch.full((f1 - f0, h, w, 3), 7, dtype=torch.uint8, device="cuda")
    scale = torch.full((f1 - f0,), -5.0, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    r, s = ctx.flow_color_fullres(f0, f1, w, h, max_value, out=rgb.data_ptr(), memkind=api.MEM_DEVICE,
                                  scale=scale.data_ptr())
    assert (r, s) == (rgb.data_ptr(), scale.data_ptr())
    ctx.sync()
    return rgb.cpu().numpy(), scale.cpu().numpy()


SMALL = "3 %d 8 8 0.05 0.95 0 8 0.4 %d 1 0 1 10 10 5 1 3 1.6 0"


@pytest.mark.parametrize("fb", [0, 1], ids=["fb0", "fb1"])
@pytest.mark.parametrize("size", [(128, 256), (121, 203)], ids=["div", "nondiv"])
@pytest.mark.parametrize("sc_l", [1, 0], ids=["sc_l1", "sc_l0"])
@pytest.mark.parametrize("nop,ch", [(2, 1), (2, 3), (1, 1), (1, 3)])
def test_color_equals_the_restatement(nop, ch, sc_l, size, fb, api):
    """Automatic and fixed scale on host and device memory, sub-ranges away from slot 0, repeated calls alternating
    with get_flow_fullres; the flows stay as they were."""
    h, w = size
    n = 3
    prm = params.from_cli_numbers((SMALL % (sc_l, fb)).split(), noc=ch, nop=nop)
    frames = synth.synthetic_sequence(n + 1, h, w, ch, seed=91, amp=3.0, stereo=(nop == 1))
    ctx = context(api, prm, h, w, n + 1)
    ctx.upload_sequence_u8(0, n, frames, w, h)
    ctx.run(n)
    flows = fullres(ctx, 0, n, h, w, nop)
    for max_value in (0.0, 2.5):
        exp_rgb, exp_scale = expected(flows, max_value)
        before = ctx.launch_count
        rgb, scale = ctx.flow_color_fullres(0, n, w, h, max_value, with_scale=True)
        assert ctx.launch_count == before + (2 if max_value == 0 else 1)
        assert_same(rgb, exp_rgb, "host rgb, max_value %g" % max_value)
        assert_same(scale, exp_scale, "host scale, max_value %g" % max_value)
        assert (rgb > 0).any() and len(np.unique(rgb.reshape(-1, 3), axis=0)) > 8
        for f0, f1 in ((1, 3), (2, 3), (1, 2)):
            # each slot's automatic scale is its own, so a sub-range colors its slots as the whole range does
            r, s = ctx.flow_color_fullres(f0, f1, w, h, max_value, with_scale=True)
            assert_same(r, exp_rgb[f0:f1], "host rgb %d..%d" % (f0, f1))
            assert_same(s, exp_scale[f0:f1], "host scale %d..%d" % (f0, f1))
            r, s = device_color(api, ctx, f0, f1, h, w, max_value)
            assert_same(r, exp_rgb[f0:f1], "device rgb %d..%d" % (f0, f1))
            assert_same(s, exp_scale[f0:f1], "device scale %d..%d" % (f0, f1))
        r, s = ctx.flow_color_fullres(0, n, w, h, max_value)
        assert s is None
        assert_same(r, exp_rgb, "host rgb without scale")
        assert_same(fullres(ctx, 0, n, h, w, nop), flows, "float flows between the color calls")
    ctx.close()


def _extremes(nop, h, w, rng):
    """Level flows with NaN of every sign and payload, the infinities, +-1e9 and the next float above, -0, next to
    ordinary values."""
    above = float(np.nextafter(f32(1e9), f32(np.inf)))
    vals = np.array([np.inf, -np.inf, 1e9, -1e9, above, -above, -0.0, 0.0, 0.5, -0.5, 3.0, -7.0], f32)
    nan_bits = np.array([0x7FC00000, 0xFFC00000, 0x7FC12345, 0xFF800001, 0x7F800001], np.uint32).view(np.float32)
    vals = np.concatenate([vals, nan_bits, rng.normal(0, 20, 32).astype(np.float32)])
    flow = rng.normal(0, 4, (h, w, nop)).astype(np.float32)
    flow.reshape(-1)[:vals.size] = vals  # every value at least once, next to each other
    flow.reshape(-1)[vals.size:2 * vals.size] = vals[::-1]
    return flow


@pytest.mark.parametrize("sc_l", [0, 1], ids=["sc_l0", "sc_l1"])
@pytest.mark.parametrize("nop", [2, 1])
def test_extreme_level_flows(nop, sc_l, api):
    """Level flows written with set_flow and colored without a run: every branch of the contract, an all-zero and an
    all-unknown slot (scale 1), max_value 1e-30 (fx, fy overflow, the angle stays finite) and 1e30; stereo slots
    marked swapped color +F."""
    h, w, n = 64, 96, 6
    prm = params.from_cli_numbers(("2 %d 8 8 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0" % sc_l).split(), noc=1,
                                  nop=nop)
    ctx = context(api, prm, h, w, n)
    rng = np.random.default_rng(92)
    lh, lw = ctx.height >> sc_l, ctx.width >> sc_l
    for f in range(4):
        ctx.set_flow(f, sc_l, _extremes(nop, lh, lw, rng))
    ctx.set_flow(4, sc_l, np.zeros((lh, lw, nop), np.float32))
    unknown = np.full((lh, lw, nop), np.nan, np.float32)
    unknown[::2] = np.inf
    ctx.set_flow(5, sc_l, unknown)
    swapped = [False] * n
    if nop == 1:
        ctx.set_swapped_slots(1, 3, 1)
        swapped[1:3] = [True, True]
    flows = fullres(ctx, 0, n, h, w, nop)
    assert np.isnan(flows).any() and np.isinf(flows).any()
    for max_value in (0.0, 1e-30, 1e30, 4.0):
        exp_rgb, exp_scale = expected(flows, max_value, swapped)
        rgb, scale = ctx.flow_color_fullres(0, n, w, h, max_value, with_scale=True)
        assert_same(rgb, exp_rgb, "host rgb, max_value %g" % max_value)
        assert_same(scale, exp_scale, "host scale, max_value %g" % max_value)
        r, s = device_color(api, ctx, 1, n, h, w, max_value)
        assert_same(r, exp_rgb[1:], "device rgb, max_value %g" % max_value)
        assert_same(s, exp_scale[1:], "device scale, max_value %g" % max_value)
        if max_value == 0:
            assert exp_scale[4] == 1 and exp_scale[5] == 1
            assert (rgb[5] == 0).all() and (rgb[4] == (255 if nop == 2 else 0)).all()
        if max_value == 1e-30 and nop == 2:
            moving = (flows[:4] != 0).any(-1) & (np.abs(flows[:4]) <= 1e9).all(-1)
            assert moving.any() and (rgb[:4][moving] <= 191).all()  # every nonzero known flow darkened by 0.75
            assert (rgb[:4][(flows[:4] == 0).all(-1)] == 255).all()  # zero flow stays white
    if sc_l == 0:  # the level flow is the full-resolution flow: every special value reaches the colors as it is
        px = ctx.flow_color_fullres(0, 1, w, h)[0][0].reshape(-1, 3)
        if nop == 2:  # pixels (inf, -inf), (1e9, -1e9), (above, -above), (-0, 0)
            assert (px[0] == 0).all() and px[1].any() and (px[2] == 0).all() and (px[3] == 255).all()
        else:  # d = -inf, +inf, -1e9, 1e9, -above, above: only d = 1e9 is valid (and beyond the scale)
            assert (px[[0, 1, 2, 4, 5]] == 0).all() and px[3].any()
    assert_same(fullres(ctx, 0, n, h, w, nop), flows, "flows after the color calls")
    ctx.close()


def test_swapped_slots_of_a_two_way_upload(api):
    """Stereo: the backward slots of upload_sequence_bidir_u8 hold the right view (marked swapped) and color +F."""
    h, w, n = 121, 203, 3
    prm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=1, nop=1)
    frames = synth.synthetic_sequence(n + 1, h, w, 1, seed=93, amp=3.0, stereo=True)
    ctx = context(api, prm, h, w, 2 * n)
    ctx.upload_sequence_bidir_u8(0, n, frames, w, h)
    ctx.run(2 * n)
    flows = fullres(ctx, 0, 2 * n, h, w, 1)
    assert (flows[:n] <= 0).mean() > 0.9 and (flows[n:] >= 0).mean() > 0.9
    exp_rgb, exp_scale = expected(flows, 0.0, [False] * n + [True] * n)
    rgb, scale = ctx.flow_color_fullres(0, 2 * n, w, h, with_scale=True)
    assert_same(rgb, exp_rgb, "both views")
    assert_same(scale, exp_scale, "both views' scales")
    assert (rgb[n:].any(-1)).mean() > 0.9  # the right view's disparities are valid
    r, s = device_color(api, ctx, n, 2 * n, h, w, 0.0)
    assert_same(r, rgb[n:], "device, right view")
    ctx.close()


def _status(api, fn, *args, **kw):
    try:
        fn(*args, **kw)
    except api.OfdisError as e:
        return int(re.match(r"status (-?\d+)", str(e)).group(1))
    return 0


def test_bad_arguments(api):
    import torch

    h, w, n = 128, 256, 2
    prm = params.operating_point(2, w, noc=1)
    cap = n + 1
    ctx = context(api, prm, h, w, cap)
    ctx.upload_sequence_u8(0, n, synth.synthetic_sequence(n + 1, h, w, 1, seed=94), w, h)
    ctx.run(n)
    buf = np.full((cap + 1) * h * w * 3 + 8, 7, np.uint8)
    sbuf = np.full(cap + 1, -5.0, np.float32)
    dev = torch.full(((cap + 1) * h * w * 3 + 8,), 7, dtype=torch.uint8, device="cuda")
    dscale = torch.full((cap + 2,), -5.0, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    L = api.lib()
    host, hscale = buf.ctypes.data, sbuf.ctypes.data

    def call(f0, f1, rgb=host, scale=hscale, mv=0.0, ww=w, hh=h, mem=api.MEM_HOST, handle=None):
        return L.ofdis_flow_color_fullres(ctx._h if handle is None else handle, f0, f1,
                                          None if rgb is None else ctypes.c_void_p(rgb),
                                          None if scale is None else ctypes.c_void_p(scale), mv, ww, hh, mem)

    bad = {"null rgb": dict(f0=0, f1=n, rgb=None), "null device rgb": dict(f0=0, f1=n, rgb=None, mem=api.MEM_DEVICE),
           "max_value nan": dict(f0=0, f1=n, mv=float("nan")), "max_value -1": dict(f0=0, f1=n, mv=-1.0),
           "max_value -1e-30": dict(f0=0, f1=n, mv=-1e-30), "max_value inf": dict(f0=0, f1=n, mv=float("inf")),
           "max_value -inf": dict(f0=0, f1=n, mv=float("-inf")),
           "odd device scale": dict(f0=0, f1=n, rgb=dev.data_ptr(), scale=dscale.data_ptr() + 2, mem=api.MEM_DEVICE),
           "f0 < 0": dict(f0=-1, f1=1), "f1 > max_frames": dict(f0=0, f1=cap + 1),
           "f0 == f1": dict(f0=1, f1=1), "f0 > f1": dict(f0=2, f1=1),
           "width": dict(f0=0, f1=n, ww=w + 1), "height": dict(f0=0, f1=n, hh=h - 64),
           "width 0": dict(f0=0, f1=n, ww=0), "height -1": dict(f0=0, f1=n, hh=-1)}
    for name, kw in bad.items():
        before = ctx.launch_count
        assert call(**kw) == -1, name
        assert ctx.launch_count == before, name
    assert call(0, n, handle=ctypes.c_void_p()) == -1, "null context"
    torch.cuda.synchronize()
    ctx.sync()
    assert (buf == 7).all() and (sbuf == -5.0).all(), "host output touched by a refused call"
    assert bool((dev == 7).all()) and bool((dscale == -5.0).all()), "device output touched by a refused call"
    # the good calls: host output anywhere, device scale 4-byte aligned or NULL, max_value 0 and FLT_MAX
    assert call(0, n) == 0 and call(0, cap, mv=3.0e38) == 0 and call(1, cap, scale=None) == 0
    assert call(0, n, rgb=host + 1, scale=hscale + 4) == 0
    assert call(0, n, rgb=dev.data_ptr() + 1, scale=dscale.data_ptr() + 4, mem=api.MEM_DEVICE) == 0
    assert call(0, n, rgb=dev.data_ptr(), scale=None, mem=api.MEM_DEVICE) == 0
    ctx.sync()
    # the same through the Python wrapper
    assert _status(api, ctx.flow_color_fullres, 0, n, w + 1, h) == -1
    assert _status(api, ctx.flow_color_fullres, 0, cap + 1, w, h) == -1
    assert _status(api, ctx.flow_color_fullres, 0, n, w, h, -2.0) == -1
    for bad_out in (np.empty((n, h, w, 3), np.int8), np.empty((n, h, w), np.uint8), np.empty((n, h, w + 1, 3), np.uint8),
                    list(np.empty((n, h, w, 3), np.uint8)), np.empty((n, h, 2 * w, 3), np.uint8)[:, :, ::2]):
        with pytest.raises(ValueError):
            ctx.flow_color_fullres(0, n, w, h, out=bad_out)
    with pytest.raises(ValueError):
        ctx.flow_color_fullres(0, n, w, h, with_scale=True, scale=np.empty(n, np.float64))
    out, sc = np.empty((n, h, w, 3), np.uint8), np.empty(n, np.float32)
    r, s = ctx.flow_color_fullres(0, n, w, h, out=out, with_scale=True, scale=sc)
    assert r is out and s is sc
    assert_same(out, expected(fullres(ctx, 0, n, h, w, 2))[0], "given out")
    ctx.close()


def test_host_scratch_is_shared_with_get_flow_fullres(api):
    """Alternating the color call and get_flow_fullres on host memory never reallocates the scratch: the color call
    fits in the size get_flow_fullres asks for, for flow and stereo."""
    h, w, n = 64, 96, 3
    for nop in (2, 1):
        prm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=1, nop=nop)
        ctx = context(api, prm, h, w, n)
        ctx.upload_sequence_u8(0, n, synth.synthetic_sequence(n + 1, h, w, 1, seed=95, stereo=(nop == 1)), w, h)
        ctx.run(n)
        flows = fullres(ctx, 0, n, h, w, nop)
        for _ in range(2):
            rgb, scale = ctx.flow_color_fullres(0, n, w, h, with_scale=True)
            assert_same(fullres(ctx, 0, n, h, w, nop), flows, "flows")
        exp = expected(flows)
        assert_same(rgb, exp[0], "rgb, nop %d" % nop)
        assert_same(scale, exp[1], "scale, nop %d" % nop)
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


def _read_rgb8_png(path):
    """An 8-bit RGB non-interlaced PNG (any row filter), checking every chunk's CRC."""
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
    assert (depth, ctype, interlace) == (8, 2, 0), (path, hdr)
    raw = np.frombuffer(zlib.decompress(b"".join(idat)), np.uint8).reshape(h, 3 * w + 1)
    img = np.zeros((h, 3 * w), np.uint8)
    up = np.zeros(3 * w, np.uint8)
    for y in range(h):
        img[y] = preprocess._unfilter(int(raw[y, 0]), raw[y, 1:], up, 3)
        up = img[y]
    return img.reshape(h, w, 3)


@pytest.mark.parametrize("exe,nop,extra", [("run_OF_INT", 2, []), ("run_DE_INT", 1, ["--bidirectional"]),
                                           ("run_OF_INT", 2, ["--bidirectional", "--kitti"]),
                                           ("run_DE_INT", 1, ["--warm-start"])],
                         ids=["flow", "stereo-bidirectional", "flow-bidirectional-kitti", "stereo-warm-start"])
@pytest.mark.parametrize("color_max", [None, "3.5"], ids=["own-max", "color-max"])
def test_batch_command_color(tmp_path, exe, nop, extra, color_max, api):
    """A chain of three pairs and two unrelated ones.  With --color every output gets a _color.png (and _bw_color.png)
    whose pixels are the restatement of the .flo / .pfm the same run writes (each pair's own maximum, or the scale
    of --color-max; _bw with the swapped sign); every other output file is byte-identical to a run without --color."""
    from of_dis_b200 import build

    bindir = build.build_host()
    ext = "flo" if nop == 2 else "pfm"
    kitti = "--kitti" in extra
    bidir = "--bidirectional" in extra
    h, w = 150, 250
    clip = synth.synthetic_sequence(4, h, w, 1, seed=96, amp=3.0, stereo=(nop == 1))
    other = synth.synthetic_sequence(3, h, w, 1, seed=97, amp=3.0, stereo=(nop == 1))
    paths = {}
    for name, fr in (("a", clip), ("b", other)):
        for t, img in enumerate(fr):
            paths[name, t] = str(tmp_path / ("%s%d.png" % (name, t)))
            _write_png(paths[name, t], img)
    pairs = [("a", 0), ("a", 1), ("a", 2), ("b", 1), ("b", 0)]
    outs = {}
    batch = [] if "--warm-start" in extra else ["--batch", "3"]
    for tag in ("plain", "color", "float"):  # "float": without --kitti, the files the colors are checked against
        oext = "png" if kitti and tag != "float" else ext
        outs[tag] = [str(tmp_path / ("%s%d.%s" % (tag, k, oext))) for k in range(len(pairs))]
        lst = tmp_path / ("%s.txt" % tag)
        lst.write_text("".join("%s %s %s\n" % (paths[nm, t], paths[nm, t + 1], outs[tag][k])
                               for k, (nm, t) in enumerate(pairs)))
        opts = [o for o in extra if tag != "float" or o != "--kitti"]
        if tag == "color":
            opts = opts + ["--color"] + (["--color-max", color_max] if color_max else [])
        r = subprocess.run([os.path.join(bindir, exe + "_batch"), str(lst)] + batch + opts + ["2"],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
    read = preprocess.read_flo if nop == 2 else preprocess.read_pfm
    mv = float(f32(color_max)) if color_max else 0.0
    with_suffix = lambda p, s, e=None: os.path.splitext(p)[0] + s + (e or os.path.splitext(p)[1])  # noqa: E731
    sides = [("", False)] + ([("_bw", True)] if bidir else [])
    for k in range(len(pairs)):
        for suffix, swapped in sides:
            flow = read(with_suffix(outs["float"][k], suffix))
            exp = (preprocess.flow_to_color(flow, mv) if nop == 2 else
                   preprocess.disp_to_color(flow, mv, swapped))[0]
            got = _read_rgb8_png(with_suffix(outs["color"][k], suffix + "_color", ".png"))
            assert_same(got, exp, "pair %d%s" % (k, suffix))
            assert (got > 0).any()
            assert not os.path.exists(with_suffix(outs["plain"][k], suffix + "_color", ".png"))
        # every other output keeps its bytes
        others = [""] + (["_bw", "_occ"] if bidir else [])
        for suffix in others:
            e = ".pgm" if suffix == "_occ" else None
            a = open(with_suffix(outs["plain"][k], suffix, e), "rb").read()
            assert a == open(with_suffix(outs["color"][k], suffix, e), "rb").read(), (k, suffix)
