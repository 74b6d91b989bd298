"""ofdis_disparity_fullres: every output byte must equal preprocess.disparity_filter of the disparities
ofdis_get_flow_fullres returns, on run flows (gray and RGB, usefbcon 0 and 1, divisible and non-divisible sizes, the
two-way upload) and on exact maps set at sc_l = 0 (one frame-wide component, a one-pixel spiral across the tile
borders, a checkerboard, components at the threshold, special values)."""
import itertools
import re

import numpy as np
import pytest
from scipy import ndimage

from of_dis_b200 import params, preprocess, synth

pytestmark = pytest.mark.gpu

OUTS = ("disp", "status", "depth", "xyz")
CAM = dict(fx=721.5, fy=721.5, cx=101.25, cy=60.5, baseline=0.54, doffs=0.25)


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


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
    out = np.empty((f1 - f0, h, w, 1), np.float32)
    ctx.get_flow_fullres(f0, f1, out, w, h)
    ctx.sync()
    return out


def expected(flows, f0, f1, b0, swapped, filt, camera):
    res = {k: [] for k in OUTS}
    for k in range(f1 - f0):
        B = flows[b0 + k] if filt["lr_check"] else None
        d, s, z, x = preprocess.disparity_filter(flows[f0 + k], B, swapped[f0 + k], camera=camera, **filt)
        for name, v in zip(OUTS, (d, s, z, x)):
            res[name].append(v)
    return {k: (np.stack(v) if v[0] is not None else None) for k, v in res.items()}


def assert_outputs(got, exp, what):
    for name, g in got.items():
        e = exp[name]
        if name == "status":
            bad = g != e
        else:
            bad = bits(g) != bits(e)
        if bad.any():
            raise AssertionError("%s %s: %d of %d differ, first at %s" % (what, name, int(bad.sum()), bad.size,
                                                                          np.argwhere(bad)[0]))


def filters(speckles=((25, 1.0), (25, 0.02))):
    """Every combination of lr_check, speckles (off, then each (size, diff)) and fill; a diff of 0.02 px cuts smooth
    run disparities into small components."""
    for lr, sp, fill in itertools.product((0, 1), (None,) + tuple(speckles), (0, 1)):
        yield dict(lr_check=lr, alpha=0.0, beta=1.0, speckle_size=sp[0] if sp else 0,
                   speckle_diff=sp[1] if sp else 1.0, fill=fill)


def small(ch, fb, sc_l=1):
    return params.from_cli_numbers(("3 %d 8 8 0.05 0.95 0 8 0.4 %d 1 0 1 10 10 5 1 3 1.6 0" % (sc_l, fb)).split(),
                                   noc=ch, nop=1)


@pytest.mark.parametrize("size", [(128, 256), (121, 203)], ids=["div", "nondiv"])
@pytest.mark.parametrize("fb", [0, 1], ids=["fb0", "fb1"])
@pytest.mark.parametrize("ch", [1, 3])
def test_run_flows_equal_the_restatement(ch, fb, size, api):
    h, w = size
    n = 3
    prm = small(ch, fb)
    frames = synth.synthetic_sequence(n + 1, h, w, ch, seed=31 + ch, amp=3.0, stereo=True)
    ctx = context(api, prm, h, w, 2 * n)
    ctx.upload_sequence_bidir_u8(0, n, frames, w, h)
    ctx.run(2 * n)
    flows = fullres(ctx, 0, 2 * n, h, w)
    swapped = [False] * n + [True] * n
    seen = set()
    # forward slots against their backward partners, a sub-range at f0 != 0, and the swapped slots against the forward
    for f0, f1, b0 in ((0, n, n), (1, 3, n + 1), (n, 2 * n, 0)):
        for filt in filters():
            exp = expected(flows, f0, f1, b0, swapped, filt, CAM)
            before = api.lib().ofdis_launch_count(ctx._h)
            got = ctx.disparity_fullres(f0, f1, b0, w, h, camera=CAM, outputs=OUTS, **filt)
            assert ctx.launch_count - before == 2 + 3 * (filt["speckle_size"] > 0) + 2 * filt["fill"]
            assert_outputs(got, exp, "slots %d..%d %s" % (f0, f1, filt))
            seen |= set(np.unique(got["status"]).tolist())
            for sub in itertools.chain.from_iterable(itertools.combinations(OUTS, r) for r in (1, 2, 3)):
                part = ctx.disparity_fullres(f0, f1, b0, w, h, camera=CAM if {"depth", "xyz"} & set(sub) else None,
                                             outputs=sub, **filt)
                assert_outputs(part, exp, "outputs %s" % (sub,))
            again = ctx.disparity_fullres(f0, f1, b0, w, h, camera=CAM, outputs=OUTS, **filt)
            assert_outputs(again, got, "repeated call")
    # usefbcon's flows pass the left-right test wherever they stay in the frame
    assert seen >= ({0, 2, 4} if fb else {0, 1, 2, 4}), seen
    # the number of launches does not depend on the number of pairs
    for n_pairs in (1, 2 * n):
        before = ctx.launch_count
        ctx.disparity_fullres(0, n_pairs, 0, w, h, lr_check=1, speckle_size=10, fill=1)
        assert ctx.launch_count - before == 7
    assert (bits(fullres(ctx, 0, 2 * n, h, w)) == bits(flows)).all(), "the flows must not change"
    ctx.close()


def test_device_outputs_on_a_caller_stream_in_graph_mode(api):
    import torch

    h, w, n = 121, 203, 2
    prm = small(1, 0)
    frames = synth.synthetic_sequence(n + 1, h, w, 1, seed=37, amp=3.0, stereo=True)
    stream = torch.cuda.Stream()
    ctx = context(api, prm, h, w, 2 * n, stream=stream.cuda_stream)
    ctx.set_graph_mode(True)
    for _ in range(2):  # capture, then replay
        ctx.upload_sequence_bidir_u8(0, n, frames, w, h)
        ctx.run(2 * n)
    flows = fullres(ctx, 0, 2 * n, h, w)
    swapped = [False] * n + [True] * n
    for filt in filters(speckles=((40, 0.05),)):
        exp = expected(flows, 0, n, n, swapped, filt, CAM)
        with torch.cuda.stream(stream):
            dev = {"disp": torch.full((n, h, w), 7.0, device="cuda"),
                   "status": torch.full((n, h, w), 9, dtype=torch.uint8, device="cuda"),
                   "depth": torch.full((n, h, w), 7.0, device="cuda"),
                   "xyz": torch.full((n, h, w, 3), 7.0, device="cuda")}
            ctx.disparity_fullres(0, n, n, w, h, camera=CAM, outputs=OUTS, memkind=api.MEM_DEVICE,
                                  out={k: v.data_ptr() for k, v in dev.items()}, **filt)
        stream.synchronize()
        got = {k: v.cpu().numpy() for k, v in dev.items()}
        assert_outputs(got, exp, "device %s" % filt)
        # host outputs on the same caller stream
        assert_outputs(ctx.disparity_fullres(0, n, n, w, h, camera=CAM, outputs=OUTS, **filt), exp, "host %s" % filt)
    with pytest.raises(ValueError):  # a requested device output without an address
        ctx.disparity_fullres(0, n, n, w, h, outputs=("disp", "status"), memkind=api.MEM_DEVICE,
                              out={"disp": dev["disp"].data_ptr()})
    ctx.close()


@pytest.mark.parametrize("ch", [1, 3])
def test_pairs_followed_by_their_swapped_copies(ch, api):
    """The pair upload of the forward pairs and their swapped copies, the copies marked with set_swapped_slots."""
    h, w, n = 121, 203, 2
    prm = small(ch, 0)
    frames = synth.synthetic_sequence(n + 1, h, w, ch, seed=41, amp=3.0, stereo=True)
    fwd = np.stack([frames[:-1], frames[1:]], axis=1)
    bwd = np.stack([frames[1:], frames[:-1]], axis=1)
    ctx = context(api, prm, h, w, 2 * n)
    ctx.upload_frames_u8(0, 2 * n, np.ascontiguousarray(np.concatenate([fwd, bwd])), w, h)
    ctx.set_swapped_slots(n, 2 * n, 1)
    ctx.run(2 * n)
    flows = fullres(ctx, 0, 2 * n, h, w)
    swapped = [False] * n + [True] * n
    for f0, b0 in ((0, n), (n, 0)):
        for filt in filters(speckles=((30, 0.05),)):
            exp = expected(flows, f0, f0 + n, b0, swapped, filt, CAM)
            assert_outputs(ctx.disparity_fullres(f0, f0 + n, b0, w, h, camera=CAM, outputs=OUTS, **filt), exp,
                           "slots %d.. %s" % (f0, filt))
    ctx.close()


def test_fill_ties_on_the_device(api):
    """Gaps bounded by +0 and -0 along rows and columns (tests/test_disparity.py's map, tiled): the sign of every
    filled zero must be the restatement's, which takes the first (left, upper) of two equal values."""
    from test_disparity import tie_map

    d = np.tile(tie_map(), (8, 16))[:56, :96]
    filt = dict(lr_check=0, alpha=0.0, beta=1.0, speckle_size=0, speckle_diff=1.0, fill=1)
    got = _map_case(api, d, filt)
    assert np.signbit(got["disp"]).any() and not np.signbit(got["disp"]).all()


def _set(ctx, d, slot):
    ctx.set_flow(slot, 0, (-np.asarray(d, np.float32))[..., None])


def _map_case(api, d, filt, partner=None):
    h, w = d.shape
    prm = params.from_cli_numbers("3 0 8 8 0.05 0.95 0 8 0.4 0 1 0 0 10 10 5 1 3 1.6 0".split(), noc=1, nop=1)
    ctx = context(api, prm, h, w, 2)
    assert (ctx.width, ctx.height) == (w, h)
    _set(ctx, d, 0)
    _set(ctx, d if partner is None else partner, 1)
    flows = fullres(ctx, 0, 2, h, w)
    assert (bits(flows[0, ..., 0]) == bits(-np.asarray(d, np.float32))).all()  # sc_l = 0: the map itself
    exp = expected(flows, 0, 1, 1, [False, False], filt, CAM)
    got = ctx.disparity_fullres(0, 1, 1, w, h, camera=CAM, outputs=OUTS, **filt)
    assert_outputs(got, exp, "map")
    ctx.close()
    return got


def test_frame_wide_component_kept_at_its_size(api):
    h, w = 1080, 1920
    y, x = np.mgrid[:h, :w]
    d = (((x // 3 + y // 5) % 4) * 0.5 + 20).astype(np.float32)
    for size, status in ((h * w - 1, 0), (h * w, 4)):
        filt = dict(lr_check=0, alpha=0.0, beta=1.0, speckle_size=size, speckle_diff=1.5, fill=0)
        got = _map_case(api, d, filt)
        assert (got["status"] == status).all()


def test_one_pixel_spiral_across_tile_borders(api):
    h, w = 200, 200
    path = np.zeros((h, w), bool)
    # a one-pixel-wide spiral path with one-pixel gaps between its turns
    y0, x0, y1, x1 = 0, 0, h - 1, w - 1
    while y0 <= y1 and x0 <= x1:
        path[y0, x0:x1 + 1] = True
        path[y0:y1 + 1, x1] = True
        path[y1, x0:x1 + 1] = True
        path[y0 + 2:y1 + 1, x0] = True
        if y0 + 2 <= y1:
            path[y0 + 2, x0:x0 + 3] = True
        y0, x0, y1, x1 = y0 + 2, x0 + 2, y1 - 2, x1 - 2
    d = np.where(path, np.float32(30.0), np.float32(-1.0)).astype(np.float32)  # off the path: d < 0, status 3
    assert ndimage.label(path)[1] == 1 and (path[1:, 1:] & path[:-1, :-1] & ~path[1:, :-1] & ~path[:-1, 1:]).sum() == 0
    npath = int(path.sum())
    for size, status in ((npath - 1, 0), (npath, 4)):
        filt = dict(lr_check=0, alpha=0.0, beta=1.0, speckle_size=size, speckle_diff=0.0, fill=1)
        got = _map_case(api, d, filt)
        assert (got["status"][0][path] == status).all()


def test_checkerboard_every_pixel_alone(api):
    h, w = 96, 160
    y, x = np.mgrid[:h, :w]
    d = np.where((x + y) % 2 == 0, 10.0, 20.0).astype(np.float32)
    for size, fill in ((1, 0), (1, 1), (0, 1)):
        filt = dict(lr_check=1, alpha=0.0, beta=1.0, speckle_size=size, speckle_diff=5.0, fill=fill)
        _map_case(api, d, filt, partner=-d)


def test_components_at_the_threshold_and_special_values(api):
    h, w = 72, 136
    rng = np.random.default_rng(5)
    d = np.full((h, w), 50.0, np.float32)
    # blocks of k pixels at disparity 10 + k, for k around the threshold 6
    for i, k in enumerate((5, 6, 7, 6, 1, 12)):
        r, c = 4 + 10 * i, 3
        d[r, c:c + k] = 10 + k
    d[60, 10], d[60, 11], d[60, 12], d[60, 13] = np.nan, np.inf, -np.inf, 2e9
    d[61, 10], d[61, 11] = 1e9, -0.0
    d[62:, 40:] = rng.uniform(0, 60, (h - 62, w - 40)).astype(np.float32)
    partner = -(d + rng.normal(0, 0.7, d.shape).astype(np.float32))
    partner[~np.isfinite(partner)] = 0
    for lr, fill in ((0, 0), (1, 1), (0, 1)):
        filt = dict(lr_check=lr, alpha=0.0, beta=1.0, speckle_size=6, speckle_diff=0.5, fill=fill)
        got = _map_case(api, d, filt, partner=partner)
        st = got["status"][0]
        if not lr:
            assert (st[4, 3:8] == 4).all() and (st[14, 3:9] == 4).all() and (st[24, 3:10] == 0).all()
        assert (st[60, 10:14] == 3).all() and st[61, 10] != 3 and st[61, 11] != 3


def _status(api, fn, *args, **kw):
    try:
        fn(*args, **kw)
    except api.OfdisError as e:
        return int(re.match(r"status (-?\d+)", str(e)).group(1))
    return 0


def test_bad_arguments(api):
    import ctypes

    h, w, n = 64, 96, 2
    prm = small(1, 0)
    ctx = context(api, prm, h, w, 2 * n)
    ctx.upload_sequence_bidir_u8(0, n, synth.synthetic_sequence(n + 1, h, w, 1, seed=38, stereo=True), w, h)
    ctx.run(2 * n)
    call = ctx.disparity_fullres
    inf, nan = float("inf"), float("nan")
    good = dict(lr_check=1, camera=CAM, outputs=OUTS)
    cases = {
        "f0 < 0": ((-1, 1, n), {}), "f1 > max": ((0, 2 * n + 1, 0), {}), "f0 == f1": ((1, 1, 0), {}),
        "b0 < 0": ((0, n, -1), {}), "b0 + n > max": ((0, n, n + 1), {}),
        "lr 2": ((0, n, n), dict(lr_check=2)), "fill 2": ((0, n, n), dict(fill=2)),
        "alpha < 0": ((0, n, n), dict(alpha=-1.0)), "alpha nan": ((0, n, n), dict(alpha=nan)),
        "beta inf": ((0, n, n), dict(beta=inf)), "speckle < 0": ((0, n, n), dict(speckle_size=-1)),
        "diff nan": ((0, n, n), dict(speckle_diff=nan)), "diff < 0": ((0, n, n), dict(speckle_diff=-0.5)),
        "no camera": ((0, n, n), dict(camera=None)),
        "fx 0": ((0, n, n), dict(camera=dict(CAM, fx=0.0))), "fy inf": ((0, n, n), dict(camera=dict(CAM, fy=inf))),
        "baseline < 0": ((0, n, n), dict(camera=dict(CAM, baseline=-1.0))),
        "cx nan": ((0, n, n), dict(camera=dict(CAM, cx=nan))), "doffs inf": ((0, n, n), dict(camera=dict(CAM, doffs=-inf))),
        "no outputs": ((0, n, n), dict(outputs=())), "width": ((0, n, n), dict(width_org=w + 1)),
        "height": ((0, n, n), dict(height_org=h - 32)),
    }
    for name, (args, kw) in cases.items():
        kw = dict(good, **kw)
        size = (kw.pop("width_org", w), kw.pop("height_org", h))
        assert _status(api, call, *args, *size, **kw) == -1, name
    assert _status(api, call, 0, n, 99, w, h, lr_check=0, outputs=("disp",)) == 0  # b0 is read only with lr_check
    assert _status(api, call, 0, n, n, w, h, outputs=("status",), camera=None) == 0
    L = api.lib()
    filt = api.DispFilter(0, 0.0, 1.0, 0, 1.0, 0)
    assert L.ofdis_disparity_fullres(ctx._h, 0, n, n, None, None, ctypes.c_void_p(256), None, None, None, w, h, 1) == -1
    for k in range(3):  # misaligned device float outputs
        ptrs = [None] * 4
        ptrs[(0, 2, 3)[k]] = ctypes.c_void_p(4096 + 2)
        cam = ctypes.byref(api.StereoCamera(*[CAM[f] for f in preprocess.STEREO_CAMERA_FIELDS]))
        assert L.ofdis_disparity_fullres(ctx._h, 0, n, n, ctypes.byref(filt), cam, *ptrs, w, h, 1) == -1
    ctx.close()
    # flow contexts are refused
    fprm = params.from_cli_numbers("3 1 8 8 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0".split(), noc=1, nop=2)
    fctx = context(api, fprm, h, w, 1)
    assert _status(api, fctx.disparity_fullres, 0, 1, 0, w, h) == -1
    fctx.close()
    # 2^31 pixels per frame or more
    big = params.from_cli_numbers("5 4 8 8 0.05 0.95 0 8 0.4 0 1 0 0 10 10 5 1 3 1.6 0".split(), noc=1, nop=1)
    bctx = api.Context(big, 65536, 32768, big.p_samp_s, 1)
    assert _status(api, bctx.disparity_fullres, 0, 1, 0, 65536, 32768) == -3
    bctx.close()


def test_host_arrays_are_checked(api):
    h, w = 64, 96
    prm = small(1, 0)
    ctx = context(api, prm, h, w, 2)
    ctx.upload_sequence_bidir_u8(0, 1, synth.synthetic_sequence(2, h, w, 1, seed=39, stereo=True), w, h)
    ctx.run(2)
    for out in (dict(disp=np.empty((1, h, w - 1), np.float32)), dict(status=np.empty((1, h, w), np.int8)),
                dict(disp=np.empty((1, h, 2 * w), np.float32)[:, :, ::2])):
        with pytest.raises(ValueError):
            ctx.disparity_fullres(0, 1, 1, w, h, out=out)
    with pytest.raises(ValueError):
        ctx.disparity_fullres(0, 1, 1, w, h, outputs=("mask",))
    disp = np.empty((1, h, w), np.float32)
    assert ctx.disparity_fullres(0, 1, 1, w, h, out=dict(disp=disp))["disp"] is disp
    ctx.close()


# ---- batch command ------------------------------------------------------------------------------------------------
def _write_png(path, img):
    import struct
    import zlib

    h, w = img.shape[:2]
    ch = 1 if img.ndim == 2 else 3
    raw = b"".join(b"\0" + row.tobytes() for row in np.ascontiguousarray(img).reshape(h, w * ch))

    def chunk(t, d):
        return struct.pack(">I", len(d)) + t + d + struct.pack(">I", zlib.crc32(t + d) & 0xFFFFFFFF)

    with open(path, "wb") as f:
        f.write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 0 if ch == 1 else 2, 0, 0, 0)))
        f.write(chunk(b"IDAT", zlib.compress(raw)) + chunk(b"IEND", b""))


def _read_ply(path):
    data = open(path, "rb").read()
    head, body = data.split(b"end_header\n", 1)
    lines = head.decode().splitlines()
    assert lines[:2] == ["ply", "format binary_little_endian 1.0"]
    count = int(lines[2].split()[2])
    assert lines[3:9] == ["property float x", "property float y", "property float z", "property uchar red",
                          "property uchar green", "property uchar blue"]
    rec = np.frombuffer(body, np.dtype([("xyz", "<f4", (3,)), ("rgb", "u1", (3,))]))
    assert rec.size == count
    return rec


@pytest.mark.parametrize("kitti", [False, True], ids=["pfm", "kitti"])
@pytest.mark.parametrize("ch", [1, 3])
def test_batch_command_disparity(tmp_path, ch, kitti, api):
    """A three-frame clip (the two-way sequence upload) and two unrelated pairs (pairs and their swapped copies),
    batches of two.  _filtered, _depth.pfm and .ply equal the Python call; the DISP lines count its statuses; every
    other output keeps its bytes and no _bw file appears without --bidirectional."""
    import os
    import subprocess

    from of_dis_b200 import build

    bindir = build.build_host()
    exe = os.path.join(bindir, ("run_DE_INT" if ch == 1 else "run_DE_RGB") + "_batch")
    h, w = 120, 200
    clip = synth.synthetic_sequence(3, h, w, ch, seed=61, amp=3.0, stereo=True)
    other = synth.synthetic_sequence(3, h, w, ch, seed=62, amp=3.0, stereo=True)
    paths, imgs = {}, {}
    for name, fr in (("a", clip), ("b", other)):
        for t, img in enumerate(fr):
            paths[name, t] = str(tmp_path / ("%s%d.png" % (name, t)))
            imgs[name, t] = img
            _write_png(paths[name, t], img)
    pairs = [("a", 0), ("a", 1), ("b", 1), ("b", 0)]
    cam = dict(fx=300.0, fy=310.0, cx=100.5, cy=59.75, baseline=0.25, doffs=0.5)
    camera = ",".join(repr(cam[k]) for k in preprocess.STEREO_CAMERA_FIELDS)
    flags = ["--lr-check", "--speckle", "30", "0.05", "--fill", "--camera", camera]
    outs, logs = {}, {}
    for tag in ("plain", "disp"):
        outs[tag] = [str(tmp_path / ("%s%d.pfm" % (tag, k))) for k in range(len(pairs))]
        lst = tmp_path / ("%s.txt" % tag)
        lst.write_text("".join("%s %s %s\n" % (paths[nm, t], paths[nm, t + 1], outs[tag][k])
                               for k, (nm, t) in enumerate(pairs)))
        opts = (["--kitti"] if kitti else []) + (flags if tag == "disp" else [])
        r = subprocess.run([exe, str(lst), "--batch", "2"] + opts + ["2"], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        logs[tag] = r.stdout
    prm = params.operating_point(2, w, noc=ch, nop=1)
    bgr = (lambda a: a[..., ::-1]) if ch == 3 else (lambda a: a)  # the decoder holds BGR
    stem = lambda q: os.path.splitext(q)[0]  # noqa: E731
    counts = []
    filt = dict(lr_check=1, alpha=0.0, beta=1.0, speckle_size=30, speckle_diff=0.05, fill=1)
    for k, (nm, t) in enumerate(pairs):
        a, b = bgr(imgs[nm, t]), bgr(imgs[nm, t + 1])
        ctx = context(api, prm, h, w, 2)
        ctx.upload_frames_u8(0, 2, np.ascontiguousarray(np.stack([np.stack([a, b]), np.stack([b, a])])), w, h)
        ctx.set_swapped_slots(1, 2, 1)
        ctx.run(2)
        exp = ctx.disparity_fullres(0, 1, 1, w, h, camera=cam, outputs=OUTS, **filt)
        ctx.close()
        D, Z, xyz = exp["disp"][0], exp["depth"][0], exp["xyz"][0]
        counts.append([int((exp["status"][0] == s).sum()) for s in range(5)] +
                      [int(((exp["status"][0] != 0) & np.isfinite(D)).sum())])
        f = stem(outs["disp"][k]) + "_filtered.pfm"
        if kitti:
            valid = D >= 0  # NaN fails
            enc = np.where(valid, np.clip(np.where(valid, D, 0) * np.float32(256), 1, 65535), 0).astype(np.uint16)
            assert np.array_equal(preprocess.read_kitti_png(f), enc), k
        else:
            assert (bits(-preprocess.read_pfm(f)[..., 0]) == bits(D)).all(), k
        assert (bits(-preprocess.read_pfm(stem(outs["disp"][k]) + "_depth.pfm")[..., 0]) == bits(Z)).all(), k
        rec = _read_ply(stem(outs["disp"][k]) + ".ply")
        keep = np.isfinite(Z)
        assert (bits(rec["xyz"]) == bits(xyz[keep])).all(), k
        img = imgs[nm, t] if ch == 3 else np.repeat(imgs[nm, t][..., None], 3, axis=2)
        assert np.array_equal(rec["rgb"], img[keep]), k
        assert open(outs["plain"][k], "rb").read() == open(outs["disp"][k], "rb").read(), k
        assert not os.path.exists(stem(outs["disp"][k]) + "_bw.pfm")
    lines = [ln for ln in logs["disp"].splitlines() if ln.startswith("DISP")]
    exp_lines = []
    for k0 in (0, 2):
        c = np.sum(counts[k0:k0 + 2], axis=0)
        exp_lines.append("DISP pairs 2 valid %d inconsistent %d leaves %d range %d speckle %d filled %d" % tuple(c))
    assert lines == exp_lines, logs["disp"]
