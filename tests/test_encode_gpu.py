"""Encoded full-resolution flows on the device: ofdis_get_flow_fullres_encoded.  Every output must be BITWISE what
preprocess.encode_f16 / encode_kitti give on ofdis_get_flow_fullres; the batch command's --kitti files decode to the
encoding of the files it writes without the flag, and KITTI ground truth gives the EVAL lines of its .flo / .pfm."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from of_dis_b200 import params, preprocess, synth

pytestmark = pytest.mark.gpu


def u16(a):
    return np.ascontiguousarray(a).view(np.uint16)


def assert_u16(got, exp, name):
    got, exp = u16(got), u16(exp)
    assert got.shape == exp.shape, (name, got.shape, exp.shape)
    bad = got != exp
    if bad.any():
        i = tuple(np.argwhere(bad)[0])
        raise AssertionError("%s: %d of %d values differ, first at %s: %#06x, expected %#06x"
                             % (name, int(bad.sum()), bad.size, i, int(got[i]), int(exp[i])))


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


def expected(flows, enc, swapped=None):
    """The restatement of each slot; `swapped` marks (stereo KITTI) per slot."""
    if enc == "f16":
        return preprocess.encode_f16(flows)
    sw = [False] * len(flows) if swapped is None else swapped
    return np.stack([preprocess.encode_kitti(f, bool(s)) for f, s in zip(flows, sw)])


def device_encoded(api, ctx, f0, f1, enc, h, w, nop):
    """The encoding into a caller-owned device tensor (f16: torch.float16, as a user would pass it)."""
    import torch

    if enc == "f16":
        t = torch.full((f1 - f0, h, w, nop), 7.0, dtype=torch.float16, device="cuda")
    else:
        t = torch.full((f1 - f0, h, w) + ((3,) if nop == 2 else ()), 7, dtype=torch.int16, device="cuda")
    torch.cuda.synchronize()
    assert ctx.get_flow_fullres_encoded(f0, f1, enc, w, h, out=t.data_ptr(), memkind=api.MEM_DEVICE) == t.data_ptr()
    ctx.sync()
    return t.cpu().numpy().view(np.uint16).view(np.float16 if enc == "f16" else np.uint16)


SMALL = "3 %d 8 8 0.05 0.95 0 8 0.4 %d 1 0 1 10 10 5 1 3 1.6 0"


@pytest.mark.parametrize("fb", [0, 1], ids=["fb0", "fb1"])
@pytest.mark.parametrize("size", [(128, 256), (121, 203)], ids=["div", "nondiv"])
@pytest.mark.parametrize("sc_l", [1, 0], ids=["sc_l1", "sc_l0"])
@pytest.mark.parametrize("nop,ch", [(2, 1), (2, 3), (1, 1), (1, 3)])
def test_encoded_equals_the_restatement(nop, ch, sc_l, size, fb, api):
    """Both encodings on host and device memory, sub-ranges away from slot 0, repeated and alternating calls; the flows
    stay as they were."""
    h, w = size
    n = 3
    prm = params.from_cli_numbers((SMALL % (sc_l, fb)).split(), noc=ch, nop=nop)
    frames = synth.synthetic_sequence(n + 1, h, w, ch, seed=81, amp=3.0, stereo=(nop == 1))
    ctx = context(api, prm, h, w, n + 1)
    ctx.upload_sequence_u8(0, n, frames, w, h)
    ctx.run(n)
    flows = fullres(ctx, 0, n, h, w, nop)
    for enc in ("f16", "kitti"):
        exp = expected(flows, enc)
        before = ctx.launch_count
        got = ctx.get_flow_fullres_encoded(0, n, enc, w, h)
        assert ctx.launch_count == before + 1
        assert_u16(got, exp, "%s host" % enc)
        assert got.dtype == (np.float16 if enc == "f16" else np.uint16)
        for f0, f1 in ((1, 3), (2, 3), (1, 2)):
            assert_u16(ctx.get_flow_fullres_encoded(f0, f1, enc, w, h), exp[f0:f1], "%s host %d..%d" % (enc, f0, f1))
            assert_u16(device_encoded(api, ctx, f0, f1, enc, h, w, nop), exp[f0:f1], "%s device %d..%d" % (enc, f0, f1))
        assert_u16(device_encoded(api, ctx, 0, n, enc, h, w, nop), exp, "%s device" % enc)
        assert_u16(fullres(ctx, 0, n, h, w, nop), flows, "float flows between the encodings")
    ctx.close()


def _extremes(nop, h, w, rng):
    """Level flows that reach every clamp, both roundings at the limits, NaN, the infinities and -0."""
    big = [1e6, -1e6, np.inf, -np.inf, np.nan, -0.0, 0.0, 65504, 65519.996, 65520, -65520, 2 ** -24, 2 ** -25]
    kitti_flow = [511.984375, 512, 512.015625, -512, -512.015625, -511.984375, 1 / 128, -1 / 128, 1 / 64]
    kitti_stereo = [255.99609375, 256, 256.5, -255.99609375, -256, -256.5, 1 / 512, -1 / 512, 2 ** -149, -2 ** -149]
    vals = np.array(big + kitti_flow + kitti_stereo, np.float32)
    nan_bits = np.array([0x7FC00000, 0xFFC00000, 0x7FC12345, 0xFF800001], np.uint32).view(np.float32)
    vals = np.concatenate([vals, nan_bits, rng.normal(0, 200, 32).astype(np.float32)])
    flow = rng.choice(vals, (h, w, nop)).astype(np.float32)
    flow.reshape(-1)[:vals.size] = vals  # every value at least once, and next to each other
    return flow


@pytest.mark.parametrize("sc_l", [0, 1], ids=["sc_l0", "sc_l1"])
@pytest.mark.parametrize("nop", [2, 1])
def test_extreme_level_flows(nop, sc_l, api):
    """Level flows written with set_flow and encoded without a run: the clamps, NaN of every sign and payload, the
    infinities, -0 and the values around the 512 px (flow) and 256 px (stereo) limits; stereo slots marked swapped
    encode +F."""
    h, w, n = 64, 96, 4
    prm = params.from_cli_numbers(("2 %d 8 8 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0" % sc_l).split(), noc=1,
                                  nop=nop)
    ctx = context(api, prm, h, w, n)
    rng = np.random.default_rng(82)
    lh, lw = ctx.height >> sc_l, ctx.width >> sc_l
    for f in range(n):
        ctx.set_flow(f, sc_l, _extremes(nop, lh, lw, rng))
    if nop == 1:
        ctx.set_swapped_slots(1, 3, 1)
    flows = fullres(ctx, 0, n, h, w, nop)
    assert np.isnan(flows).any() and np.isinf(flows).any()
    swapped = [False, True, True, False] if nop == 1 else None
    for enc in ("f16", "kitti"):
        exp = expected(flows, enc, swapped)
        assert_u16(ctx.get_flow_fullres_encoded(0, n, enc, w, h), exp, "%s host" % enc)
        assert_u16(device_encoded(api, ctx, 1, n, enc, h, w, nop), exp[1:], "%s device" % enc)
    if sc_l == 0:  # the level flow is the full-resolution flow: every special value reaches the encoder as it is
        e16 = u16(ctx.get_flow_fullres_encoded(0, 1, "f16", w, h))
        assert {0x7E00, 0x7C00, 0xFC00, 0x8000, 0x7BFF} <= set(e16.reshape(-1).tolist())
        assert not ({0xFE00, 0x7E09} & set(e16.reshape(-1).tolist()))
        ek = ctx.get_flow_fullres_encoded(0, n, "kitti", w, h)
        assert {0, 1, 65535} <= set(ek.reshape(-1).tolist())
    assert_u16(fullres(ctx, 0, n, h, w, nop), flows, "flows after the encodings")
    ctx.close()


def test_swapped_slots_of_a_two_way_upload(api):
    """Stereo: the backward slots of upload_sequence_bidir_u8 hold the right view (marked swapped) and encode +F, so
    both views give KITTI's positive disparities."""
    h, w, n = 121, 203, 3
    prm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=1, nop=1)
    frames = synth.synthetic_sequence(n + 1, h, w, 1, seed=83, amp=3.0, stereo=True)
    ctx = context(api, prm, h, w, 2 * n)
    ctx.upload_sequence_bidir_u8(0, n, frames, w, h)
    ctx.run(2 * n)
    flows = fullres(ctx, 0, 2 * n, h, w, 1)
    assert (flows[:n] <= 0).mean() > 0.9 and (flows[n:] >= 0).mean() > 0.9
    got = ctx.get_flow_fullres_encoded(0, 2 * n, "kitti", w, h)
    assert_u16(got, expected(flows, "kitti", [False] * n + [True] * n), "kitti, both views")
    assert (got[n:] > 0).mean() > 0.9  # the right view's disparities are valid
    assert_u16(device_encoded(api, ctx, n, 2 * n, "kitti", h, w, 1), got[n:], "device, right view")
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
    ctx.upload_sequence_u8(0, n, synth.synthetic_sequence(n + 1, h, w, 1, seed=84), w, h)
    ctx.run(n)
    buf = np.zeros((cap + 1) * h * w * 3 + 8, np.uint16)
    dev = torch.zeros((cap + 1) * h * w * 3 + 8, dtype=torch.int16, device="cuda")
    torch.cuda.synchronize()
    L = api.lib()
    host = buf.ctypes.data

    def call(f0, f1, enc=2, out=host, ww=w, hh=h, mem=api.MEM_HOST, handle=None):
        return L.ofdis_get_flow_fullres_encoded(ctx._h if handle is None else handle, f0, f1, enc,
                                                None if out is None else ctypes.c_void_p(out), ww, hh, mem)

    assert call(0, n) == 0 and call(0, cap, enc=1) == 0 and call(1, cap) == 0
    assert call(0, n, out=host + 1) == 0  # host output may sit anywhere
    assert call(0, n, out=dev.data_ptr(), mem=api.MEM_DEVICE) == 0
    assert call(0, n, out=dev.data_ptr() + 2, mem=api.MEM_DEVICE) == 0
    for name, kw in {"encoding 0": dict(f0=0, f1=n, enc=0), "encoding 3": dict(f0=0, f1=n, enc=3),
                     "encoding -1": dict(f0=0, f1=n, enc=-1), "null out": dict(f0=0, f1=n, out=None),
                     "null device out": dict(f0=0, f1=n, out=None, mem=api.MEM_DEVICE),
                     "odd device out": dict(f0=0, f1=n, out=dev.data_ptr() + 1, mem=api.MEM_DEVICE),
                     "f0 < 0": dict(f0=-1, f1=1), "f1 > max_frames": dict(f0=0, f1=cap + 1),
                     "f0 == f1": dict(f0=1, f1=1), "f0 > f1": dict(f0=2, f1=1),
                     "width": dict(f0=0, f1=n, ww=w + 1), "height": dict(f0=0, f1=n, hh=h - 64),
                     "width 0": dict(f0=0, f1=n, ww=0), "height -1": dict(f0=0, f1=n, hh=-1)}.items():
        assert call(**kw) == -1, name
    assert call(0, n, handle=ctypes.c_void_p()) == -1, "null context"
    torch.cuda.synchronize()
    # the same through the Python wrapper
    assert _status(api, ctx.get_flow_fullres_encoded, 0, n, "kitti", w + 1, h) == -1
    assert _status(api, ctx.get_flow_fullres_encoded, 0, cap + 1, "f16", w, h) == -1
    assert _status(api, ctx.get_flow_fullres_encoded, 0, n, "f16", w, h, memkind=api.MEM_DEVICE) == -1
    with pytest.raises(ValueError):
        ctx.get_flow_fullres_encoded(0, n, "png", w, h)
    ctx.close()


def test_host_out_is_checked(api):
    h, w, n = 64, 96, 2
    for nop in (2, 1):
        prm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=1, nop=nop)
        ctx = context(api, prm, h, w, n)
        ctx.upload_sequence_u8(0, n, synth.synthetic_sequence(n + 1, h, w, 1, seed=85, stereo=(nop == 1)), w, h)
        ctx.run(n)
        kshape = (n, h, w, 3) if nop == 2 else (n, h, w)
        ro = np.empty(kshape, np.uint16)
        ro.flags.writeable = False
        for enc, bad in (("f16", np.empty((n, h, w, nop), np.uint16)), ("f16", np.empty((n, h, w, nop), np.float32)),
                         ("f16", np.empty((n, h, w + 1, nop), np.float16)), ("f16", np.empty((n, h, w), np.float16)),
                         ("kitti", np.empty(kshape, np.int16)), ("kitti", np.empty((n - 1,) + kshape[1:], np.uint16)),
                         ("kitti", np.empty((n, h, 2 * w) + kshape[3:], np.uint16)[:, :, ::2]), ("kitti", ro),
                         ("kitti", list(np.empty(kshape, np.uint16))), ("kitti", np.empty((n, h, w, 2), np.uint16))):
            with pytest.raises(ValueError):
                ctx.get_flow_fullres_encoded(0, n, enc, w, h, out=bad)
        out = np.empty(kshape, np.uint16)
        got = ctx.get_flow_fullres_encoded(0, n, "kitti", w, h, out=out)
        assert got is out
        assert_u16(out, expected(fullres(ctx, 0, n, h, w, nop), "kitti"), "given out, nop %d" % nop)
        ctx.close()


# ---- batch front-end --------------------------------------------------------------------------------------------
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


@pytest.mark.parametrize("exe,nop,bidir", [("run_OF_INT", 2, False), ("run_DE_INT", 1, True), ("run_OF_INT", 2, True)],
                         ids=["flow", "stereo-bidirectional", "flow-bidirectional"])
def test_batch_command_kitti(tmp_path, exe, nop, bidir, api):
    """A chain of three pairs and two unrelated ones in batches of 3.  With --kitti the outputs are PNGs (named .png
    and, for one pair, with the .flo/.pfm extension) whose samples are encode_kitti of what the same list writes
    without it; the masks keep their bytes.  --gt with KITTI PNG ground truth prints the EVAL lines of the .flo / .pfm
    ground truth that kitti_to_flow gives, NaN where the PNG is invalid."""
    from of_dis_b200 import build

    bindir = build.build_host()
    ext = "flo" if nop == 2 else "pfm"
    h, w = 150, 250
    clip = synth.synthetic_sequence(4, h, w, 1, seed=86, amp=3.0, stereo=(nop == 1))
    other = synth.synthetic_sequence(3, h, w, 1, seed=87, amp=3.0, stereo=(nop == 1))
    paths = {}
    for name, fr in (("a", clip), ("b", other)):
        for t, img in enumerate(fr):
            paths[name, t] = str(tmp_path / ("%s%d.png" % (name, t)))
            _write_png(paths[name, t], img)
    pairs = [("a", 0), ("a", 1), ("a", 2), ("b", 1), ("b", 0)]
    # KITTI ground truth: the synthetic flow, quantised by the encoding, with invalid pixels
    u, v = synth.synthetic_flow(h, w, 3.0, stereo=(nop == 1))
    base = np.stack([u, v], -1)[..., :nop].astype(np.float32)
    rng = np.random.default_rng(88)
    gt_png, gt_float = [], []
    for k in range(len(pairs)):
        enc = preprocess.encode_kitti(base + rng.normal(0, 0.5, base.shape).astype(np.float32))
        enc[rng.random((h, w)) < 0.2] = 0  # invalid
        gt_png.append(str(tmp_path / ("gt%d.png" % k)))
        preprocess.write_kitti_png(gt_png[-1], enc)
        gt_float.append(str(tmp_path / ("gt%d.%s" % (k, ext))))
        (preprocess.write_flo if nop == 2 else preprocess.write_pfm)(gt_float[-1], preprocess.kitti_to_flow(enc, nop))
    runs = {"plain": ext, "kitti": "png", "kitti_gt": "png", "plain_gt": ext}
    outs, evals = {}, {}
    for tag, oext in runs.items():
        outs[tag] = [str(tmp_path / ("%s%d.%s" % (tag, k, oext if k != 4 else ext))) for k in range(len(pairs))]
        lst = tmp_path / ("%s.txt" % tag)
        lst.write_text("".join("%s %s %s\n" % (paths[nm, t], paths[nm, t + 1], outs[tag][k])
                               for k, (nm, t) in enumerate(pairs)))
        cmd = [os.path.join(bindir, exe + "_batch"), str(lst), "--batch", "3"] + (["--bidirectional"] if bidir else [])
        if tag.endswith("_gt"):
            gl = tmp_path / ("%s_list.txt" % tag)
            gl.write_text("\n".join(gt_png if tag.startswith("kitti") else gt_float) + "\n")
            cmd += ["--gt", str(gl)]
        cmd += (["--kitti"] if tag.startswith("kitti") else []) + ["2"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        evals[tag] = [ln for ln in r.stdout.splitlines() if ln.startswith("EVAL")]
    assert evals["kitti_gt"] and evals["kitti_gt"] == evals["plain_gt"]
    read = preprocess.read_flo if nop == 2 else preprocess.read_pfm
    with_suffix = lambda p, s, e=None: os.path.splitext(p)[0] + s + (e or os.path.splitext(p)[1])  # noqa: E731
    for k in range(len(pairs)):
        ref = read(outs["plain"][k])
        for tag in ("kitti", "kitti_gt"):
            got = preprocess.read_kitti_png(outs[tag][k])
            assert_u16(got, preprocess.encode_kitti(ref), "%s pair %d" % (tag, k))
            if bidir:
                bw = preprocess.read_kitti_png(with_suffix(outs[tag][k], "_bw"))
                assert_u16(bw, preprocess.encode_kitti(read(with_suffix(outs["plain"][k], "_bw")), swapped=True),
                           "%s pair %d backward" % (tag, k))
                if nop == 1:
                    assert (bw > 0).mean() > 0.9  # the right view's disparities are positive
                occ = lambda p: open(with_suffix(p, "_occ", ".pgm"), "rb").read()  # noqa: E731
                assert occ(outs[tag][k]) == occ(outs["plain"][k])
        # without --kitti the bytes do not depend on --gt
        assert open(outs["plain"][k], "rb").read() == open(outs["plain_gt"][k], "rb").read()
