"""Evaluation against ground truth on the device: ofdis_flow_error_fullres.  Stats and error maps must be BITWISE
what preprocess.flow_error gives on ofdis_get_flow_fullres; the batch command's EVAL lines are recomputed from the
files it wrote."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from of_dis_b200 import params, preprocess, synth

pytestmark = pytest.mark.gpu


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def assert_bits(got, exp, name):
    got, exp = np.asarray(got), np.asarray(exp)
    assert got.shape == exp.shape, (name, got.shape, exp.shape)
    bad = bits(got) != bits(exp)
    if bad.any():
        raise AssertionError("%s: %d of %d values differ bitwise, first at %s" % (name, int(bad.sum()), bad.size,
                                                                                 np.argwhere(bad)[0]))


def assert_stats(got, exp, name):
    assert got.dtype == exp.dtype and got.shape == exp.shape, (name, got.shape, exp.shape)
    assert got.tobytes() == exp.tobytes(), (name, got, exp)


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


def ground_truth(n, h, w, nop, seed):
    """The synthetic flow of the clip (stereo: its disparity), with unknown pixels of every kind sprinkled in."""
    u, v = synth.synthetic_flow(h, w, 3.0, stereo=(nop == 1))
    gt = np.repeat(np.stack([u, v], -1)[None, ..., :nop].astype(np.float32), n, axis=0)
    rng = np.random.default_rng(seed)
    flat = gt.reshape(-1, nop)
    idx = rng.choice(flat.shape[0], 40, replace=False)
    for k, val in zip(idx, [np.nan, np.inf, -np.inf, 1e10, np.float32(1e9)] * 8):
        flat[k, rng.integers(nop)] = val
    return np.ascontiguousarray(gt)


SMALL = "3 %d 8 8 0.05 0.95 0 8 0.4 %d 1 0 1 10 10 5 1 3 1.6 0"


@pytest.mark.parametrize("fb", [0, 1], ids=["fb0", "fb1"])
@pytest.mark.parametrize("size", [(128, 256), (121, 203)], ids=["div", "nondiv"])
@pytest.mark.parametrize("sc_l", [1, 0], ids=["sc_l1", "sc_l0"])
@pytest.mark.parametrize("nop,ch", [(2, 1), (2, 3), (1, 1), (1, 3)])
def test_flow_error_equals_the_restatement(nop, ch, sc_l, size, fb, api):
    """Host and device memory, with and without the map and the classes; sub-ranges; repeated calls; the flows stay."""
    import torch

    h, w = size
    n = 3
    prm = params.from_cli_numbers((SMALL % (sc_l, fb)).split(), noc=ch, nop=nop)
    frames = synth.synthetic_sequence(n + 1, h, w, ch, seed=61, amp=3.0, stereo=(nop == 1))
    ctx = context(api, prm, h, w, n + 1)
    ctx.upload_sequence_u8(0, n, frames, w, h)
    ctx.run(n)
    flows = fullres(ctx, 0, n, h, w, nop)
    gt = ground_truth(n, h, w, nop, seed=62)
    classes = np.random.default_rng(63).integers(0, 5, (n, h, w)).astype(np.uint8)  # 3 and 4 are not counted
    classes[0, :5] = 255
    exp1 = preprocess.flow_error(flows, gt)
    exp3 = preprocess.flow_error(flows, gt, classes, 3)
    assert (exp1[0]["n"] < h * w).all() and (exp1[0]["n_outlier"] > 0).any()

    before = ctx.launch_count
    stats, err = ctx.flow_error_fullres(0, n, gt, w, h, with_err=True)
    assert ctx.launch_count == before + 2
    assert_stats(stats, exp1[0], "host stats")
    assert_bits(err, exp1[1], "host err")
    stats, err = ctx.flow_error_fullres(0, n, gt, w, h, classes=classes, nclasses=3)
    assert err is None
    assert_stats(stats, exp3[0], "host stats, classes")
    again, _ = ctx.flow_error_fullres(0, n, gt, w, h, classes=classes, nclasses=3)
    assert_stats(again, stats, "repeated call")
    if nop == 1:  # stereo ground truth may also come without the channel axis
        st, _ = ctx.flow_error_fullres(0, n, gt[..., 0].copy(), w, h)
        assert_stats(st, exp1[0], "host stats, (n, h, w) ground truth")
    # sub-ranges are the matching rows of the whole range
    for f0, f1 in ((1, 3), (2, 3), (0, 1)):
        st, er = ctx.flow_error_fullres(f0, f1, gt[f0:f1].copy(), w, h, classes=classes[f0:f1].copy(), nclasses=3,
                                        with_err=True)
        assert_stats(st, exp3[0][f0:f1], "slots %d..%d" % (f0, f1))
        assert_bits(er, exp1[1][f0:f1], "slots %d..%d err" % (f0, f1))
    # device memory
    dgt = torch.from_numpy(gt).cuda()
    dcls = torch.from_numpy(classes).cuda()
    derr = torch.full((n, h, w), 7.0, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    st, _ = ctx.flow_error_fullres(0, n, dgt.data_ptr(), w, h, classes=dcls.data_ptr(), nclasses=3,
                                   memkind=api.MEM_DEVICE, err=derr.data_ptr())
    assert_stats(st, exp3[0], "device stats, classes")
    assert_bits(derr.cpu().numpy(), exp1[1], "device err")
    st, _ = ctx.flow_error_fullres(0, n, dgt.data_ptr(), w, h, memkind=api.MEM_DEVICE)
    assert_stats(st, exp1[0], "device stats, no classes, no map")
    assert_bits(fullres(ctx, 0, n, h, w, nop), flows, "flows after the evaluation")
    ctx.close()


@pytest.mark.parametrize("nop", [2, 1])
def test_consistency_mask_as_classes(nop, api):
    """The device mask of a bidirectional run passed straight in as the classes (0 consistent, 1 inconsistent,
    2 leaves the frame)."""
    import torch

    h, w, n = 121, 203, 3
    prm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=1, nop=nop)
    frames = synth.synthetic_sequence(n + 1, h, w, 1, seed=64, amp=3.0, stereo=(nop == 1))
    ctx = context(api, prm, h, w, 2 * n)
    ctx.upload_sequence_bidir_u8(0, n, frames, w, h)
    ctx.run(2 * n)
    flows = fullres(ctx, 0, n, h, w, nop)
    gt = ground_truth(n, h, w, nop, seed=65)
    dmask = torch.empty((n, h, w), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    ctx.consistency_fullres(0, n, n, w, h, memkind=api.MEM_DEVICE, mask=dmask.data_ptr())
    dgt = torch.from_numpy(gt).cuda()
    derr = torch.empty((n, h, w), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    st, _ = ctx.flow_error_fullres(0, n, dgt.data_ptr(), w, h, classes=dmask.data_ptr(), nclasses=3,
                                   memkind=api.MEM_DEVICE, err=derr.data_ptr())
    mask = dmask.cpu().numpy()
    assert {0, 2} <= set(np.unique(mask).tolist()) <= {0, 1, 2}
    exp = preprocess.flow_error(flows, gt, mask, 3)
    assert_stats(st, exp[0], "stats by consistency class")
    assert_bits(derr.cpu().numpy(), exp[1], "err")
    st_host, _ = ctx.flow_error_fullres(0, n, gt, w, h, classes=mask, nclasses=3)
    assert_stats(st_host, exp[0], "host")
    ctx.close()


def _status(api, fn, *args, **kw):
    try:
        fn(*args, **kw)
    except api.OfdisError as e:
        return int(re.match(r"status (-?\d+)", str(e)).group(1))
    return 0


def test_bad_arguments(api):
    h, w, n = 128, 256, 2
    prm = params.operating_point(2, w, noc=1)
    cap = n + 1
    ctx = context(api, prm, h, w, cap)
    ctx.upload_sequence_u8(0, n, synth.synthetic_sequence(n + 1, h, w, 1, seed=66), w, h)
    ctx.run(n)
    gt = np.zeros((cap + 1, h, w, 2), np.float32)
    cls = np.zeros((cap + 1, h, w), np.uint8)
    stats = np.zeros((cap + 1, 16), api.ERROR_STATS_DTYPE)
    L = api.lib()
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731

    def call(f0, f1, g=gt, c=None, nc=1, s=stats, ww=w, hh=h, handle=None):
        return L.ofdis_flow_error_fullres(ctx._h if handle is None else handle, f0, f1, None if g is None else p(g),
                                          None if c is None else p(c), nc, None if s is None else p(s), None, ww, hh,
                                          api.MEM_HOST)

    assert call(0, n) == 0 and call(0, n, c=cls, nc=16) == 0 and call(0, cap, c=cls, nc=2) == 0
    for name, kw in {"f0 < 0": dict(f0=-1, f1=1), "f1 > max_frames": dict(f0=0, f1=cap + 1),
                     "f0 == f1": dict(f0=1, f1=1), "f0 > f1": dict(f0=2, f1=1), "null gt": dict(f0=0, f1=n, g=None),
                     "null stats": dict(f0=0, f1=n, s=None), "nclasses 0": dict(f0=0, f1=n, c=cls, nc=0),
                     "nclasses 17": dict(f0=0, f1=n, c=cls, nc=17), "nclasses -1": dict(f0=0, f1=n, nc=-1),
                     "null classes, nclasses 2": dict(f0=0, f1=n, nc=2),
                     "width": dict(f0=0, f1=n, ww=w + 1), "height": dict(f0=0, f1=n, hh=h - 64),
                     "width 0": dict(f0=0, f1=n, ww=0)}.items():
        assert call(**kw) == -1, name
    assert call(0, n, handle=ctypes.c_void_p()) == -1, "null context"
    # the same through the Python wrapper
    assert _status(api, ctx.flow_error_fullres, 0, n, np.zeros((n, h, w + 1, 2), np.float32), w + 1, h) == -1
    assert _status(api, ctx.flow_error_fullres, 0, n, gt[:n], w, h, classes=cls[:n], nclasses=17) == -1
    assert _status(api, ctx.flow_error_fullres, 0, n, None, w, h, memkind=api.MEM_DEVICE) == -1
    with pytest.raises(ValueError):
        ctx.flow_error_fullres(0, n, gt[:n], w, h, classes=cls[:n])  # nclasses is required with classes
    ctx.close()


def test_host_arrays_are_checked(api):
    h, w, n = 64, 96, 2
    prm = params.from_cli_numbers((SMALL % (1, 0)).split(), noc=1, nop=2)
    ctx = context(api, prm, h, w, n)
    ctx.upload_sequence_u8(0, n, synth.synthetic_sequence(n + 1, h, w, 1, seed=67), w, h)
    ctx.run(n)
    gt = np.zeros((n, h, w, 2), np.float32)
    cls = np.zeros((n, h, w), np.uint8)
    ro = np.empty((n, h, w), np.float32)
    ro.flags.writeable = False
    for kw in (dict(gt=gt.astype(np.float64)), dict(gt=gt[:, :, :-1]), dict(gt=gt[..., 0].copy()),
               dict(gt=np.zeros((n, h, 2 * w, 2), np.float32)[:, :, ::2]), dict(gt=list(gt)),
               dict(classes=cls.astype(np.int8), nclasses=2), dict(classes=cls[:1], nclasses=2),
               dict(classes=np.zeros((n, h, 2 * w), np.uint8)[:, :, ::2], nclasses=2),
               dict(with_err=True, err=np.empty((n, h, w), np.float64)), dict(with_err=True, err=ro),
               dict(with_err=True, err=np.empty((n, h, w - 1), np.float32))):
        args = dict(gt=gt)
        args.update(kw)
        g = args.pop("gt")
        with pytest.raises(ValueError):
            ctx.flow_error_fullres(0, n, g, w, h, **args)
    err = np.empty((n, h, w), np.float32)
    stats, got = ctx.flow_error_fullres(0, n, gt, w, h, with_err=True, err=err)
    assert got is err and stats.shape == (n, 1) and stats.dtype == api.ERROR_STATS_DTYPE
    ctx.close()


def test_large_frames():
    """7680x4352 RGB stereo with the finest level 0: a context frame of more than 2 GB; the evaluation of its slot
    matches the restatement."""
    from of_dis_b200 import api

    prm = params.from_cli_numbers("5 0 8 8 0.05 0.95 0 8 0.4 0 0 0 0 10 10 5 1 3 1.6 0".split(), noc=3, nop=1)
    W, H = 7680, 4352
    ctx = api.Context(prm, W, H, prm.p_samp_s, 1)
    assert ctx.packed_frame_floats * 4 > 2 ** 31
    frames = np.zeros((2, H, W, 3), np.uint8)
    frames[0, :, :W // 2] = 200
    frames[1, :, : W // 2 - 3] = 200
    ctx.upload_frames_u8(0, 1, frames[None], W, H)
    ctx.run(1)
    flow = fullres(ctx, 0, 1, H, W, 1)
    gt = np.full((1, H, W, 1), -3.0, np.float32)
    gt[0, ::97, ::89] = np.nan
    cls = (np.arange(H * W, dtype=np.int64) % 3).astype(np.uint8).reshape(1, H, W)
    stats, err = ctx.flow_error_fullres(0, 1, gt, W, H, classes=cls, nclasses=2, with_err=True)
    exp = preprocess.flow_error(flow, gt, cls, 2)
    assert_stats(stats, exp[0], "stats")
    assert_bits(err, exp[1], "err")
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


def _eval_line(label, pairs, s):
    head = "EVAL %s(%d pairs) n %d" % (label + " " if label else "", pairs, s["n"])
    if s["n"] == 0:
        return head + " epe nan over1 nan over3 nan over5 nan outliers nan"
    n = float(s["n"])
    return head + " epe %.6f over1 %.6f over3 %.6f over5 %.6f outliers %.6f" % (
        s["sum_err"] / n, 100.0 * int(s["n_over"][0]) / n, 100.0 * int(s["n_over"][1]) / n,
        100.0 * int(s["n_over"][2]) / n, 100.0 * int(s["n_outlier"]) / n)


def _add(t, s):
    for k in ("n", "n_outlier", "sum_err"):
        t[k] += s[k]
    t["n_over"] += s["n_over"]


@pytest.mark.parametrize("bidir", [False, True], ids=["forward", "bidirectional"])
@pytest.mark.parametrize("exe,ch,nop,args", [
    ("run_OF_INT", 1, 2, ["2"]),
    ("run_DE_RGB", 3, 1, "3 1 8 8 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 1".split()),
])
def test_batch_command_gt(tmp_path, exe, ch, nop, args, bidir, api):
    """A chain of three pairs and two unrelated ones in batches of 3: the output files are the bytes written without
    --gt, and the EVAL lines are the list-order totals of preprocess.flow_error on the written files (with
    --bidirectional: classes from the written _occ.pgm)."""
    from of_dis_b200 import build

    bindir = build.build_host()
    ext = "flo" if nop == 2 else "pfm"
    h, w = 150, 250
    clip = synth.synthetic_sequence(4, h, w, ch, seed=71, amp=3.0, stereo=(nop == 1))
    other = synth.synthetic_sequence(3, h, w, ch, seed=72, amp=3.0, stereo=(nop == 1))
    paths = {}
    for name, fr in (("a", clip), ("b", other)):
        for t, img in enumerate(fr):
            paths[name, t] = str(tmp_path / ("%s%d.png" % (name, t)))
            _write_png(paths[name, t], img if ch == 1 else img[..., ::-1])
    pairs = [("a", 0), ("a", 1), ("a", 2), ("b", 1), ("b", 0)]
    gts = ground_truth(len(pairs), h, w, nop, seed=73)
    gt_paths = []
    for k in range(len(pairs)):
        gt_paths.append(str(tmp_path / ("gt%d.%s" % (k, ext))))
        (preprocess.write_flo if nop == 2 else preprocess.write_pfm)(gt_paths[-1], gts[k])
    (tmp_path / "truth.txt").write_text("\n".join(gt_paths) + "\n")
    read = preprocess.read_flo if nop == 2 else preprocess.read_pfm
    for k in range(len(pairs)):  # the files hold the ground truth bit for bit (NaN included)
        assert_bits(read(gt_paths[k]), gts[k], "gt file %d" % k)
    outs = {}
    for tag in ("plain", "gt"):
        lst = tmp_path / ("%s.txt" % tag)
        outs[tag] = [str(tmp_path / ("%s%d.%s" % (tag, k, ext))) for k in range(len(pairs))]
        lst.write_text("".join("%s %s %s\n" % (paths[nm, t], paths[nm, t + 1], outs[tag][k])
                               for k, (nm, t) in enumerate(pairs)))
        cmd = [os.path.join(bindir, exe + "_batch"), str(lst), "--batch", "3"] + (["--bidirectional"] if bidir else [])
        cmd += (["--gt", str(tmp_path / "truth.txt")] if tag == "gt" else []) + args
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        if tag == "gt":
            lines = [ln for ln in r.stdout.splitlines() if ln.startswith("EVAL")]
            time_at = [i for i, ln in enumerate(r.stdout.splitlines()) if ln.startswith("TIME")]
            assert time_at and r.stdout.splitlines().index(lines[0]) > time_at[0]
        else:
            assert "EVAL" not in r.stdout
    suffixes = ["", "_bw"] if bidir else [""]
    for k in range(len(pairs)):
        for suf in suffixes:
            a = outs["plain"][k][:-len(ext) - 1] + suf + "." + ext
            b = outs["gt"][k][:-len(ext) - 1] + suf + "." + ext
            assert open(a, "rb").read() == open(b, "rb").read(), (k, suf)
        if bidir:
            occ = lambda o: open(o[:-len(ext) - 1] + "_occ.pgm", "rb").read()  # noqa: E731
            assert occ(outs["plain"][k]) == occ(outs["gt"][k]), k
    # the EVAL lines, recomputed from the files
    nclasses = 3 if bidir else 1
    total = np.zeros(1, api.ERROR_STATS_DTYPE)
    per_class = np.zeros(nclasses, api.ERROR_STATS_DTYPE)
    for k in range(len(pairs)):
        flow = read(outs["gt"][k])
        classes = None
        if bidir:
            pgm = open(outs["gt"][k][:-len(ext) - 1] + "_occ.pgm", "rb").read()
            head = b"P5\n%d %d\n255\n" % (w, h)
            px = np.frombuffer(pgm[len(head):], np.uint8).reshape(h, w)
            classes = np.select([px == 0, px == 255, px == 128], [0, 1, 2], 9).astype(np.uint8)
            assert (classes < 3).all()
        st, _ = preprocess.flow_error(flow, gts[k], classes, nclasses)
        for c in range(nclasses):
            _add(total[0], st[c])
            _add(per_class[c], st[c])
    exp = [_eval_line("", len(pairs), total[0])]
    if bidir:
        exp += [_eval_line(nm, len(pairs), per_class[c]) for c, nm in enumerate(("consistent", "inconsistent", "leaves"))]
    assert lines == exp
