"""Bidirectional flows and consistency masks: ofdis_upload_sequence_bidir_u8, ofdis_set_swapped_slots and
ofdis_consistency_fullres.  Every pyramid, flow and mask must be BITWISE what the existing paths give: the pair
upload of the forward and the swapped pairs, a right-camera context for stereo, the oracle driven level by level as
the right camera, and preprocess.consistency_check on ofdis_get_flow_fullres."""
import ctypes
import re

import numpy as np
import pytest

from of_dis_b200 import params, preprocess, synth

pytestmark = pytest.mark.gpu

SMALL = "3 1 8 8 0.05 0.95 0 8 0.4 %d 1 0 1 10 10 5 1 3 1.6 0"


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def assert_bits(got, exp, name):
    got, exp = np.asarray(got), np.asarray(exp)
    assert got.shape == exp.shape, (name, got.shape, exp.shape)
    bad = bits(got) != bits(exp)
    if bad.any():
        raise AssertionError("%s: %d of %d values differ bitwise, first at %s" % (name, int(bad.sum()), bad.size,
                                                                                 np.argwhere(bad)[0]))


@pytest.fixture(scope="module")
def api():
    from of_dis_b200 import api as _api

    _api.lib()
    return _api


def fwd_pairs(frames):
    return np.ascontiguousarray(np.stack([frames[:-1], frames[1:]], axis=1))


def bwd_pairs(frames):
    return np.ascontiguousarray(np.stack([frames[1:], frames[:-1]], axis=1))


def context(api, prm, h, w, max_frames):
    scf = 1 << prm.sc_f
    W, H = (w + scf - 1) // scf * scf, (h + scf - 1) // scf * scf
    return api.Context(prm, W, H, prm.p_samp_s, max_frames)


def fullres(ctx, f0, f1, h, w, nop):
    out = np.empty((f1 - f0, h, w, nop), np.float32)
    ctx.get_flow_fullres(f0, f1, out, w, h)
    ctx.sync()
    return out


def small(nop, ch, fb):
    return params.from_cli_numbers((SMALL % fb).split(), noc=ch, nop=nop)


@pytest.mark.parametrize("fb", [0, 1], ids=["fb0", "fb1"])
@pytest.mark.parametrize("f0", [0, 2])
@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("ch", [1, 3])
def test_bidir_pyramids_equal_the_pair_upload(ch, n, f0, fb, api):
    """Every slot, level and array == upload_frames_u8 of the forward and the swapped pairs; the slot behind
    [f0, f0+2n) (and those before it) keep what an earlier upload put there."""
    h, w = 121, 203
    prm = small(2, ch, fb)
    frames = synth.synthetic_sequence(n + 1, h, w, ch, seed=40 + n)
    cap = f0 + 2 * n + 1
    earlier = fwd_pairs(synth.synthetic_sequence(cap + 1, h, w, ch, seed=98))
    a, b = context(api, prm, h, w, cap), context(api, prm, h, w, cap)
    for ctx in (a, b):
        ctx.upload_frames_u8(0, cap, earlier, w, h)
    a.upload_sequence_bidir_u8(f0, n, frames, w, h)
    b.upload_frames_u8(f0, f0 + n, fwd_pairs(frames), w, h)
    b.upload_frames_u8(f0 + n, f0 + 2 * n, bwd_pairs(frames), w, h)
    for f in range(cap):
        for lv in range(prm.sc_l, prm.sc_f + 1):
            for which in range(4):
                assert_bits(a.get_level(f, lv, which), b.get_level(f, lv, which), "slot %d level %d array %d" % (f, lv, which))
    a.close()
    b.close()


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("fb", [0, 1], ids=["fb0", "fb1"])
@pytest.mark.parametrize("nop,ch", [(2, 1), (2, 3), (1, 1), (1, 3)])
def test_bidir_flows(nop, ch, fb, graph, api):
    """Forward slots == the one-way sequence run; backward slots == a run of the swapped pairs (stereo: marked
    swapped, and without usefbcon also == a context set to the right camera)."""
    h, w, n = 120, 200, 3
    prm = small(nop, ch, fb)
    frames = synth.synthetic_sequence(n + 1, h, w, ch, seed=21, amp=3.0, stereo=(nop == 1))
    reps = 2 if graph else 1  # graph: capture, then replay

    def runs(setup, nslots):
        ctx = context(api, prm, h, w, nslots)
        ctx.set_graph_mode(graph)
        outs = []
        for _ in range(reps):
            setup(ctx)
            ctx.run(nslots)
            outs.append(fullres(ctx, 0, nslots, h, w, nop))
        ctx.close()
        for k in range(1, reps):
            assert_bits(outs[k], outs[0], "replay %d" % k)
        return outs[0]

    both = runs(lambda c: c.upload_sequence_bidir_u8(0, n, frames, w, h), 2 * n)
    assert_bits(both[:n], runs(lambda c: c.upload_sequence_u8(0, n, frames, w, h), n), "forward slots")

    def swapped(c):
        c.upload_frames_u8(0, n, bwd_pairs(frames), w, h)
        if nop == 1:
            c.set_swapped_slots(0, n, 1)

    assert_bits(both[n:], runs(swapped, n), "backward slots")
    if nop == 1 and not fb:
        def right_camera(c):
            c.set_camlr(1)
            c.upload_frames_u8(0, n, bwd_pairs(frames), w, h)

        assert_bits(both[n:], runs(right_camera, n), "backward slots against camlr 1")
    if nop == 1:
        # the mark matters: the same pairs as the left camera give other disparities
        left = runs(lambda c: c.upload_frames_u8(0, n, bwd_pairs(frames), w, h), n)
        assert (bits(left) != bits(both[n:])).any()


def _right_camera_oracle(pyr, prm):
    """The oracle's level loop (dis_run_fb without usefbcon) with every level made as the right camera."""
    from oracle import port_driver as pd

    lib, cp = pd.lib(), prm.to_c()
    fp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_float)) if a is not None else None  # noqa: E731
    prev = None
    for sl in range(prm.sc_f, prm.sc_l - 1, -1):
        L = pd.make_level(pyr, prm, sl, camlr=1)
        n_p = L.nopw * L.noph
        p = np.zeros((n_p, prm.nop), np.float32)
        pw = np.zeros((n_p, prm.noc * prm.p_samp_s ** 2), np.float32)
        conv, cnt = np.zeros(n_p, np.int32), np.zeros(n_p, np.int32)
        lib.dis_patches_level(ctypes.byref(L), ctypes.byref(cp), fp(pyr.i0[sl]), fp(pyr.i0x[sl]), fp(pyr.i0y[sl]),
                              fp(pyr.i1[sl]), fp(prev), fp(p), fp(pw), conv.ctypes.data_as(ctypes.POINTER(ctypes.c_int)),
                              cnt.ctypes.data_as(ctypes.POINTER(ctypes.c_int)))
        dense = np.zeros((L.h, L.w, prm.nop), np.float32)
        lib.dis_densify(ctypes.byref(L), ctypes.byref(cp), fp(p), fp(pw), fp(dense))
        if prm.usetvref:
            lib.dis_varref_level(ctypes.byref(L), ctypes.byref(cp), fp(pyr.i0[sl]), fp(pyr.i1[sl]), fp(dense))
        prev = dense
    return prev


def test_backward_stereo_slots_equal_the_right_camera_oracle(api, oracle_port):
    h, w, n = 120, 200, 2
    prm = small(1, 1, 0)
    frames = synth.synthetic_sequence(n + 1, h, w, 1, seed=22, amp=3.0, stereo=True)
    ctx = context(api, prm, h, w, 2 * n)
    ctx.upload_sequence_bidir_u8(0, n, frames, w, h)
    ctx.run(2 * n)
    for t in range(n):
        pyr = preprocess.PairPyramids(frames[t + 1], frames[t], prm.sc_f, prm.p_samp_s)
        exp = _right_camera_oracle(pyr, prm)
        got = ctx.get_flow(n + t, prm.sc_l)
        assert_bits(got, exp, "backward pair %d" % t)
        assert (got >= 0).all()  # the right camera's disparities are clamped to >= 0
    ctx.close()


def test_graph_replay_follows_the_marks(api):
    h, w, n = 120, 200, 2
    prm = small(1, 1, 0)
    frames = synth.synthetic_sequence(n + 1, h, w, 1, seed=23, amp=3.0, stereo=True)
    ref = {}
    for graph in (False, True):
        ctx = context(api, prm, h, w, n)
        ctx.set_graph_mode(graph)
        ctx.upload_frames_u8(0, n, bwd_pairs(frames), w, h)
        for mark in (0, 1, 0, 1):
            ctx.set_swapped_slots(0, n, mark)
            ctx.run(n)
            out = fullres(ctx, 0, n, h, w, 1)
            if graph:
                assert_bits(out, ref[mark], "graph, mark %d" % mark)
            else:
                ref.setdefault(mark, out)
                assert_bits(out, ref[mark], "eager, mark %d" % mark)
        ctx.close()
    assert (bits(ref[0]) != bits(ref[1])).any()


@pytest.mark.parametrize("fb", [0, 1], ids=["fb0", "fb1"])
@pytest.mark.parametrize("size", [(128, 256), (121, 203)], ids=["div", "nondiv"])
@pytest.mark.parametrize("nop", [2, 1])
@pytest.mark.parametrize("sc_l", [1, 0], ids=["sc_l1", "sc_l0"])
def test_consistency_equals_the_restatement(sc_l, nop, size, fb, api):
    """sc_l = 0 takes the upsampling's integer-pixel path (level flow read at the crop offsets), sc_l = 1 the
    interpolated one."""
    import torch

    h, w = size
    n = 3
    prm = params.from_cli_numbers(("3 %d 8 8 0.05 0.95 0 8 0.4 %d 1 0 1 10 10 5 1 3 1.6 0" % (sc_l, fb)).split(),
                                  noc=1, nop=nop)
    frames = synth.synthetic_sequence(n + 1, h, w, 1, seed=24, amp=3.0, stereo=(nop == 1))
    ctx = context(api, prm, h, w, 2 * n)
    ctx.upload_sequence_bidir_u8(0, n, frames, w, h)
    ctx.run(2 * n)
    flows = fullres(ctx, 0, 2 * n, h, w, nop)
    seen = set()
    for alpha, beta in ((None, None), (0.05, 0.25), (0.0, 0.0)):
        da, db = api.CONSISTENCY_DEFAULTS[nop]
        a_, b_ = (da, db) if alpha is None else (alpha, beta)
        for f0, b0 in ((0, n), (n, 0)):  # forward against backward, and the other way round
            exp = [preprocess.consistency_check(flows[f0 + i], flows[b0 + i], a_, b_) for i in range(n)]
            before = ctx.launch_count
            mask, err = ctx.consistency_fullres(f0, f0 + n, b0, w, h, alpha, beta, with_err=True)
            assert ctx.launch_count == before + 1
            for i in range(n):
                assert (mask[i] == exp[i][0]).all(), (alpha, f0, i, int((mask[i] != exp[i][0]).sum()))
                assert_bits(err[i], exp[i][1], "err %d" % i)
            m2, e2 = ctx.consistency_fullres(f0, f0 + n, b0, w, h, alpha, beta)
            assert e2 is None and (m2 == mask).all()
            dm = torch.empty((n, h, w), dtype=torch.uint8, device="cuda")
            de = torch.empty((n, h, w), dtype=torch.float32, device="cuda")
            torch.cuda.synchronize()
            ctx.consistency_fullres(f0, f0 + n, b0, w, h, alpha, beta, memkind=api.MEM_DEVICE, mask=dm.data_ptr(),
                                    err=de.data_ptr())
            ctx.sync()
            assert (dm.cpu().numpy() == mask).all()
            assert_bits(de.cpu().numpy(), err, "device err")
            seen |= set(np.unique(mask).tolist())
    assert seen == {0, 1, 2}, "the case should exercise every outcome"
    assert_bits(fullres(ctx, 0, 2 * n, h, w, nop), flows, "flows after the check")
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
    cap = 2 * n + 1
    ctx = context(api, prm, h, w, cap)
    frames = synth.synthetic_sequence(n + 1, h, w, 1, seed=25)
    up = ctx.upload_sequence_bidir_u8
    for name, args in {"f0 < 0": (-1, n, frames, w, h), "n < 1": (0, 0, frames, w, h),
                       "f0 + 2n > max_frames": (2, n, frames, w, h), "null": (0, n, None, w, h),
                       "width": (0, n, frames, w + 1, h), "height": (0, n, frames, w, h - 64)}.items():
        assert _status(api, up, *args) == -1, name
    for name, args in {"f0 < 0": (-1, 1, 1), "f1 > max_frames": (0, cap + 1, 1), "f0 == f1": (1, 1, 1),
                       "swapped 2": (0, 1, 2), "swapped -1": (0, 1, -1)}.items():
        assert _status(api, ctx.set_swapped_slots, *args) == -1, name
    up(0, n, frames, w, h)
    ctx.run(2 * n)
    cons = ctx.consistency_fullres
    inf, nan = float("inf"), float("nan")
    for name, (args, kw) in {
            "f0 < 0": ((-1, 1, n, w, h), {}), "f1 > max_frames": ((0, cap + 1, 0, w, h), {}),
            "f0 == f1": ((1, 1, 0, w, h), {}), "b0 < 0": ((0, n, -1, w, h), {}),
            "b0 + n > max_frames": ((0, n, cap - 1, w, h), {}),
            "null mask": ((0, n, n, w, h), dict(memkind=api.MEM_DEVICE)),
            "alpha < 0": ((0, n, n, w, h), dict(alpha=-0.1)), "alpha nan": ((0, n, n, w, h), dict(alpha=nan)),
            "alpha inf": ((0, n, n, w, h), dict(alpha=inf)), "beta < 0": ((0, n, n, w, h), dict(beta=-1.0)),
            "beta nan": ((0, n, n, w, h), dict(beta=nan)), "beta inf": ((0, n, n, w, h), dict(beta=inf)),
            "width": ((0, n, n, w + 1, h), {}), "height": ((0, n, n, w, h - 64), {})}.items():
        assert _status(api, cons, *args, **kw) == -1, name
    assert _status(api, cons, 0, n, n, w, h) == 0
    ctx.close()
    # finest level above 8: the box sums are no longer exact in float32
    prm = params.from_cli_numbers("9 9 4 4 0.05 0.95 0 4 0.4 0 1 0 0 10 10 5 1 3 1.6 0".split(), noc=1)
    ctx = api.Context(prm, 1024, 512, prm.p_samp_s, 2)
    assert _status(api, ctx.upload_sequence_bidir_u8, 0, 1, np.zeros((2, 512, 1024), np.uint8), 1024, 512) == -3
    ctx.close()


def test_host_arrays_are_checked(api):
    h, w, n = 64, 96, 1
    prm = small(2, 1, 0)
    ctx = context(api, prm, h, w, 2 * n)
    ctx.upload_sequence_bidir_u8(0, n, synth.synthetic_sequence(n + 1, h, w, 1, seed=26), w, h)
    ctx.run(2 * n)
    for kw in (dict(mask=np.empty((n, h, w - 1), np.uint8)), dict(mask=np.empty((n, h, w), np.int8)),
               dict(mask=np.empty((n, h, 2 * w), np.uint8)[:, :, ::2]),
               dict(with_err=True, err=np.empty((n, h, w), np.float64))):
        with pytest.raises(ValueError):
            ctx.consistency_fullres(0, n, n, w, h, **kw)
    mask, err = np.empty((n, h, w), np.uint8), np.empty((n, h, w), np.float32)
    got = ctx.consistency_fullres(0, n, n, w, h, with_err=True, mask=mask, err=err)
    assert got[0] is mask and got[1] is err
    ctx.close()


def test_large_frames_are_still_accepted(api):
    """7680x4352 RGB with the finest level 0: a frame of more than 2 GB, which a context takes as before (the
    swapped marks are reached in 16-byte units); a stereo pass over a marked slot reads them."""
    prm = params.from_cli_numbers("5 0 8 8 0.05 0.95 0 8 0.4 0 0 0 0 10 10 5 1 3 1.6 0".split(), noc=3, nop=1)
    ctx = api.Context(prm, 7680, 4352, prm.p_samp_s, 1)
    assert ctx.packed_frame_floats * 4 > 2 ** 31
    frames = np.zeros((2, 4352, 7680, 3), np.uint8)
    frames[1, :, 100:] = 255
    ctx.upload_frames_u8(0, 1, frames[None], 7680, 4352)
    ctx.set_swapped_slots(0, 1, 1)
    ctx.run(1)
    assert (ctx.get_flow(0, prm.sc_l) >= 0).all()  # run as the right camera: disparities clamped to >= 0
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


@pytest.mark.parametrize("exe,ch,nop,args", [
    ("run_OF_INT", 1, 2, ["2"]),
    ("run_DE_RGB", 3, 1, "3 1 8 8 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 1".split()),
])
def test_batch_command_bidirectional(tmp_path, exe, ch, nop, args, api):
    """A list with a 4-frame chain (one batch: two-way sequence upload) and two unrelated pairs (pair upload of the
    pairs and their swapped copies): forward files are the bytes written without the flag, backward files the
    C-ABI's backward runs, written as the binaries write them, and _occ.pgm the restatement on the written flows."""
    import os
    import subprocess

    from of_dis_b200 import build

    bindir = build.build_host()
    ext = "flo" if nop == 2 else "pfm"
    h, w = 150, 250
    clip = synth.synthetic_sequence(4, h, w, ch, seed=51, amp=3.0, stereo=(nop == 1))
    other = synth.synthetic_sequence(3, h, w, ch, seed=52, amp=3.0, stereo=(nop == 1))
    paths = {}
    for name, fr in (("a", clip), ("b", other)):
        for t, img in enumerate(fr):
            paths[name, t] = str(tmp_path / ("%s%d.png" % (name, t)))
            _write_png(paths[name, t], img if ch == 1 else img[..., ::-1])  # files store RGB, the pipeline BGR
    pairs = [(clip, "a", 0), (clip, "a", 1), (clip, "a", 2), (other, "b", 0), (other, "b", 1)]
    lst_fw, lst_bi = tmp_path / "fw.txt", tmp_path / "bi.txt"
    outs_fw = [str(tmp_path / ("fw%d.%s" % (k, ext))) for k in range(len(pairs))]
    outs_bi = [str(tmp_path / ("bi%d.%s" % (k, ext))) for k in range(len(pairs))]
    # the b pairs are listed apart so that they are not a chain: b1->b2 after a2->a3, then b0->b1
    order = [0, 1, 2, 4, 3]
    for lst, outs in ((lst_fw, outs_fw), (lst_bi, outs_bi)):
        lst.write_text("".join("%s %s %s\n" % (paths[pairs[k][1], pairs[k][2]], paths[pairs[k][1], pairs[k][2] + 1],
                                                 outs[k]) for k in order))
    exe_path = os.path.join(bindir, exe + "_batch")
    r = subprocess.run([exe_path, str(lst_fw), "--batch", "3"] + args, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    r = subprocess.run([exe_path, str(lst_bi), "--batch", "3", "--bidirectional"] + args, capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    prm = params.from_cli_numbers(args, noc=ch, nop=nop) if len(args) == 20 else \
        params.operating_point(int(args[0]), w, noc=ch, nop=nop)
    read = preprocess.read_flo if nop == 2 else preprocess.read_pfm
    alpha, beta = api.CONSISTENCY_DEFAULTS[nop]
    levels = np.array([0, 255, 128], np.uint8)
    for k, (fr, name, t) in enumerate(pairs):
        assert open(outs_bi[k], "rb").read() == open(outs_fw[k], "rb").read(), k
        stem = outs_bi[k][:-len(ext) - 1]
        bw = read(stem + "_bw." + ext)
        # the C-ABI's backward run of this pair: the swapped pair, marked swapped
        ctx = context(api, prm, h, w, 1)
        ctx.upload_frames_u8(0, 1, bwd_pairs(fr[t:t + 2]), w, h)
        ctx.set_swapped_slots(0, 1, 1)
        ctx.run(1)
        assert_bits(bw, fullres(ctx, 0, 1, h, w, nop)[0], "backward file %d" % k)
        ctx.close()
        mask, _ = preprocess.consistency_check(read(outs_bi[k]), bw, alpha, beta)
        pgm = open(stem + "_occ.pgm", "rb").read()
        head = b"P5\n%d %d\n255\n" % (w, h)
        assert pgm.startswith(head) and pgm[len(head):] == levels[mask].tobytes(), k
