"""ofdis_upload_sequence_u8: the flows of consecutive frames from one upload per frame.  Every pyramid array and
every flow must be BITWISE what ofdis_upload_frames_u8 of the duplicated pairs (frame t, frame t+1) gives, and the
batch front-end's chains must write the single-pair binary's files byte for byte."""
import os
import re
import struct
import subprocess
import zlib

import numpy as np
import pytest

from of_dis_b200 import build, params, preprocess, synth

pytestmark = pytest.mark.gpu

SMALL = "3 1 8 8 0.05 0.95 0 8 0.4 %d 1 0 1 10 10 5 1 3 1.6 0"


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def assert_bits(got, exp, name):
    got, exp = np.asarray(got), np.asarray(exp)
    assert got.shape == exp.shape, (name, got.shape, exp.shape)
    bad = bits(got) != bits(exp)
    # +0/-0 and NaN payloads count as different on purpose
    if bad.any():
        d = np.abs(got.astype(np.float64) - exp.astype(np.float64))
        raise AssertionError("%s: %d of %d values differ bitwise, max-abs %.3e, first at %s" %
                             (name, int(bad.sum()), bad.size, float(np.nanmax(d)), np.argwhere(bad)[0]))


@pytest.fixture(scope="module")
def api():
    from of_dis_b200 import api as _api

    _api.lib()
    return _api


def pairs_of(frames):
    """[n][2][h][w][C] block of the pairs (frame t, frame t+1), as ofdis_upload_frames_u8 takes it."""
    return np.ascontiguousarray(np.stack([frames[:-1], frames[1:]], axis=1))


def geometry(prm, h, w):
    scf = 1 << prm.sc_f
    return (w + scf - 1) // scf * scf, (h + scf - 1) // scf * scf


def context(api, prm, h, w, max_frames):
    W, H = geometry(prm, h, w)
    return api.Context(prm, W, H, prm.p_samp_s, max_frames)


def run_fullres(ctx, n, h, w, nop):
    ctx.run(n)
    out = np.empty((n, h, w, nop), np.float32)
    ctx.get_flow_fullres(0, n, out, w, h)
    ctx.sync()
    return out


@pytest.mark.parametrize("f0", [0, 2])
@pytest.mark.parametrize("n", [1, 3, 5])
@pytest.mark.parametrize("ch,size", [(1, (436, 1024)), (3, (121, 203)), (1, (128, 256))])
def test_sequence_pyramids_equal_the_pair_upload(ch, size, n, f0, api):
    """Every slot, level and array after upload_sequence_u8 == upload_frames_u8 of the duplicated pairs; slots
    outside [f0, f0+n) keep what an earlier upload put there."""
    h, w = size
    prm = params.operating_point(2, w, noc=ch) if w >= 256 else params.from_cli_numbers((SMALL % 0).split(), noc=ch)
    frames = synth.synthetic_sequence(n + 1, h, w, ch, seed=7 + n)
    cap = f0 + n + 1
    earlier = pairs_of(synth.synthetic_sequence(cap + 1, h, w, ch, seed=99))
    a, b = context(api, prm, h, w, cap), context(api, prm, h, w, cap)
    for ctx in (a, b):
        ctx.upload_frames_u8(0, cap, earlier, w, h)
    a.upload_sequence_u8(f0, f0 + n, frames, w, h)
    b.upload_frames_u8(f0, f0 + n, pairs_of(frames), w, h)
    for f in range(cap):
        for lv in range(prm.sc_l, prm.sc_f + 1):
            for which in range(4):
                assert_bits(a.get_level(f, lv, which), b.get_level(f, lv, which), "slot %d level %d array %d" % (f, lv, which))
    a.close()
    b.close()


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("fb", [0, 1], ids=["fb0", "fb1"])
@pytest.mark.parametrize("nop,ch", [(2, 1), (2, 3), (1, 1), (1, 3)])
def test_sequence_flows_equal_the_pair_upload(nop, ch, fb, graph, api):
    """Flow and stereo, gray and RGB, usefbcon 0 and 1 (the swapped backward frames), eager and graph replay."""
    h, w, n = 120, 200, 3
    prm = params.from_cli_numbers((SMALL % fb).split(), noc=ch, nop=nop)
    frames = synth.synthetic_sequence(n + 1, h, w, ch, seed=11, amp=3.0, stereo=(nop == 1))
    out = []
    for seq in (True, False):
        ctx = context(api, prm, h, w, n)
        ctx.set_graph_mode(graph)
        for _ in range(2 if graph else 1):  # graph: capture, then replay
            if seq:
                ctx.upload_sequence_u8(0, n, frames, w, h)
            else:
                ctx.upload_frames_u8(0, n, pairs_of(frames), w, h)
            out.append(run_fullres(ctx, n, h, w, nop))
        ctx.close()
    for k in range(1, len(out)):
        assert_bits(out[k], out[0], "run %d" % k)


def test_sequence_level_flows_equal_the_oracle(api, oracle_port):
    h, w, n = 120, 200, 3
    prm = params.from_cli_numbers((SMALL % 1).split(), noc=1, nop=2)
    frames = synth.synthetic_sequence(n + 1, h, w, 1, seed=12, amp=3.0)
    ctx = context(api, prm, h, w, n)
    ctx.upload_sequence_u8(0, n, frames, w, h)
    ctx.run(n)
    for t in range(n):
        pyr = preprocess.PairPyramids(frames[t], frames[t + 1], prm.sc_f, prm.p_samp_s)
        assert_bits(ctx.get_flow(t, prm.sc_l), oracle_port.port_run(pyr, prm), "pair %d" % t)
    ctx.close()


def test_streaming_in_chunks_equals_one_call_and_the_pair_path(api):
    """9 frames as two chunks of 4 pairs (frame 4 sent twice) == one 8-pair call == the pair path."""
    h, w, nop = 128, 256, 2
    prm = params.operating_point(2, w, noc=1)
    frames = synth.synthetic_sequence(9, h, w, 1, seed=13)
    ctx = context(api, prm, h, w, 4)
    chunks = []
    for c in range(2):
        ctx.upload_sequence_u8(0, 4, np.ascontiguousarray(frames[4 * c:4 * c + 5]), w, h)
        chunks.append(run_fullres(ctx, 4, h, w, nop))
    ctx.close()
    streamed = np.concatenate(chunks)
    ctx = context(api, prm, h, w, 8)
    ctx.upload_sequence_u8(0, 8, frames, w, h)
    assert_bits(run_fullres(ctx, 8, h, w, nop), streamed, "one call")
    ctx.upload_frames_u8(0, 8, pairs_of(frames), w, h)
    assert_bits(run_fullres(ctx, 8, h, w, nop), streamed, "pair path")
    ctx.close()


def test_device_input_equals_host_input(api):
    import torch

    h, w, n, ch = 121, 203, 3, 3
    prm = params.from_cli_numbers((SMALL % 0).split(), noc=ch)
    frames = synth.synthetic_sequence(n + 1, h, w, ch, seed=14, amp=3.0)
    dev = torch.from_numpy(frames).cuda()
    a, b = context(api, prm, h, w, n), context(api, prm, h, w, n)
    a.upload_sequence_u8(0, n, frames, w, h)
    torch.cuda.synchronize()
    b.upload_sequence_u8(0, n, dev.data_ptr(), w, h, memkind=api.MEM_DEVICE)
    for f in range(n):
        for lv in range(prm.sc_l, prm.sc_f + 1):
            for which in range(4):
                assert_bits(b.get_level(f, lv, which), a.get_level(f, lv, which), "slot %d level %d array %d" % (f, lv, which))
    assert_bits(run_fullres(b, n, h, w, 2), run_fullres(a, n, h, w, 2), "flows")
    a.close()
    b.close()


def _status(api, fn, *args):
    try:
        fn(*args)
    except api.OfdisError as e:
        return int(re.match(r"status (-?\d+)", str(e)).group(1))
    return 0


def test_bad_arguments_give_the_status_of_the_pair_upload(api):
    h, w, n = 128, 256, 3
    prm = params.operating_point(2, w, noc=1)
    ctx = context(api, prm, h, w, n)
    frames = synth.synthetic_sequence(n + 1, h, w, 1, seed=15)
    pairs = pairs_of(frames)
    cases = {"f0 < 0": (-1, 2, w, h), "f1 > max_frames": (0, n + 1, w, h), "f0 == f1": (1, 1, w, h),
             "f0 > f1": (2, 1, w, h), "null": (0, n, w, h), "width": (0, n, w + 1, h), "height": (0, n, w, h - 64)}
    for name, (f0, f1, ww, hh) in cases.items():
        sa = None if name == "null" else frames
        sb = None if name == "null" else pairs
        got = _status(api, ctx.upload_sequence_u8, f0, f1, sa, ww, hh)
        exp = _status(api, ctx.upload_frames_u8, f0, f1, sb, ww, hh)
        assert got == exp == -1, (name, got, exp)
    ctx.close()
    # finest level above 8: the box sums are no longer exact in float32
    prm = params.from_cli_numbers("9 9 4 4 0.05 0.95 0 4 0.4 0 1 0 0 10 10 5 1 3 1.6 0".split(), noc=1)
    ctx = api.Context(prm, 1024, 512, prm.p_samp_s, 1)
    one = np.zeros((2, 512, 1024), np.uint8)
    got = _status(api, ctx.upload_sequence_u8, 0, 1, one, 1024, 512)
    exp = _status(api, ctx.upload_frames_u8, 0, 1, one[None], 1024, 512)
    assert got == exp == -3, (got, exp)
    ctx.close()


# ---- batch front-end ------------------------------------------------------------------------------------------------
def write_png(path, img):
    """8-bit gray or RGB PNG, filter type 0."""
    h, w = img.shape[:2]
    ch = 1 if img.ndim == 2 else 3
    raw = b"".join(b"\0" + row.tobytes() for row in np.ascontiguousarray(img).reshape(h, w * ch))

    def chunk(t, d):
        return struct.pack(">I", len(d)) + t + d + struct.pack(">I", zlib.crc32(t + d) & 0xFFFFFFFF)

    with open(path, "wb") as f:
        f.write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 0 if ch == 1 else 2, 0, 0, 0)))
        f.write(chunk(b"IDAT", zlib.compress(raw)) + chunk(b"IEND", b""))


def _clip(tmp_path, name, n_frames, h, w, ch, seed, stereo):
    frames = synth.synthetic_sequence(n_frames, h, w, ch, seed=seed, amp=3.0, stereo=stereo)
    paths = []
    for t, img in enumerate(frames):
        paths.append(str(tmp_path / ("%s%d.png" % (name, t))))
        write_png(paths[-1], img if ch == 1 else img[..., ::-1])  # files store RGB, the pipeline works in BGR
    return paths


@pytest.mark.parametrize("exe,ch,nop,args", [
    ("run_OF_INT", 1, 2, ["2"]),
    # 20 numbers, usefbcon = 1, verbosity 1
    ("run_DE_RGB", 3, 1, "3 1 8 8 0.05 0.95 0 8 0.4 1 1 0 1 10 10 5 1 3 1.6 1".split()),
])
def test_batch_front_end_chains_write_the_files_of_the_single_pair_binary(tmp_path, exe, ch, nop, args):
    """A 7-frame chain at 218x500 split across batches, a break, a 3-frame chain at 150x250, one unchained pair."""
    bindir = build.build_host()
    ext = "flo" if nop == 2 else "pfm"
    a = _clip(tmp_path, "a", 7, 218, 500, ch, 31, nop == 1)
    b = _clip(tmp_path, "b", 3, 150, 250, ch, 32, nop == 1)
    c = _clip(tmp_path, "c", 2, 218, 500, ch, 33, nop == 1)
    pairs = [(a[t], a[t + 1]) for t in range(6)] + [(b[0], b[1]), (b[1], b[2]), (c[0], c[1])]
    outs = [str(tmp_path / ("batch%d.%s" % (k, ext))) for k in range(len(pairs))]
    lst = tmp_path / "list.txt"
    lst.write_text("".join("%s %s %s\n" % (p, q, o) for (p, q), o in zip(pairs, outs)))
    r = subprocess.run([os.path.join(bindir, exe + "_batch"), str(lst), "--batch", "4"] + args, capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "TIME (9 pairs" in r.stdout
    # batches [a0..a4] [a4..a6] [b0..b2] [c0 c1]: a4 is decoded once, c is a single pair
    assert "SEQUENCE (8 of 9 pairs from 10 decoded frames)" in r.stdout, r.stdout
    for k, ((p, q), o) in enumerate(zip(pairs, outs)):
        single = o + ".single"
        r = subprocess.run([os.path.join(bindir, exe), p, q, single] + args, capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        assert open(single, "rb").read() == open(o, "rb").read(), k
    # no chain: no SEQUENCE line
    lst.write_text("%s %s %s\n%s %s %s\n" % (a[0], a[1], outs[0], a[2], a[3], outs[1]))
    r = subprocess.run([os.path.join(bindir, exe + "_batch"), str(lst)] + args, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "TIME (2 pairs" in r.stdout and "SEQUENCE" not in r.stdout
