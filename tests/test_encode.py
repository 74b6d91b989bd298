"""The encodings of ofdis_get_flow_fullres_encoded restated in numpy (preprocess.encode_f16 / encode_kitti), which
tests/test_encode_gpu.py uses as its checker; KITTI's 16-bit PNG files; and the batch command's --kitti grammar and
KITTI ground-truth errors, which are refused before any device work."""
import os
import struct
import subprocess
import zlib

import numpy as np
import pytest

from of_dis_b200 import api, preprocess

f32 = np.float32


def u16(a):
    return np.ascontiguousarray(a).view(np.uint16)


def f32_of_bits(*bits):
    return np.array(bits, np.uint32).view(f32)


# ---- binary16 --------------------------------------------------------------------------------------------------------
def test_f16_equals_numpy_on_numbers():
    rng = np.random.default_rng(1)
    vals = np.concatenate([
        rng.normal(0, 30, 5000).astype(f32),
        rng.normal(0, 3e4, 2000).astype(f32),
        (rng.random(2000) * 2 ** -14).astype(f32) * rng.choice([-1, 1], 2000).astype(f32),  # binary16 subnormals
        np.array([65504, -65504, 65519.996, 65520, -65520, 1e6, -1e6, np.inf, -np.inf, 0.0, -0.0, 2 ** -24,
                  2 ** -25, 2 ** -25 * 1.0001, 3 * 2 ** -26, 1 + 2 ** -11, 1 + 3 * 2 ** -11], f32),
    ])
    with np.errstate(over="ignore"):
        exp = vals.astype(np.float16)
    got = preprocess.encode_f16(vals)
    assert got.dtype == np.float16 and got.shape == vals.shape
    assert (u16(got) == u16(exp)).all()
    special = u16(preprocess.encode_f16(np.array([65504, 65520, -65520, -0.0, 2 ** -25, 1 + 2 ** -11], f32)))
    assert special.tolist() == [0x7BFF, 0x7C00, 0xFC00, 0x8000, 0x0000, 0x3C00]  # ties to even, overflow to inf
    flow = vals[:4000].reshape(10, 20, 10, 2)  # shape kept
    assert (u16(preprocess.encode_f16(flow)) == u16(flow.astype(np.float16))).all()


def test_f16_nan_is_canonical():
    nans = f32_of_bits(0x7FC00000, 0xFFC00000, 0x7FC12345, 0xFFFFFFFF, 0x7F800001, 0xFF800001, 0x7FBFFFFF)
    assert np.isnan(nans).all()
    assert (u16(preprocess.encode_f16(nans)) == preprocess.F16_NAN).all()
    assert u16(nans[:1].astype(np.float16)).tolist() == [preprocess.F16_NAN]  # the library's quiet NaN
    # numpy itself keeps sign and payload, so the restatement has to make the NaN canonical
    assert u16(f32_of_bits(0xFFC00000).astype(np.float16)).tolist() == [0xFE00]
    assert u16(f32_of_bits(0x7FC12345).astype(np.float16)).tolist() == [0x7E09]


# ---- KITTI -------------------------------------------------------------------------------------------------------------
def test_kitti_flow_edges():
    below = f32(512 - 1 / 64)
    vals = [(512, 0), (-512, 0), (below, -below), (-below, below), (1 / 128, -1 / 128), (-0.0, 0.0),
            (1e6, -1e6), (np.inf, -np.inf), (np.nan, 3), (3, np.nan), (np.nan, np.nan), (-513, 600),
            (0.3, -0.3), (1 / 64, -1 / 64)]
    flow = np.array(vals, f32).reshape(1, -1, 2)
    enc = preprocess.encode_kitti(flow)
    assert enc.dtype == np.uint16 and enc.shape == (1, len(vals), 3)
    exp = [(65535, 32768, 1), (0, 32768, 1), (65535, 1, 1), (1, 65535, 1),  # 512 itself is one past the top
           (32768, 32767, 1),  # 32768.5 and 32767.5 truncate
           (32768, 32768, 1), (65535, 0, 1), (65535, 0, 1), (0, 0, 0), (0, 0, 0), (0, 0, 0), (0, 65535, 1),
           (32787, 32748, 1),  # 32787.2 and 32748.8 truncate
           (32769, 32767, 1)]
    assert enc[0].tolist() == [list(e) for e in exp]


def test_kitti_stereo_edges():
    tiny = f32_of_bits(0x00000001)[0]
    F = np.array([-0.0, 0.0, -tiny, tiny, -255.99, -f32(256 - 1 / 256), -256, -300, -1e6, -np.inf, 0.5, 3, np.nan,
                  -1 / 512], f32)
    enc = preprocess.encode_kitti(F[:, None])
    assert enc.shape == F.shape and enc.dtype == np.uint16
    # d = -F: -0 -> +0 and +0 -> -0 are both valid (1); a tiny positive d rounds up to the minimum 1; 255.99 * 256 =
    # 65533.44 truncates; 256 and more clamp to 65535; negative d and NaN are invalid
    assert enc.tolist() == [1, 1, 1, 0, 65533, 65535, 65535, 65535, 65535, 65535, 0, 0, 0, 1]
    # a swapped slot holds the right view: d = +F
    sw = preprocess.encode_kitti(-F[:, None], swapped=True)
    assert sw.tolist() == enc.tolist()
    two = preprocess.encode_kitti(np.stack([F, F])[..., None])  # batches keep their leading axes
    assert two.shape == (2, F.size) and (two == enc).all()


def test_kitti_to_flow_inverts_representable_values():
    rng = np.random.default_rng(2)
    k = rng.integers(0, 65536, (3, 17, 19, 2))
    flow = ((k.astype(np.float64) - 32768) / 64).astype(f32)
    flow[0, 0, 0, 0] = np.nan
    flow[1, 2, 3, 1] = np.nan
    enc = preprocess.encode_kitti(flow)
    back = preprocess.kitti_to_flow(enc, 2)
    assert back.dtype == f32 and back.shape == flow.shape
    invalid = np.isnan(flow).any(-1)
    assert (np.isnan(back) == invalid[..., None]).all()
    assert (back[~invalid] == flow[~invalid]).all()
    assert (back[invalid].view(np.uint32) == 0x7FC00000).all()  # the quiet NaN
    # stereo: d = val / 256 for val in [1, 65535]; the library's sign is -d, and invalid (0) is NaN
    val = rng.integers(0, 65536, (2, 9, 11)).astype(np.uint16)
    d = preprocess.kitti_to_flow(val, 1)
    assert d.shape == val.shape + (1,) and d.dtype == f32
    assert (np.isnan(d[..., 0]) == (val == 0)).all()
    assert (d[val > 0, 0] == -(val[val > 0].astype(np.float64) / 256)).all()
    assert (preprocess.encode_kitti(d) == val).all()
    assert (preprocess.encode_kitti(-d, swapped=True) == val).all()


def test_kitti_to_flow_feeds_flow_error():
    """Invalid KITTI pixels are unknown ground truth for flow_error."""
    enc = np.zeros((4, 5, 3), np.uint16)
    enc[..., 0] = 32768 + 64
    enc[..., 1] = 32768
    enc[:2, :, 2] = 1
    gt = preprocess.kitti_to_flow(enc, 2)
    (s,), err = preprocess.flow_error(np.zeros((4, 5, 2), f32), gt)
    assert s["n"] == 10 and s["sum_err"] == 10.0 and np.isnan(err[2:]).all()


# ---- 16-bit PNG ---------------------------------------------------------------------------------------------------------
def _filter_row(ft, row, prior, bpp):
    """Encoder side of the five PNG filter types (the reader must undo them)."""
    out = bytearray(len(row))
    for x in range(len(row)):
        a = row[x - bpp] if x >= bpp else 0
        b = prior[x]
        c = prior[x - bpp] if x >= bpp else 0
        if ft == 0:
            pred = 0
        elif ft == 1:
            pred = a
        elif ft == 2:
            pred = b
        elif ft == 3:
            pred = (a + b) >> 1
        else:
            p = a + b - c
            pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
            pred = a if (pa <= pb and pa <= pc) else (b if pb <= pc else c)
        out[x] = (row[x] - pred) & 0xFF
    return bytes(out)


def _write_png_filtered(path, enc, filters, chunked=False):
    h, w = enc.shape[:2]
    ch = 3 if enc.ndim == 3 else 1
    rows = np.ascontiguousarray(enc, ">u2").reshape(h, -1).view(np.uint8)
    raw, prior = b"", bytes(w * ch * 2)
    for y in range(h):
        ft = filters[y % len(filters)]
        raw += bytes([ft]) + _filter_row(ft, rows[y].tobytes(), prior, 2 * ch)
        prior = rows[y].tobytes()

    def chunk(t, d):
        return struct.pack(">I", len(d)) + t + d + struct.pack(">I", zlib.crc32(t + d) & 0xFFFFFFFF)

    z = zlib.compress(raw, 9)
    idat = [z[:len(z) // 2], z[len(z) // 2:]] if chunked else [z]
    with open(path, "wb") as f:
        f.write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 16, 2 if ch == 3 else 0, 0, 0, 0)))
        f.write(chunk(b"tEXt", b"Comment\0test"))
        for part in idat:
            f.write(chunk(b"IDAT", part))
        f.write(chunk(b"IEND", b""))


def _random_enc(rng, shape):
    enc = rng.integers(0, 65536, shape).astype(np.uint16)
    enc[::3] = enc[::3] & 0xFF  # rows of small values: neighbouring bytes carry between them
    if len(shape) == 3:
        enc[..., 2] = rng.integers(0, 2, shape[:2])
    return enc


@pytest.mark.parametrize("shape", [(13, 11, 3), (12, 17)], ids=["flow", "stereo"])
def test_png_round_trip(tmp_path, shape):
    rng = np.random.default_rng(3)
    enc = _random_enc(rng, shape)
    p = str(tmp_path / "a.png")
    preprocess.write_kitti_png(p, enc)
    got = preprocess.read_kitti_png(p)
    assert got.dtype == np.uint16 and got.shape == enc.shape and (got == enc).all()
    with open(p, "rb") as f:
        b = f.read()
    assert b[:8] == b"\x89PNG\r\n\x1a\n" and b[12:16] == b"IHDR"
    w, h, depth, ctype, comp, filt, inter = struct.unpack(">IIBBBBB", b[16:29])
    assert (w, h, depth, ctype, comp, filt, inter) == (shape[1], shape[0], 16, 2 if len(shape) == 3 else 0, 0, 0, 0)
    # every filter type, alone and mixed row by row, in one or two IDAT chunks
    for filters in ([0], [1], [2], [3], [4], [4, 3, 2, 1, 0]):
        q = str(tmp_path / ("f%s.png" % "".join(map(str, filters))))
        _write_png_filtered(q, enc, filters, chunked=len(filters) > 1)
        assert (preprocess.read_kitti_png(q) == enc).all(), filters


def test_png_independent_decoder(tmp_path):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(4)
    for shape in ((9, 14, 3), (10, 7)):
        enc = _random_enc(rng, shape)
        p = str(tmp_path / "c.png")
        preprocess.write_kitti_png(p, enc)
        im = cv2.imread(p, cv2.IMREAD_UNCHANGED)
        assert im.dtype == np.uint16
        assert (im[..., ::-1] == enc).all() if len(shape) == 3 else (im == enc).all()  # cv2 returns BGR


def test_png_reader_refusals(tmp_path):
    p = str(tmp_path / "r.png")
    preprocess.write_kitti_png(p, np.zeros((3, 4), np.uint16))
    b = open(p, "rb").read()
    for name, data in (("not a png", b"P5\n1 1\n255\n\0"), ("8-bit", b[:24] + b"\x08" + b[25:])):
        q = str(tmp_path / (name.replace(" ", "_") + ".png"))
        open(q, "wb").write(data)
        with pytest.raises(ValueError):
            preprocess.read_kitti_png(q)
    with pytest.raises(AssertionError):
        preprocess.write_kitti_png(p, np.zeros((3, 4, 2), np.uint16))


def test_encodings_table():
    assert api.ENCODINGS == {"f16": 1, "kitti": 2}
    assert "ofdis_get_flow_fullres_encoded" in api.EXPORTS


# ---- batch front-end: --kitti grammar and KITTI ground-truth errors (all refused before the device is touched) ------
@pytest.fixture(scope="module")
def bindir():
    from of_dis_b200 import build

    return build.build_host()


def _pgm(path, w, h):
    with open(path, "wb") as f:
        f.write(b"P5\n%d %d\n255\n" % (w, h) + bytes(range(w)) * h)


@pytest.mark.parametrize("exe", ["run_OF_INT_batch", "run_DE_RGB_batch"])
def test_batch_command_kitti_grammar(bindir, tmp_path, exe):
    path = os.path.join(bindir, exe)
    stereo = "_DE_" in exe
    for k in range(3):
        _pgm(str(tmp_path / ("i%d.pgm" % k)), 40, 30)
    lst = tmp_path / "list.txt"
    lst.write_text("".join("%s %s %s\n" % (tmp_path / ("i%d.pgm" % k), tmp_path / ("i%d.pgm" % (k + 1)),
                                           tmp_path / ("o%d.png" % k)) for k in range(2)))

    def run(*args):
        return subprocess.run([path, str(lst)] + list(args), capture_output=True, text=True)

    def gtlist(name, paths):
        p = tmp_path / name
        p.write_text(" ".join(paths) + "\n")
        return str(p)

    r = subprocess.run([path], capture_output=True, text=True)
    assert r.returncode == 2 and "--kitti" in r.stderr
    # --kitti is a flag in any position among the options; the others keep their rules
    r = run("--kitti", "--warm-start", "--bidirectional")
    assert r.returncode == 2 and "no --bidirectional" in r.stderr, r.stderr
    r = run("--warm-start", "--kitti", "--batch", "4")
    assert r.returncode == 2 and "no --batch" in r.stderr, r.stderr
    r = run("--kitti", "1", "2")
    assert r.returncode == 2 and "expected 0, 1 or exactly 20 numbers, got 2" in r.stderr, r.stderr
    # KITTI ground truth is checked before any device work: exit 1 with the file and the problem named
    good = np.zeros((30, 40) if stereo else (30, 40, 3), np.uint16)
    g0 = str(tmp_path / "g0.png")
    preprocess.write_kitti_png(g0, good)
    wrong_size = str(tmp_path / "wrong_size.png")
    preprocess.write_kitti_png(wrong_size, good[:, :-1])
    wrong_kind = str(tmp_path / "wrong_kind.png")
    preprocess.write_kitti_png(wrong_kind, np.zeros((30, 40, 3) if stereo else (30, 40), np.uint16))
    eight = str(tmp_path / "eight.png")
    b = bytearray(open(g0, "rb").read())
    b[24] = 8
    open(eight, "wb").write(bytes(b))
    truncated = str(tmp_path / "truncated.png")
    open(truncated, "wb").write(open(g0, "rb").read()[:40])
    for bad, msg in ((wrong_size, "size differs"), (wrong_kind, "KITTI PNG"), (eight, "KITTI PNG"),
                     (truncated, "ground-truth file")):
        r = run("--kitti", "--gt", gtlist("l.txt", [g0, bad]))
        assert r.returncode == 1 and os.path.basename(bad) in r.stderr and msg in r.stderr, (bad, r.stderr)
    assert not any(os.path.exists(str(tmp_path / ("o%d.png" % k))) for k in range(2))
