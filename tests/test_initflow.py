"""Init flow from a full-resolution flow (the reference's commented-out file input, run_dense.cpp:292-301,355-378),
on CPU: the restatement preprocess.initflow_from_fullres against cv2, the C oracle's run from that init flow against
the reference build (SHA-256 digests in golden/initflow_digests.json, written by golden/make_initflow_golden.py, and
the build itself where it exists), and the
command lines' argument and file errors, which all fail before any device is touched."""
import ctypes
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

from of_dis_b200 import build, params, preprocess, synth
from oracle import ref_driver

GOLDEN_DIR = os.path.join(os.path.dirname(__file__), "golden")
DIGESTS_PATH = os.path.join(GOLDEN_DIR, "initflow_digests.json")

# name: (h, w, channels, cli numbers with %d = usefbcon, nop).  Sizes where the 2^(sc_f+1) padding differs from the
# 2^sc_f padding; the last case has sc_f = 0, s = 2 with one channel (OpenCV's SIMD-body order).
CASES = {
    "flow_gray_fb0": (120, 200, 1, "3 1 12 12 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 2),
    "flow_gray_fb1": (120, 200, 1, "3 1 8 8 0.05 0.95 0 8 0.4 1 1 0 1 10 10 5 1 3 1.6 0", 2),
    "flow_rgb_fb0": (104, 184, 3, "3 1 16 16 0.05 0.95 0 12 0.75 0 1 1 1 10 10 5 1 3 1.6 0", 2),
    "flow_rgb_fb1": (104, 184, 3, "3 1 8 8 0.05 0.95 0 12 0.75 1 1 1 1 10 10 5 1 3 1.6 0", 2),
    "stereo_gray_fb0": (96, 232, 1, "3 1 24 24 0.05 0.95 0 12 0.75 0 1 0 1 10 10 5 1 3 1.6 0", 1),
    "stereo_gray_fb1": (96, 232, 1, "3 1 12 12 0.05 0.95 0 8 0.4 1 1 0 1 10 10 5 1 3 1.6 0", 1),
    "stereo_rgb_fb0": (90, 170, 3, "2 0 12 12 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 1),
    "stereo_gray_s2": (61, 91, 1, "0 0 8 8 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 1),
}


def digest(a, dtype=np.float32):
    a = np.ascontiguousarray(a, dtype)
    return "%s:%s" % ("x".join(map(str, a.shape)), hashlib.sha256(a.tobytes()).hexdigest())


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def fullres_flow(h, w, nop, seed):
    """A full-resolution init flow near the synthetic ground truth: flow (h, w, 2) or disparity (h, w, 1) <= 0."""
    u, v = synth.synthetic_flow(h, w, 4.0, stereo=(nop == 1))
    rng = np.random.default_rng(seed)
    gt = np.stack([u, v], -1)[..., :nop]
    fl = gt * 0.8 + rng.standard_normal(gt.shape) * 0.3
    if nop == 1:
        fl = -np.abs(fl)
    return np.ascontiguousarray(fl, np.float32)


def initflow_inputs(name):
    """(img0, img1, pyr padded to 2^(sc_f+1), prm, full-resolution init flow, its level sc_f+1)."""
    h, w, ch, cli, nop = CASES[name]
    prm = params.from_cli_numbers(cli.split(), noc=ch, nop=nop)
    i0, i1, _ = synth.synthetic_pair(h, w, ch, seed=50 + len(name), amp=4.0, stereo=(nop == 1))
    pyr = preprocess.PairPyramids(i0, i1, prm.sc_f, prm.p_samp_s, div_level=prm.sc_f + 1)
    fl = fullres_flow(h, w, nop, seed=len(name))
    return i0, i1, pyr, prm, fl, preprocess.initflow_from_fullres(fl, prm.sc_f)


def ref_run_initflow(pyr, prm, initflow):
    """The reference's OFClass constructor on one pair with `initflow` (level sc_f+1)."""
    lib = ref_driver._lib(prm.flavour())
    h, w = pyr.level_shape(prm.sc_l)
    out = np.zeros((h, w, prm.nop), dtype=np.float32)
    init = np.ascontiguousarray(initflow, np.float32)
    cp = prm.to_c()
    ptrs = [ref_driver._pyr_ptrs(x) for x in (pyr.i0, pyr.i0x, pyr.i0y, pyr.i1, pyr.i1x, pyr.i1y)]
    lib.ofdis_ref_run(*ptrs, ctypes.c_int(pyr.imgpadding), ref_driver._fp(out), ref_driver._fp(init),
                      ctypes.c_int(pyr.width), ctypes.c_int(pyr.height), ctypes.byref(cp))
    return out


def make_digests():
    out = {}
    for name in CASES:
        i0, i1, pyr, prm, fl, init = initflow_inputs(name)
        out[name + "_input"] = digest(np.stack([i0, i1]), np.uint8)
        out[name + "_initflow_fullres"] = digest(fl)
        out[name + "_initflow"] = digest(init)
        out[name + "_run"] = digest(ref_run_initflow(pyr, prm, init))
    return out


# ---- the restatement against cv2 ------------------------------------------------------------------------------------
def _cv2_area(fl, lv_f):
    """flow * 2^-(lv_f+1) (after the replicate padding), then cv2.resize(INTER_AREA) by 2^(lv_f+1)."""
    cv2 = pytest.importorskip("cv2")
    s = 2 ** (lv_f + 1)
    v = preprocess.pad_to_multiple(fl, lv_f + 1)[0] * np.float32(2.0 ** -(lv_f + 1))
    src = v if v.shape[2] == 2 else v[..., 0]
    return cv2.resize(np.ascontiguousarray(src), None, fx=1.0 / s, fy=1.0 / s, interpolation=cv2.INTER_AREA)


def _sequential_s2(fl, lv_f):
    """s = 2, one channel, in the order of OpenCV's scalar tail: 0 + (((a + b) + c) + d), times 0.25."""
    v = preprocess.pad_to_multiple(fl, lv_f + 1)[0][..., 0] * np.float32(0.5)
    a, b, c, d = v[0::2, 0::2], v[0::2, 1::2], v[1::2, 0::2], v[1::2, 1::2]
    return ((np.float32(0) + (((a + b) + c) + d)) * np.float32(0.25)).astype(np.float32)


@pytest.mark.parametrize("nop", [1, 2])
@pytest.mark.parametrize("lv_f", [0, 1, 2, 3, 4, 5])
@pytest.mark.parametrize("size", [(64, 128), (37, 101), (130, 77)], ids=["divisible", "pad_odd", "pad_tall"])
def test_initflow_from_fullres_equals_cv2(size, lv_f, nop):
    h, w = size
    s = 2 ** (lv_f + 1)
    rng = np.random.default_rng(lv_f * 10 + nop)
    fl = (rng.standard_normal((h, w, nop)) * 20).astype(np.float32)
    # blocks whose terms are all -0 sum to -0: the sum's 0 start makes them +0
    fl[:min(h, s), :min(w, s)] = -0.0
    got = preprocess.initflow_from_fullres(fl, lv_f)
    H, W = -(-h // s), -(-w // s)
    assert got.shape == (H, W, nop) and got.dtype == np.float32
    exp = _cv2_area(fl, lv_f).reshape(got.shape)
    if s == 2 and nop == 1:
        # cv2: the SIMD body ((a + b) + (c + d)) * 0.25, the scalar tail (last columns, build-dependent) the
        # sequential order.  Compare where cv2 is one function of the block (both orders agree); elsewhere cv2 must
        # be one of the two, and the restatement is the SIMD body's.
        seq = _sequential_s2(fl, lv_f).reshape(got.shape)
        same = bits(seq) == bits(got)
        assert np.array_equal(bits(exp)[same], bits(got)[same])
        assert np.all((bits(exp) == bits(got)) | (bits(exp) == bits(seq)))
        assert bits(got)[0, 0, 0] == bits(np.float32(-0.0))  # the SIMD body keeps -0
        return
    assert np.array_equal(bits(got), bits(exp)), np.argwhere(bits(got) != bits(exp))[:5]
    assert bits(got)[0, 0, 0] == 0  # +0


def test_initflow_from_fullres_accepts_a_disparity_plane():
    fl = np.random.default_rng(1).standard_normal((33, 50)).astype(np.float32)
    assert np.array_equal(bits(preprocess.initflow_from_fullres(fl, 2)),
                          bits(preprocess.initflow_from_fullres(fl[..., None], 2)))


def test_read_pfm_is_the_inverse_of_write_pfm(tmp_path):
    d = np.random.default_rng(2).standard_normal((17, 23, 1)).astype(np.float32)
    d[0, 0, 0], d[1, 1, 0] = -0.0, 0.0
    p = str(tmp_path / "d.pfm")
    preprocess.write_pfm(p, d)
    got = preprocess.read_pfm(p)
    assert got.shape == (17, 23, 1) and np.array_equal(bits(got), bits(d))
    q = str(tmp_path / "e.pfm")
    preprocess.write_pfm(q, got)
    assert open(p, "rb").read() == open(q, "rb").read()


def test_pair_pyramids_take_the_divisibility_level():
    i0, i1, _ = synth.synthetic_pair(120, 200, 1, seed=3)
    a = preprocess.PairPyramids(i0, i1, 3, 8)
    b = preprocess.PairPyramids(i0, i1, 3, 8, div_level=3)
    c = preprocess.PairPyramids(i0, i1, 3, 8, div_level=4)
    assert (a.width, a.height) == (b.width, b.height) == (200, 120)
    assert (c.width, c.height, c.padw, c.padh) == (208, 128, 8, 8)


# ---- the oracle against the reference build ------------------------------------------------------------------------
@pytest.fixture(scope="module")
def digests():
    with open(DIGESTS_PATH) as f:
        return json.load(f)


@pytest.mark.parametrize("name", list(CASES))
def test_port_run_from_initflow_equals_reference_digests(name, oracle_port, digests):
    DIGESTS = digests
    i0, i1, pyr, prm, fl, init = initflow_inputs(name)
    assert digest(np.stack([i0, i1]), np.uint8) == DIGESTS[name + "_input"], "synthetic inputs moved"
    assert digest(fl) == DIGESTS[name + "_initflow_fullres"], "synthetic init flow moved"
    assert digest(init) == DIGESTS[name + "_initflow"]
    got = oracle_port.port_run(pyr, prm, init)
    assert digest(got) == DIGESTS[name + "_run"]
    # the init flow changes the result (the run does start from it)
    assert digest(got) != digest(oracle_port.port_run(pyr, prm))


@pytest.mark.parametrize("name", list(CASES))
def test_port_run_from_initflow_equals_the_reference_build(name, oracle_port):
    h, w, ch, cli, nop = CASES[name]
    flavour = params.from_cli_numbers(cli.split(), noc=ch, nop=nop).flavour()
    if not ref_driver.ref_available(flavour):
        pytest.skip("oracle/_ref not built")
    _, _, pyr, prm, _, init = initflow_inputs(name)
    assert np.array_equal(bits(oracle_port.port_run(pyr, prm, init)), bits(ref_run_initflow(pyr, prm, init)))


# ---- command-line errors (before any device work) ------------------------------------------------------------------
NUMS = "3 1 8 8 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0".split()


@pytest.fixture(scope="module")
def bindir():
    return build.build_host()


@pytest.fixture()
def images(tmp_path):
    paths = []
    for k in range(2):
        p = str(tmp_path / ("i%d.pgm" % k))
        with open(p, "wb") as f:
            f.write(b"P5\n40 30\n255\n" + bytes(range(40)) * 30)
        paths.append(p)
    return paths


def _flo(path, w, h, data=None, tag=b"PIEH"):
    with open(path, "wb") as f:
        f.write(tag + np.array([w, h], "<i4").tobytes())
        f.write((np.zeros((h, w, 2), "<f4") if data is None else data).tobytes())


def _run(bindir, exe, images, out, extra):
    return subprocess.run([os.path.join(bindir, exe)] + images + [out] + NUMS + extra, capture_output=True, text=True)


def test_cli_argument_counts(bindir, images, tmp_path):
    out = str(tmp_path / "o.flo")
    for extra in (["1"], ["0", "x.flo"], ["1", "a.flo", "b"]):
        r = _run(bindir, "run_OF_INT", images, out, extra)
        assert r.returncode == 2, (extra, r.stderr)
    r = subprocess.run([os.path.join(bindir, "run_OF_INT_batch"), "list.txt", "--warm-start", "--batch", "4"],
                       capture_output=True, text=True)
    assert r.returncode == 2 and "--warm-start" in r.stderr
    r = subprocess.run([os.path.join(bindir, "run_OF_INT_batch")], capture_output=True, text=True)
    assert r.returncode == 2 and "--warm-start" in r.stderr


@pytest.mark.parametrize("exe,case,message", [
    ("run_OF_INT", "missing", "cannot read the init-flow file"),
    ("run_OF_INT", "tag", "not a .flo file"),
    ("run_OF_INT", "size", "size differs"),
    ("run_OF_INT", "short", "length does not match"),
    ("run_OF_INT", "long", "length does not match"),
    ("run_DE_INT", "flo_for_stereo", "not a .pfm file"),
    ("run_DE_INT", "pfm_scale", "scale is not negative"),
    ("run_DE_INT", "pfm_size", "size differs"),
    ("run_DE_INT", "pfm_short", "length does not match"),
    ("run_DE_INT", "pfm_magic", "not a one-channel .pfm"),
])
def test_cli_init_flow_file_errors(bindir, images, tmp_path, exe, case, message):
    """A bad init-flow file exits with 1 and names the problem; these checks run before the device is touched (the
    messages come from the file check, and the same calls fail this way on a machine without a GPU)."""
    f = str(tmp_path / "init")
    if case == "tag":
        _flo(f, 40, 30, tag=b"PIEX")
    elif case == "size":
        _flo(f, 41, 30, data=np.zeros((30, 41, 2), "<f4"))
    elif case == "short":
        with open(f, "wb") as fh:
            fh.write(b"PIEH" + np.array([40, 30], "<i4").tobytes() + np.zeros(40 * 30 * 2 - 1, "<f4").tobytes())
    elif case == "long":
        with open(f, "wb") as fh:
            fh.write(b"PIEH" + np.array([40, 30], "<i4").tobytes() + np.zeros(40 * 30 * 2 + 1, "<f4").tobytes())
    elif case == "flo_for_stereo":
        _flo(f, 40, 30)
    elif case.startswith("pfm"):
        w = 39 if case == "pfm_size" else 40
        scale = b"1.000000" if case == "pfm_scale" else b"-1.000000"
        magic = b"PF" if case == "pfm_magic" else b"Pf"
        n = w * 30 - (1 if case == "pfm_short" else 0)
        with open(f, "wb") as fh:
            fh.write(magic + b"\n%d 30\n" % w + scale + b"\n" + np.zeros(n, "<f4").tobytes())
    r = _run(bindir, exe, images, str(tmp_path / "o"), ["1", f])
    assert r.returncode == 1, r.stdout + r.stderr
    assert message in r.stderr, r.stderr
    assert not os.path.exists(str(tmp_path / "o"))
