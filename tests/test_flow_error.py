"""preprocess.flow_error: the numpy restatement of the device evaluation against ground truth
(ofdis_flow_error_fullres), which tests/test_flow_error_gpu.py uses as its checker; the stats dtype against the C
struct; and the batch command's --gt argument errors, which are refused before any device work."""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest

from of_dis_b200 import api, preprocess

f32 = np.float32


def _direct_f64(flow, gt):
    """End-point error in float64, straight from the definition."""
    d = flow.astype(np.float64) - gt.astype(np.float64)
    return np.sqrt((d * d).sum(-1))


def _row_order_sum(err, counted):
    """The contract's order with Python floats: per row x ascending, then the rows y ascending."""
    total = 0.0
    for y in range(err.shape[0]):
        row = 0.0
        for x in range(err.shape[1]):
            if counted[y, x]:
                row += float(err[y, x])
        total += row
    return total


def _case(seed, h=23, w=37, nop=2):
    rng = np.random.default_rng(seed)
    gt = rng.normal(0, 6, (h, w, nop)).astype(f32)
    flow = (gt + rng.normal(0, 2.5, gt.shape)).astype(f32)
    return flow, gt


def test_against_a_float64_direct_formula():
    flow, gt = _case(1)
    stats, err = preprocess.flow_error(flow, gt)
    assert stats.dtype == api.ERROR_STATS_DTYPE and stats.shape == (1,) and err.shape == gt.shape[:2]
    e64 = _direct_f64(flow, gt)
    assert np.allclose(err, e64, rtol=1e-6, atol=0)
    s = stats[0]
    assert s["n"] == gt.shape[0] * gt.shape[1]
    assert list(s["n_over"]) == [int((e64 > t).sum()) for t in (1, 3, 5)]
    g64 = np.sqrt((gt.astype(np.float64) ** 2).sum(-1))
    assert s["n_outlier"] == int(((e64 > 3) & (e64 > 0.05 * g64)).sum())
    assert 0 < s["n_outlier"] < s["n"] and 0 < s["n_over"][2] < s["n_over"][0] < s["n"]


def test_sum_is_the_row_order_sum_and_close_to_fsum():
    flow, gt = _case(2)
    classes = (np.arange(gt.shape[0] * gt.shape[1]) % 3).astype(np.uint8).reshape(gt.shape[:2])
    stats, err = preprocess.flow_error(flow, gt, classes, 3)
    for c in range(3):
        counted = classes == c
        assert stats[c]["sum_err"] == _row_order_sum(err, counted)  # bit for bit
        ref = math.fsum(float(v) for v in err[counted])
        assert abs(stats[c]["sum_err"] - ref) <= 1e-12 * ref
        assert stats[c]["n"] == int(counted.sum())


def test_unknown_ground_truth():
    """NaN and +-inf are unknown, exactly 1e9 is known, the next float32 above 1e9 is unknown; the map holds the
    quiet NaN 0x7fc00000 there."""
    h, w = 4, 6
    gt = np.zeros((h, w, 2), f32)
    flow = np.ones((h, w, 2), f32)
    above = np.nextafter(f32(1e9), f32(np.inf))
    gt[0, 0, 0] = np.nan
    gt[0, 1, 1] = np.nan
    gt[0, 2, 0] = np.inf
    gt[0, 3, 1] = -np.inf
    gt[1, 0, 0] = above
    gt[1, 1, 1] = -above
    gt[2, 0, 0] = f32(1e9)
    gt[2, 1, 1] = f32(-1e9)
    (s,), err = preprocess.flow_error(flow, gt)
    unknown = np.zeros((h, w), bool)
    unknown[0, :4] = unknown[1, :2] = True
    assert s["n"] == h * w - unknown.sum()
    assert (err[unknown].view(np.uint32) == 0x7FC00000).all()
    assert not np.isnan(err[~unknown]).any()
    # F = (1, 1): e = sqrt(2) where G = 0; the two |G| = 1e9 pixels have e ~ g = 1e9, above 5 and outliers
    assert list(s["n_over"]) == [s["n"], 2, 2] and s["n_outlier"] == 2
    # stereo: the same rules on the one component
    gs = gt[..., :1].copy()
    (st,), es = preprocess.flow_error(flow[..., :1], gs)
    unk = np.isnan(gs[..., 0]) | ~(np.abs(gs[..., 0]) <= 1e9)
    assert unk.sum() == 3 and st["n"] == h * w - unk.sum() and (es[unk].view(np.uint32) == 0x7FC00000).all()


def test_classes_at_or_above_nclasses_are_excluded():
    flow, gt = _case(3, 10, 12)
    classes = np.zeros(gt.shape[:2], np.uint8)
    classes[0] = 1
    classes[1] = 2
    classes[2] = 255
    stats, err = preprocess.flow_error(flow, gt, classes, 2)
    assert stats.shape == (2,)
    assert stats[0]["n"] == 7 * 12 and stats[1]["n"] == 12
    all1, _ = preprocess.flow_error(flow, gt)
    assert all1["n"] == 120
    assert (err.view(np.uint32) == preprocess.flow_error(flow, gt)[1].view(np.uint32)).all()  # classes leave the map
    # 16 classes: every byte below 16 counts for its own class
    classes = (np.arange(120) % 20).astype(np.uint8).reshape(10, 12)
    s16, _ = preprocess.flow_error(flow, gt, classes, 16)
    assert [int(s["n"]) for s in s16] == [int((classes == c).sum()) for c in range(16)]


def test_threshold_edges():
    """e exactly 1, 3 or 5 is not above it; an outlier needs e > 3 and e > 0.05 g."""
    flow = np.zeros((1, 6, 2), f32)
    gt = np.array([[[1, 0], [3, 0], [5, 0], [0, 3.5], [0, 100], [60, 80]]], f32)  # e = |G| since F = 0
    (s,), err = preprocess.flow_error(flow, gt)
    assert err.tolist() == [[1, 3, 5, 3.5, 100, 100]]
    assert list(s["n_over"]) == [5, 4, 2]
    assert s["n_outlier"] == 4  # 5 > 0.25, 3.5 > 0.175, 100 > 5 twice; 3 and below fail e > 3
    # e > 0.05 g is strict too: g = 80 gives 0.05f * 80 = 4 in float32, so e = 4 is above 3 but no outlier
    gt = np.array([[[0, 80]]], f32)
    assert f32(0.05) * f32(80) == f32(4)
    (st,), e = preprocess.flow_error(np.array([[[0, 76]]], f32), gt)
    assert e[0, 0] == 4 and st["n_over"][1] == 1 and st["n_outlier"] == 0


def test_stereo():
    rng = np.random.default_rng(4)
    gt = -np.abs(rng.normal(0, 20, (9, 31))).astype(f32)
    d = (gt + rng.normal(0, 3, gt.shape)).astype(f32)
    stats, err = preprocess.flow_error(d, gt)
    (s,) = stats
    assert (err == np.abs(d - gt)).all()
    assert s["n"] == gt.size and s["sum_err"] == _row_order_sum(err, np.ones(gt.shape, bool))
    assert s["n_outlier"] == int(((err > 3) & (err > f32(0.05) * np.abs(gt))).sum())
    s3, e3 = preprocess.flow_error(d[..., None], gt[..., None])  # (h, w, 1) == (h, w)
    assert s3.tobytes() == stats.tobytes() and (e3 == err).all()


def test_batch_equals_the_pairs():
    pairs = [_case(10 + k, 11, 13) for k in range(3)]
    flow = np.stack([p[0] for p in pairs])
    gt = np.stack([p[1] for p in pairs])
    classes = (np.arange(3 * 11 * 13) % 2).astype(np.uint8).reshape(3, 11, 13)
    stats, err = preprocess.flow_error(flow, gt, classes, 2)
    assert stats.shape == (3, 2) and err.shape == (3, 11, 13)
    for k in range(3):
        s, e = preprocess.flow_error(flow[k], gt[k], classes[k], 2)
        assert s.tobytes() == stats[k].tobytes() and (e == err[k]).all()


def test_nan_flow_is_counted():
    flow, gt = _case(5, 5, 7)
    flow[2, 3, 0] = np.nan
    (s,), err = preprocess.flow_error(flow, gt)
    assert s["n"] == 35 and math.isnan(s["sum_err"]) and np.isnan(err[2, 3])
    assert s["n_over"][0] == int((np.nan_to_num(err, nan=0) > 1).sum())


def test_stats_dtype_is_the_c_struct():
    class Stats(ctypes.Structure):
        _fields_ = [("n", ctypes.c_longlong), ("n_over", ctypes.c_longlong * 3), ("n_outlier", ctypes.c_longlong),
                    ("sum_err", ctypes.c_double)]

    dt = api.ERROR_STATS_DTYPE
    assert dt.itemsize == ctypes.sizeof(Stats) == 48
    for name, _ in Stats._fields_:
        assert dt.fields[name][1] == getattr(Stats, name).offset, name
    assert dt.fields["n_over"][0].shape == (3,)
    assert "ofdis_flow_error_fullres" in api.EXPORTS


# ---- batch front-end: --gt argument and file errors (all refused before the device is touched) --------------------
@pytest.fixture(scope="module")
def bindir():
    from of_dis_b200 import build

    return build.build_host()


def _pgm(path, w, h):
    with open(path, "wb") as f:
        f.write(b"P5\n%d %d\n255\n" % (w, h) + bytes(range(w)) * h)


def _flo(path, w, h, tag=b"PIEH"):
    with open(path, "wb") as f:
        f.write(tag + np.array([w, h], "<i4").tobytes() + np.zeros((h, w, 2), "<f4").tobytes())


def _pfm(path, w, h):
    with open(path, "wb") as f:
        f.write(b"Pf\n%d %d\n-1.000000\n" % (w, h) + np.zeros(w * h, "<f4").tobytes())


@pytest.mark.parametrize("exe", ["run_OF_INT_batch", "run_DE_RGB_batch"])
def test_batch_command_gt_errors(bindir, tmp_path, exe):
    path = os.path.join(bindir, exe)
    stereo = "_DE_" in exe
    for k in range(3):
        _pgm(str(tmp_path / ("i%d.pgm" % k)), 40, 30)
    lst = tmp_path / "list.txt"
    lst.write_text("".join("%s %s %s\n" % (tmp_path / ("i%d.pgm" % k), tmp_path / ("i%d.pgm" % (k + 1)),
                                           tmp_path / ("o%d" % k)) for k in range(2)))
    good = [str(tmp_path / ("g%d" % k)) for k in range(2)]
    for g in good:
        (_pfm if stereo else _flo)(g, 40, 30)

    def run(*args):
        return subprocess.run([path, str(lst)] + list(args), capture_output=True, text=True)

    def gtlist(name, paths):
        p = tmp_path / name
        p.write_text(" ".join(paths) + "\n")
        return str(p)

    # argument errors: exit 2
    r = run("--gt")
    assert r.returncode == 2 and "--gt" in r.stderr, r.stderr
    r = run("--gt", gtlist("a.txt", good), "--gt", gtlist("b.txt", good))
    assert r.returncode == 2 and "--gt" in r.stderr, r.stderr
    r = run("--gt", gtlist("short.txt", good[:1]))
    assert r.returncode == 2 and "1 ground-truth files for 2 pairs" in r.stderr, r.stderr
    r = run("--gt", gtlist("long.txt", good + good[:1]))
    assert r.returncode == 2, r.stderr
    # file errors: exit 1, the message names the file and the problem
    r = run("--gt", str(tmp_path / "missing.txt"))
    assert r.returncode == 1 and "cannot read" in r.stderr, r.stderr
    r = run("--gt", gtlist("m.txt", [good[0], str(tmp_path / "nope")]))
    assert r.returncode == 1 and "cannot read the ground-truth file" in r.stderr, r.stderr
    wrong = str(tmp_path / "wrong")
    (_pfm if stereo else _flo)(wrong, 41, 30)
    r = run("--gt", gtlist("w.txt", [good[0], wrong]))
    assert r.returncode == 1 and "wrong" in r.stderr and "size differs" in r.stderr, r.stderr
    other = str(tmp_path / "other")
    (_flo if stereo else _pfm)(other, 40, 30)
    r = run("--gt", gtlist("o.txt", [other, good[1]]))
    assert r.returncode == 1 and ("not a .pfm file" if stereo else "not a .flo file") in r.stderr, r.stderr
    # every check ran before the device: no output file was written
    assert not any(os.path.exists(str(tmp_path / ("o%d" % k))) for k in range(2))
    r = subprocess.run([path], capture_output=True, text=True)
    assert r.returncode == 2 and "--gt gtlist" in r.stderr
