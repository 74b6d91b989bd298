"""preprocess.consistency_check: the float32 restatement of the device's forward-backward / left-right check
(ofdis_consistency_fullres), which tests/test_bidir_gpu.py uses as its checker."""
import numpy as np

from of_dis_b200 import preprocess

FLOW, STEREO = (0.01, 0.5), (0.0, 1.0)


def test_zero_flows_are_consistent():
    for nop in (1, 2):
        z = np.zeros((17, 23, nop), np.float32)
        mask, err = preprocess.consistency_check(z, z, *FLOW)
        assert mask.dtype == np.uint8 and mask.shape == (17, 23)
        assert not mask.any() and not err.any()


def test_translation_and_its_negative():
    """F = (3, -2), B = -F: consistent where (x + 3, y - 2) stays in the frame, 2 where it leaves."""
    h, w = 20, 30
    fw = np.broadcast_to(np.float32([3, -2]), (h, w, 2)).copy()
    mask, err = preprocess.consistency_check(fw, -fw, *FLOW)
    x, y = np.meshgrid(np.arange(w), np.arange(h))
    inside = (x + 3 <= w - 1) & (y - 2 >= 0)
    assert (mask[inside] == 0).all() and (err[inside] == 0).all()
    assert (mask[~inside] == 2).all() and np.isinf(err[~inside]).all()
    # the same B shifted by one pixel's worth of error: inconsistent inside (|F + b|^2 = 4 > 0.01 * 26 + 0.5)
    mask, _ = preprocess.consistency_check(fw, -fw + np.float32([2, 0]), *FLOW)
    assert (mask[inside] == 1).all() and (mask[~inside] == 2).all()


def test_nan_leaves_the_frame():
    fw = np.zeros((8, 9, 2), np.float32)
    fw[3, 4, 0] = np.nan
    fw[5, 1, 1] = np.nan
    mask, err = preprocess.consistency_check(fw, np.zeros_like(fw), *FLOW)
    assert mask[3, 4] == 2 and mask[5, 1] == 2 and np.isinf(err[3, 4])
    assert (np.delete(mask.reshape(-1), [3 * 9 + 4, 5 * 9 + 1]) == 0).all()


def test_stereo_left_right():
    """d_L = -4, d_R = +4: consistent where x - 4 >= 0; a right disparity off by 2 px fails |d_L + d_R| <= 1."""
    h, w = 6, 25
    dl = np.full((h, w, 1), -4, np.float32)
    mask, err = preprocess.consistency_check(dl, -dl, *STEREO)
    assert (mask[:, 4:] == 0).all() and (mask[:, :4] == 2).all() and (err[:, 4:] == 0).all()
    mask, err = preprocess.consistency_check(dl, -dl + np.float32(2), *STEREO)
    assert (mask[:, 4:] == 1).all() and (err[:, 4:] == 4).all()
    # (h, w) input means the same as (h, w, 1)
    m2, e2 = preprocess.consistency_check(dl[..., 0], -dl[..., 0], *STEREO)
    assert (m2 == preprocess.consistency_check(dl, -dl, *STEREO)[0]).all()


def _direct_f64(fw, bw, alpha, beta):
    """The same definition in float64 with plain bilinear sampling."""
    h, w = fw.shape[:2]
    nop = fw.shape[2]
    F, B = fw.astype(np.float64), bw.astype(np.float64)
    mask = np.zeros((h, w), np.uint8)
    err = np.zeros((h, w))
    margin = np.zeros((h, w))
    for y in range(h):
        for x in range(w):
            u = F[y, x, 0]
            v = F[y, x, 1] if nop == 2 else 0.0
            xs, ys = x + u, y + v
            if not (0 <= xs <= w - 1 and 0 <= ys <= h - 1):
                mask[y, x], err[y, x] = 2, np.inf
                continue
            x0, y0 = int(np.floor(xs)), int(np.floor(ys))
            x1, y1 = min(x0 + 1, w - 1), min(y0 + 1, h - 1)
            fx, fy = xs - x0, ys - y0
            b = (B[y0, x0] * (1 - fx) + B[y0, x1] * fx) * (1 - fy) + (B[y1, x0] * (1 - fx) + B[y1, x1] * fx) * fy
            fv = np.array([u, v][:nop])
            d = fv + b
            err[y, x] = float(d @ d)
            thr = alpha * (float(fv @ fv) + float(b @ b)) + beta
            margin[y, x] = abs(err[y, x] - thr) / max(1.0, thr)
            mask[y, x] = 0 if err[y, x] <= thr else 1
    return mask, err, margin


def test_against_a_float64_direct_formula():
    rng = np.random.default_rng(5)
    h, w = 24, 31
    for nop, (alpha, beta) in ((2, FLOW), (1, STEREO), (2, (0.05, 0.0))):
        base = rng.normal(0, 3, (h, w, nop)).astype(np.float32)
        fw = base + rng.normal(0, 0.3, base.shape).astype(np.float32)
        bw = (-base + rng.normal(0, 0.6, base.shape)).astype(np.float32)
        mask, err = preprocess.consistency_check(fw, bw, alpha, beta)
        m64, e64, margin = _direct_f64(fw, bw, alpha, beta)
        assert ((mask == 2) == (m64 == 2)).all()
        near = margin < 1e-4  # rounding may flip a pixel right at the threshold
        assert (mask[~near] == m64[~near]).all(), nop
        inside = m64 != 2
        assert np.allclose(err[inside], e64[inside], rtol=1e-5, atol=1e-5)
        assert {0, 1} <= set(np.unique(mask[inside]).tolist()), "the case should exercise both outcomes"


def test_write_pgm(tmp_path):
    img = (np.arange(6 * 7) % 3 * 127).astype(np.uint8).reshape(6, 7)
    p = tmp_path / "m.pgm"
    preprocess.write_pgm(str(p), img)
    data = p.read_bytes()
    assert data.startswith(b"P5\n7 6\n255\n")
    assert np.frombuffer(data[len(b"P5\n7 6\n255\n"):], np.uint8).reshape(6, 7).tolist() == img.tolist()


def test_batch_command_argument_errors(tmp_path):
    """--bidirectional with --warm-start is refused before any file or device work, in either order; the usage
    text names the option; a wrong number count is refused as without it."""
    import os
    import subprocess

    from of_dis_b200 import build

    bindir = build.build_host()
    lst = str(tmp_path / "missing.txt")
    for exe in ("run_OF_INT_batch", "run_DE_RGB_batch"):
        path = os.path.join(bindir, exe)
        for args in (["--bidirectional", "--warm-start"], ["--warm-start", "--bidirectional"]):
            r = subprocess.run([path, lst] + args, capture_output=True, text=True)
            assert r.returncode == 2 and "--bidirectional" in r.stderr, (exe, args, r.stderr)
        r = subprocess.run([path, lst, "--bidirectional", "1", "2"], capture_output=True, text=True)
        assert r.returncode == 2, r.stderr
        r = subprocess.run([path], capture_output=True, text=True)
        assert r.returncode == 2 and "--bidirectional" in r.stderr and "_occ.pgm" in r.stderr
        r = subprocess.run([path, lst, "--bidirectional"], capture_output=True, text=True)
        assert r.returncode == 1 and "cannot read" in r.stderr  # the options parse; the list does not exist
