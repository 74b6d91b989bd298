"""preprocess.disparity_filter (the restatement of ofdis_disparity_fullres) against a plain per-pixel loop written from
the header: range and left-right status, a BFS flood fill for the speckles, explicit row and column scans for the
fill, and per-pixel depth and xyz.  No device needed."""
from collections import deque

import numpy as np
import pytest

from of_dis_b200 import preprocess

f32 = np.float32
QNAN = np.uint32(0x7FC00000).view(np.float32)
CAM = dict(fx=700.0, fy=690.0, cx=40.5, cy=20.25, baseline=0.12, doffs=0.0)


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def smaller(a, b):
    return b if b < a else a


def loop_filter(F, B, swapped, lr_check, alpha, beta, speckle_size, speckle_diff, fill, camera):
    h, w = F.shape
    d = np.empty((h, w), f32)
    st = np.zeros((h, w), np.uint8)
    mask = preprocess.consistency_check(F, B, alpha, beta)[0] if lr_check else None
    for y in range(h):
        for x in range(w):
            d[y, x] = F[y, x] if swapped else -F[y, x]
            if not (d[y, x] >= 0 and d[y, x] <= f32(1e9)):
                st[y, x] = 3
            elif lr_check:
                st[y, x] = mask[y, x]
    if speckle_size > 0:
        seen = np.zeros((h, w), bool)
        for y in range(h):
            for x in range(w):
                if st[y, x] != 0 or seen[y, x]:
                    continue
                comp, q = [], deque([(y, x)])
                seen[y, x] = True
                while q:
                    cy, cx = q.popleft()
                    comp.append((cy, cx))
                    for ny, nx in ((cy, cx - 1), (cy, cx + 1), (cy - 1, cx), (cy + 1, cx)):
                        if 0 <= ny < h and 0 <= nx < w and not seen[ny, nx] and st[ny, nx] == 0 and \
                                abs(f32(d[cy, cx] - d[ny, nx])) <= f32(speckle_diff):
                            seen[ny, nx] = True
                            q.append((ny, nx))
                if len(comp) <= speckle_size:
                    for cy, cx in comp:
                        st[cy, cx] = 4
    v = [[d[y, x] if st[y, x] == 0 else None for x in range(w)] for y in range(h)]
    if fill:
        def fill_line(line):
            n = len(line)
            idx = [i for i in range(n) if line[i] is not None]
            if not idx:
                return line
            out = list(line)
            for i in range(n):
                if line[i] is not None:
                    continue
                lefts = [j for j in idx if j < i]
                rights = [j for j in idx if j > i]
                if lefts and rights:
                    out[i] = smaller(line[lefts[-1]], line[rights[0]])
                else:
                    out[i] = line[lefts[-1]] if lefts else line[rights[0]]
            return out

        v = [fill_line(row) for row in v]
        cols = [fill_line([v[y][x] for y in range(h)]) for x in range(w)]
        v = [[cols[x][y] for x in range(w)] for y in range(h)]
    disp = np.array([[QNAN if v[y][x] is None else v[y][x] for x in range(w)] for y in range(h)], f32)
    depth = xyz = None
    if camera is not None:
        c = {k: f32(camera[k]) for k in camera}
        fb = f32(c["fx"] * c["baseline"])
        depth = np.empty((h, w), f32)
        xyz = np.empty((h, w, 3), f32)
        with np.errstate(all="ignore"):
            for y in range(h):
                for x in range(w):
                    s = f32(disp[y, x] + c["doffs"])
                    Z = f32(fb / s) if s > 0 else QNAN
                    Z = QNAN if np.isnan(Z) else Z
                    X = f32(f32(f32(x) - c["cx"]) * Z) / c["fx"]
                    Y = f32(f32(f32(y) - c["cy"]) * Z) / c["fy"]
                    depth[y, x] = Z
                    xyz[y, x] = [QNAN if np.isnan(X) else X, QNAN if np.isnan(Y) else Y, Z]
    return disp, st, depth, xyz


def check(F, B=None, swapped=False, lr_check=0, alpha=0.0, beta=1.0, speckle_size=0, speckle_diff=1.0, fill=0,
          camera=None):
    F = np.asarray(F, f32)
    B = np.zeros_like(F) if B is None else np.asarray(B, f32)
    got = preprocess.disparity_filter(F, B, swapped, lr_check, alpha, beta, speckle_size, speckle_diff, fill, camera)
    exp = loop_filter(F, B, swapped, lr_check, alpha, beta, speckle_size, speckle_diff, fill, camera)
    assert (got[1] == exp[1]).all(), np.argwhere(got[1] != exp[1])[:5]
    for k in (0, 2, 3):
        if exp[k] is None:
            assert got[k] is None
        else:
            assert (bits(got[k]) == bits(exp[k])).all(), (k, np.argwhere(bits(got[k]) != bits(exp[k]))[:5])
    return got


def test_component_sizes_at_the_threshold():
    F = -np.full((6, 12), 20.0, f32)
    F[1, 1:4] = -5.0   # 3 pixels
    F[3, 1:5] = -50.0  # 4 pixels
    for size in (3, 4):
        disp, st, _, _ = check(F, speckle_size=size, speckle_diff=1.0)
        assert (st[1, 1:4] == 4).all()
        assert (st[3, 1:5] == (4 if size == 4 else 0)).all()


def test_diagonal_contact_does_not_join():
    F = -np.full((5, 5), 100.0, f32)
    F[1, 1] = F[2, 2] = F[3, 3] = -10.0
    _, st, _, _ = check(F, speckle_size=1, speckle_diff=0.5)
    assert st[1, 1] == st[2, 2] == st[3, 3] == 4


def test_speckle_diff_exact_and_one_ulp_above():
    diff = f32(0.75)
    above = np.nextafter(diff, f32(2))
    F = -np.full((3, 8), 40.0, f32)
    F[1, 2], F[1, 3] = -2.0, -(2.0 + diff)  # 2.75 - 2 is exactly 0.75
    F[1, 5], F[1, 6] = 0.0, -above          # d = -0 and one ulp above 0.75
    assert f32(f32(2.0) + diff) - f32(2.0) == diff and above - f32(0) > diff
    _, st, _, _ = check(F, speckle_size=1, speckle_diff=float(diff))
    assert st[1, 2] == st[1, 3] == 0
    assert st[1, 5] == st[1, 6] == 4


def test_special_values():
    F = -np.arange(40, dtype=f32).reshape(5, 8)
    F[0, 0], F[0, 1], F[0, 2] = np.nan, np.inf, -np.inf
    F[1, 0], F[1, 1], F[1, 2] = 0.0, 5.0, -2e9
    F[2, 3] = -np.float32(1e9)
    for sw in (False, True):
        disp, st, _, _ = check(F if not sw else -F, swapped=sw, fill=1, camera=CAM)
        assert st[0, 0] == st[0, 1] == st[0, 2] == 3  # NaN, -inf and +inf
        assert st[1, 0] == 0 and np.signbit(disp[1, 0])  # d = -0 either way, and it passes
        assert st[1, 1] == 3 and st[1, 2] == 3 and st[2, 3] == 0


def test_negative_zero_passes():
    F = np.zeros((2, 3), f32)  # d = -0 everywhere
    disp, st, depth, _ = check(F, camera=CAM)
    assert (st == 0).all() and np.signbit(disp).all()
    assert np.isnan(depth).all()  # D + doffs = +0 is not > 0


@pytest.mark.parametrize("swapped", [False, True])
def test_fill_rows_and_columns(swapped):
    F = np.full((9, 11), np.nan, f32)
    s = 1.0 if swapped else -1.0
    F[2, 0] = s * 7.0           # row with a single valid pixel at the left border
    F[4, 3], F[4, 8] = s * 9.0, s * 4.0  # interior gap, gaps at both borders
    F[5, 10] = s * 3.0           # single pixel at the right border
    # rows 0, 1 (top), 3 (interior), 6..8 (bottom) are empty
    disp, st, _, _ = check(F, swapped=swapped, fill=1)
    assert (st == 3).sum() == 9 * 11 - 4
    assert (disp[2] == 7.0).all() and (disp[0] == 7.0).all() and (disp[8] == 3.0).all()
    assert (disp[4, :4] == 9.0).all() and (disp[4, 4:8] == 4.0).all() and (disp[4, 8:] == 4.0).all()
    assert (disp[3] == np.minimum(disp[2], disp[4])).all()


def test_all_invalid_frame_stays_empty():
    F = np.full((4, 6), 3.0, f32)  # d = -3 everywhere
    disp, st, depth, xyz = check(F, fill=1, speckle_size=2, camera=CAM)
    assert (st == 3).all() and (bits(disp) == 0x7FC00000).all()
    assert (bits(depth) == 0x7FC00000).all() and (bits(xyz) == 0x7FC00000).all()


def test_doffs_makes_the_denominator_non_positive():
    F = -np.array([[1.0, 2.0, 3.0, 4.0]], f32)
    cam = dict(CAM, doffs=-2.5)
    disp, st, depth, xyz = check(F, camera=cam)
    assert np.isnan(depth[0, :2]).all() and (depth[0, 2:] > 0).all()
    cam = dict(CAM, doffs=-2.0)
    _, _, depth, _ = check(F, camera=cam)
    assert np.isnan(depth[0, 1]) and depth[0, 2] > 0


@pytest.mark.parametrize("seed", range(6))
def test_random_frames_against_the_loop(seed):
    rng = np.random.default_rng(seed)
    h, w = rng.integers(3, 23), rng.integers(3, 41)
    F = -np.round(rng.uniform(-3, 30, (h, w)) * 2).astype(f32) / 2
    F[rng.random((h, w)) < 0.1] = np.nan
    B = -F + rng.normal(0, 0.8, (h, w)).astype(f32)
    B = np.where(np.isnan(B), f32(0), B).astype(f32)
    for lr in (0, 1):
        for sp in (0, 1, 3):
            for fill in (0, 1):
                check(F, B, bool(seed % 2), lr, 0.0, 1.0, sp, 0.5, fill, CAM if fill else None)


def test_left_right_status_is_the_consistency_mask():
    rng = np.random.default_rng(7)
    h, w = 12, 30
    F = -rng.uniform(0, 6, (h, w)).astype(f32)
    B = (-F + rng.normal(0, 1.5, (h, w))).astype(f32)
    mask = preprocess.consistency_check(F, B, 0.0, 1.0)[0]
    _, st, _, _ = check(F, B, lr_check=1)
    assert (st == mask).all()
    assert set(np.unique(st).tolist()) >= {0, 1, 2}


def tie_map():
    """Gaps bounded by +0 on one side and -0 on the other, along a row and along a column: the fill takes the first
    (left, upper) of two equal values, so the sign of the filled zeros tells the operand order."""
    d = np.full((7, 6), -1.0, f32)  # status 3 everywhere else
    d[1, 0], d[1, 4] = 0.0, -0.0     # row 1: +0 | gap | -0
    d[3, 0], d[3, 4] = -0.0, 0.0     # row 3: -0 | gap | +0
    d[5, :] = 0.0                    # row 5: +0 with one -0; rows 0, 2, 4 and 6 are empty
    d[5, 2] = -0.0
    return d


def test_fill_tie_takes_the_first_of_two_equal_values():
    d = tie_map()
    disp, st, _, _ = check(-d, fill=1)
    assert not np.signbit(disp[1, 1:4]).any() and np.signbit(disp[3, 1:4]).all()
    assert np.signbit(disp[1, 5]) and not np.signbit(disp[3, 5])  # right of the last value: that value
    # column pass: row 2 lies between rows 1 and 3, row 4 between rows 3 and 5; the upper row wins every tie
    assert (bits(disp[2]) == bits(disp[1])).all() and (bits(disp[4]) == bits(disp[3])).all()


def test_layered_stereo_scene():
    from of_dis_b200 import synth

    left, right, gt, occ = synth.layered_stereo(60, 100, 1, seed=3)
    y, x = np.mgrid[:60, :100]
    xr = x - gt.astype(np.int64)
    vis = ~occ
    assert (left[vis] == right[y[vis], xr[vis]]).all()
    assert set(np.unique(gt).tolist()) == {8.0, 24.0} and 0 < occ.mean() < 0.5
    # the hidden background strip left of the block (width d_fg - d_bg) and the left border (d_bg columns)
    assert occ[:, :8].all() and occ[30, 30 - 16:30].all() and not occ[30, 30:70].any()


# ---- batch command: the disparity flags are refused where they do not apply (no device needed) ------------------
CAMERA = "721.5,721.5,100,60,0.54,0.25"


@pytest.mark.parametrize("exe,args", [
    ("run_OF_INT", ["--lr-check"]), ("run_OF_RGB", ["--fill"]), ("run_OF_INT", ["--speckle", "10", "1"]),
    ("run_OF_INT", ["--camera", CAMERA]),
    ("run_DE_INT", ["--warm-start", "--fill"]), ("run_DE_RGB", ["--warm-start", "--lr-check"]),
    ("run_DE_INT", ["--speckle", "0", "1"]), ("run_DE_INT", ["--speckle", "10", "-1"]),
    ("run_DE_INT", ["--speckle", "10", "nan"]), ("run_DE_INT", ["--speckle", "x", "1"]),
    ("run_DE_INT", ["--speckle", "10"]), ("run_DE_INT", ["--speckle", "5", "1", "--speckle", "5", "1"]),
    ("run_DE_INT", ["--camera", "1,1,0,0,1"]), ("run_DE_INT", ["--camera", "0,1,0,0,1,0"]),
    ("run_DE_INT", ["--camera", "1,1,0,0,-1,0"]), ("run_DE_INT", ["--camera", "1,inf,0,0,1,0"]),
    ("run_DE_INT", ["--camera", "1,1,0,0,1,0,"]), ("run_DE_INT", ["--camera", "1,1,nan,0,1,0"]),
    ("run_DE_INT", ["--camera"])])
def test_batch_command_refuses_disparity_flags(tmp_path, exe, args):
    import subprocess

    from of_dis_b200 import build

    bindir = build.build_host()
    lst = tmp_path / "list.txt"
    lst.write_text("")
    r = subprocess.run([str(bindir) + "/" + exe + "_batch", str(lst)] + args, capture_output=True, text=True,
                       cwd=str(tmp_path))
    assert r.returncode == 2, (args, r.stdout, r.stderr)


def test_batch_command_accepts_disparity_flags(tmp_path):
    import subprocess

    from of_dis_b200 import build

    bindir = build.build_host()
    lst = tmp_path / "list.txt"
    lst.write_text("")
    args = ["--lr-check", "--speckle", "50", "0.5", "--fill", "--camera", CAMERA, "--kitti"]
    r = subprocess.run([str(bindir) + "/run_DE_RGB_batch", str(lst)] + args, capture_output=True, text=True,
                       cwd=str(tmp_path))
    assert r.returncode == 0, (r.stdout, r.stderr)
