"""preprocess.scene_flow (the restatement of ofdis_scene_flow_fullres) against a per-pixel loop written from the
header, on random frames seeded with every edge case the header names, and on synth.layered_scene_flow's exact
scene."""
import math

import numpy as np
import pytest

from of_dis_b200 import preprocess, synth

f32 = np.float32
QNAN = np.uint32(0x7FC00000).view(np.float32)
CAM = dict(fx=721.5, fy=707.0, cx=5.25, cy=4.5, baseline=0.54, doffs=0.25)


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def known(d):
    return bool(d >= 0) and bool(d <= f32(1e9))


def outlier(e, g):
    return bool(e > f32(3)) and bool(e > f32(0.05) * g)


def loop(F, D0, D1, edge_diff, cam, gt, cls, nclasses):
    """One pair, pixel by pixel, every operation a float32 scalar one, as the header states it."""
    h, w = D0.shape
    d1w = np.empty((h, w), f32)
    status = np.empty((h, w), np.uint8)
    motion = np.empty((h, w, 3), f32)
    stats = np.zeros(nclasses, preprocess.SF_STATS_DTYPE)
    inf = f32(np.inf)
    with np.errstate(all="ignore"):
        for y in range(h):
            for x in range(w):
                u, v = F[y, x, 0], F[y, x, 1]
                d0 = D0[y, x]
                xs, ys = f32(x) + u, f32(y) + v
                inside = bool(xs >= 0) and bool(xs <= f32(w - 1)) and bool(ys >= 0) and bool(ys <= f32(h - 1))
                d1 = QNAN
                if inside:
                    x0, y0 = int(math.floor(xs)), int(math.floor(ys))
                    x1, y1 = min(x0 + 1, w - 1), min(y0 + 1, h - 1)
                    fx, fy = f32(xs - f32(x0)), f32(ys - f32(y0))
                    c = [D1[y0, x0], D1[y0, x1], D1[y1, x0], D1[y1, x1]]
                    if all(known(a) for a in c) and f32(max(c) - min(c)) <= f32(edge_diff):
                        r0 = c[0] * (f32(1) - fx) + c[1] * fx
                        r1 = c[2] * (f32(1) - fx) + c[3] * fx
                        d1 = f32(r0 * (f32(1) - fy) + r1 * fy)
                    else:
                        d1 = D1[y1 if fy >= f32(0.5) else y0, x1 if fx >= f32(0.5) else x0]
                k0 = known(d0)
                k1 = inside and known(d1)
                st = (0 if k0 else 1) | (0 if inside else 2) | (4 if inside and not k1 else 0)
                status[y, x] = st
                d1w[y, x] = d1 if k1 else QNAN
                m = [QNAN] * 3
                if cam is not None:
                    c = {k: f32(cam[k]) for k in preprocess.STEREO_CAMERA_FIELDS}
                    fb = f32(c["fx"] * c["baseline"])
                    s0, s1 = f32(d0 + c["doffs"]), f32(d1 + c["doffs"])
                    if st == 0 and s0 > 0 and s1 > 0:
                        Z0, Z1 = f32(fb / s0), f32(fb / s1)
                        X0 = f32(f32((f32(x) - c["cx"]) * Z0) / c["fx"])
                        Y0 = f32(f32((f32(y) - c["cy"]) * Z0) / c["fy"])
                        X1 = f32(f32((xs - c["cx"]) * Z1) / c["fx"])
                        Y1 = f32(f32((ys - c["cy"]) * Z1) / c["fy"])
                        m = [f32(X1 - X0), f32(Y1 - Y0), f32(Z1 - Z0)]
                        m = [QNAN if np.isnan(a) else a for a in m]
                    motion[y, x] = m
                if gt is not None:
                    G0, G1, Gu, Gv = gt[0][y, x], gt[1][y, x], gt[2][y, x, 0], gt[2][y, x, 1]
                    kg0, kg1 = known(G0), known(G1)
                    kgf = bool(abs(Gu) <= f32(1e9)) and bool(abs(Gv) <= f32(1e9))
                    e0 = abs(f32(d0 - G0)) if k0 else inf
                    e1 = abs(f32(d1w[y, x] - G1)) if k1 else inf
                    du, dv = f32(u - Gu), f32(v - Gv)
                    kf = bool(abs(u) <= f32(1e9)) and bool(abs(v) <= f32(1e9))
                    ef = f32(np.sqrt(f32(du * du + dv * dv))) if kf else inf
                    gf = f32(np.sqrt(f32(Gu * Gu + Gv * Gv)))
                    o = (outlier(e0, abs(G0)), outlier(e1, abs(G1)), outlier(ef, gf))
                    k = cls[y, x] if cls is not None else 0
                    if k < nclasses:
                        s = stats[k]
                        ksf = kg0 and kg1 and kgf
                        for name, cnt in (("n_d1", kg0), ("n_d2", kg1), ("n_fl", kgf), ("n_sf", ksf),
                                          ("out_d1", kg0 and o[0]), ("out_d2", kg1 and o[1]),
                                          ("out_fl", kgf and o[2]), ("out_sf", ksf and any(o))):
                            s[name] += int(cnt)
    return d1w, status, motion if cam is not None else None, stats if gt is not None else None


def edge_case_pair(rng, h, w, edge_diff):
    """Random flows and disparities with the header's edge cases planted at known pixels."""
    F = rng.uniform(-3, 3, (h, w, 2)).astype(f32)
    D0 = rng.uniform(0, 40, (h, w)).astype(f32)
    D1 = rng.uniform(0, 40, (h, w)).astype(f32)
    for D in (D0, D1):
        idx = rng.choice(h * w, 12, replace=False)
        D.flat[idx[:4]] = np.nan
        D.flat[idx[4:7]] = -0.0
        D.flat[idx[7:9]] = -1.5
        D.flat[idx[9:10]] = np.inf
        D.flat[idx[10:12]] = f32(1e9)
    # targets exactly on and one ulp past the frame's edges
    F[0, 0] = (f32(w - 1), f32(0))
    F[0, 1] = (np.nextafter(f32(w - 1), f32(np.inf)) - f32(1), 0)
    F[1, 0] = (0, f32(h - 2))
    F[1, 1] = (0, np.nextafter(f32(h - 1), f32(np.inf)) - f32(1))
    F[2, 2] = (np.nextafter(f32(-2), f32(-np.inf)), 0)
    F[2, 3] = (f32(-3), f32(-2))
    # NaN flows
    F[3, 3] = (np.nan, 0)
    F[3, 4] = (0, np.nan)
    # fx, fy exactly 0.5 and one ulp below it (exact only where x or y is 0)
    F[4, 4] = (f32(1.5), f32(0.5))
    F[5, 0] = (np.nextafter(f32(0.5), f32(0)), f32(0.5))
    F[0, 6] = (f32(0.5), np.nextafter(f32(0.5), f32(0)))
    # corner spreads at and one ulp above edge_diff around the target (2.25, 6.75) of pixel (1, 6)
    F[6, 1] = (f32(1.25), f32(0.75))
    D1[6:8, 2:4] = [[10, 10], [10, f32(10) + f32(edge_diff)]]
    # both disparities unknown at a target inside the frame (status 5)
    F[8, 8] = (0, 0)
    D0[8, 8] = D1[8, 8] = np.nan
    return F, D0, D1


def gt_for(rng, F, D0, d1w, h, w):
    """Ground truth near the estimates, with outliers at and beside 3 px and 5 % and unknown entries."""
    G0 = (D0 + rng.choice([0, 1, 3, 5, 8], D0.shape).astype(f32)).astype(f32)
    G1 = (np.nan_to_num(d1w, nan=20.0) - rng.choice([0, 2, 3, 4], D0.shape).astype(f32)).astype(f32)
    GF = (np.nan_to_num(F) + rng.choice([0, 1, 3, 4], F.shape).astype(f32)).astype(f32)
    # exactly 3 px, one ulp beside it, and 5 % of a large disparity, one ulp beside that
    G0[0, 2], D0[0, 2] = f32(13), f32(10)
    G0[0, 3], D0[0, 3] = np.nextafter(f32(13), f32(20)), f32(10)
    G0[0, 4], D0[0, 4] = f32(100), f32(105)
    G0[0, 5], D0[0, 5] = f32(100), np.nextafter(f32(105), f32(200))
    GF[1, 2], F[1, 2] = (f32(100), f32(0)), (f32(105), f32(0))
    GF[1, 3], F[1, 3] = (f32(100), f32(0)), (np.nextafter(f32(105), f32(200)), f32(0))
    for G in (G0, G1):
        idx = rng.choice(h * w, 6, replace=False)
        G.flat[idx[:3]] = np.nan
        G.flat[idx[3:]] = -2.0
    GF[2, 0] = (np.nan, 0)
    GF[2, 1] = (0, 2e9)
    return G0, G1, GF


@pytest.mark.parametrize("edge_diff", [1.0, 0.0, np.inf])
@pytest.mark.parametrize("doffs", [0.25, -12.0])
def test_restatement_equals_the_per_pixel_loop(edge_diff, doffs):
    rng = np.random.default_rng(5 + int(doffs < 0))
    h, w, n, ncls = 9, 12, 3, 3
    cam = dict(CAM, doffs=doffs)
    Fs, D0s, D1s = zip(*[edge_case_pair(rng, h, w, 1.0 if np.isinf(edge_diff) else edge_diff) for _ in range(n)])
    F, D0, D1 = np.stack(Fs), np.stack(D0s), np.stack(D1s)
    d1w, _, _, _ = preprocess.scene_flow(F, D0, D1, edge_diff)
    gts = [gt_for(rng, F[k], D0[k], d1w[k], h, w) for k in range(n)]
    gt = tuple(np.stack(a) for a in zip(*gts))
    cls = rng.integers(0, ncls + 1, (n, h, w)).astype(np.uint8)  # ncls itself is ignored
    got = preprocess.scene_flow(F, D0, D1, edge_diff, cam, gt, cls, ncls)
    seen = set()
    for k in range(n):
        exp = loop(F[k], D0[k], D1[k], edge_diff, cam, tuple(a[k] for a in gt), cls[k], ncls)
        assert (bits(got[0][k]) == bits(exp[0])).all()
        assert (got[1][k] == exp[1]).all()
        assert (bits(got[2][k]) == bits(exp[2])).all()
        assert (got[3][k] == exp[3]).all(), (got[3][k], exp[3])
        seen |= set(np.unique(exp[1]).tolist())
        single = preprocess.scene_flow(F[k], D0[k], D1[k], edge_diff, cam, tuple(a[k] for a in gt), cls[k], ncls)
        assert (bits(single[2]) == bits(exp[2])).all() and (single[3] == exp[3]).all()
    assert {0, 1, 2, 3, 4, 5} <= seen, seen  # every status bit, alone and together
    if doffs < 0:  # a denominator <= 0 leaves a status-0 pixel without motion
        st0 = got[1] == 0
        assert np.isnan(got[2][st0]).any() and not np.isnan(got[2][st0]).all()
    assert got[3]["out_d1"].sum() > 0 and got[3]["out_fl"].sum() < got[3]["n_fl"].sum()


def test_planted_cases():
    """The planted pixels give what the header says."""
    rng = np.random.default_rng(1)
    h, w = 9, 12
    F, D0, D1 = edge_case_pair(rng, h, w, 1.0)
    D0[:] = 5
    d1w, st, _, _ = preprocess.scene_flow(F, D0, D1, 1.0)
    assert st[0, 0] & 2 == 0 and st[0, 1] & 2 == 2  # on the edge, one ulp past it
    assert st[1, 0] & 2 == 0 and st[1, 1] & 2 == 2
    assert st[2, 2] & 2 == 2 and st[2, 3] & 2 == 0
    assert st[3, 3] & 2 == 2 and st[3, 4] & 2 == 2  # NaN flows fail
    # spread == edge_diff blends: (2.25, 6.75) -> 10 except the corner (3, 7) at 11 with weight 0.25 * 0.75
    r1 = f32(10) * f32(0.75) + f32(11) * f32(0.25)
    assert d1w[6, 1] == f32(f32(10) * f32(0.25) + r1 * f32(0.75))
    # one ulp above edge_diff takes the nearest corner
    D1b = D1.copy()
    D1b[7, 3] = np.nextafter(f32(11), f32(20))
    d1b, _, _, _ = preprocess.scene_flow(F, D0, D1b, 1.0)
    assert d1b[6, 1] == D1b[7, 2]  # fx 0.25 -> x0 = 2, fy 0.75 -> y1 = 7
    inf, _, _, _ = preprocess.scene_flow(F, D0, D1b, np.inf)
    assert inf[6, 1] != d1b[6, 1]
    # fx exactly 0.5 rounds up to x1, one ulp below to x0
    D1c = np.arange(h * w, dtype=f32).reshape(h, w) * 50
    d1c, _, _, _ = preprocess.scene_flow(F, D0, D1c, 1.0)
    assert d1c[4, 4] == D1c[5, 6]
    assert d1c[5, 0] == D1c[6, 0] and d1c[0, 6] == D1c[0, 7]


def test_exact_scene_has_no_outliers_and_its_motion():
    h, w = 48, 80
    frames, gt = synth.layered_scene_flow(h, w, 1, seed=3, d_bg=6, d_fg=(18, 22), dx=5)
    assert frames.shape == (4, h, w)
    occ = gt["occluded"]
    assert 0 < occ.sum() < occ.size / 2
    cls = occ.astype(np.uint8)
    truth = (gt["disp0"], gt["disp1"], gt["flow"])
    d1w, st, motion, stats = preprocess.scene_flow(gt["flow"], gt["disp0"], gt["disp_t1"], 1.0, CAM, truth, cls, 2)
    assert stats[0]["n_sf"] == (~occ).sum()
    for name in ("out_d1", "out_d2", "out_fl", "out_sf"):
        assert stats[0][name] == 0, (name, stats)
    assert stats[1]["out_d2"] > 0  # background points hidden by the moved rectangle
    assert (d1w[~occ] == gt["disp1"][~occ]).all() and (st[~occ] == 0).all()
    # the scene's motion, in float64
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    c = {k: float(v) for k, v in CAM.items()}

    def point(px, py, d):
        Z = c["fx"] * c["baseline"] / (d + c["doffs"])
        return np.stack([(px - c["cx"]) * Z / c["fx"], (py - c["cy"]) * Z / c["fy"], Z], -1)

    scene = point(x + gt["flow"][..., 0], y + gt["flow"][..., 1], gt["disp1"]) - point(x, y, gt["disp0"])
    np.testing.assert_allclose(motion[~occ], scene[~occ], rtol=1e-5, atol=1e-5)
    moving = ~occ & (gt["flow"][..., 0] != 0)
    assert moving.any() and (np.abs(motion[moving][:, 2]) > 0.1).all()


def test_scene_views_are_consistent():
    """Every point visible in all four views has the same bytes in each."""
    h, w, dx = 40, 72, 4
    frames, gt = synth.layered_scene_flow(h, w, 3, seed=9, d_bg=5, d_fg=(15, 12), dx=dx)
    l0, r0, l1, r1 = frames.astype(np.int64)
    y, x = np.mgrid[0:h, 0:w]
    ok = ~gt["occluded"]
    xt = x + gt["flow"][..., 0].astype(np.int64)
    assert (l0[ok] == r0[y[ok], (x - gt["disp0"].astype(np.int64))[ok]]).all()
    assert (l0[ok] == l1[y[ok], xt[ok]]).all()
    assert (l0[ok] == r1[y[ok], (xt - gt["disp1"].astype(np.int64))[ok]]).all()


# ---- batch command: --scene-flow and --gt-scene-flow are refused where they do not apply (no device needed) ----------
CAMERA = "721.5,707,5.25,4.5,0.54,0.25"


def _batch(tmp_path, exe, args, pairs=0):
    import subprocess

    from of_dis_b200 import build

    bindir = build.build_host()
    img = np.zeros((24, 32), np.uint8)
    lines = []
    for k in range(pairs):
        preprocess.write_pgm(str(tmp_path / ("a%d.pgm" % k)), img)
        preprocess.write_pgm(str(tmp_path / ("b%d.pgm" % k)), img)
        lines.append("a%d.pgm b%d.pgm out%d.flo" % (k, k, k))
    (tmp_path / "list.txt").write_text("\n".join(lines) + "\n")
    return subprocess.run([str(bindir) + "/" + exe + "_batch", "list.txt"] + args, capture_output=True, text=True,
                          cwd=str(tmp_path))


@pytest.mark.parametrize("exe,args", [
    ("run_DE_INT", ["--scene-flow", "d.txt"]), ("run_DE_RGB", ["--scene-flow", "d.txt", "--camera", CAMERA]),
    ("run_OF_INT", ["--warm-start", "--scene-flow", "d.txt"]), ("run_OF_RGB", ["--gt-scene-flow", "g.txt"]),
    ("run_OF_INT", ["--scene-flow", "d.txt", "--lr-check"]), ("run_OF_INT", ["--scene-flow", "d.txt", "--fill"]),
    ("run_OF_INT", ["--scene-flow", "d.txt", "--camera", "1,1,0,0,-1,0"]), ("run_OF_INT", ["--scene-flow"])])
def test_batch_command_refuses_scene_flow_flags(tmp_path, exe, args):
    (tmp_path / "d.txt").write_text("")
    (tmp_path / "g.txt").write_text("")
    r = _batch(tmp_path, exe, args)
    assert r.returncode == 2, (args, r.stdout, r.stderr)


@pytest.mark.parametrize("case", ["few_disparities", "bad_disparity_size", "few_ground_truths", "bad_flow_size"])
def test_batch_command_refuses_lists_that_do_not_match_the_pairs(tmp_path, case):
    good = np.zeros((24, 32), np.float32)
    preprocess.write_pfm(str(tmp_path / "d.pfm"), good)
    preprocess.write_pfm(str(tmp_path / "small.pfm"), good[:20])
    preprocess.write_flo(str(tmp_path / "f.flo"), np.zeros((24, 32, 2), np.float32))
    preprocess.write_flo(str(tmp_path / "fs.flo"), np.zeros((24, 30, 2), np.float32))
    disps = {"few_disparities": "d.pfm d.pfm\nd.pfm\n", "bad_disparity_size": "d.pfm d.pfm\nd.pfm small.pfm\n"}
    gts = {"few_ground_truths": "d.pfm d.pfm f.flo\nd.pfm d.pfm\n", "bad_flow_size": "d.pfm d.pfm f.flo\nd.pfm d.pfm fs.flo\n"}
    (tmp_path / "d.txt").write_text(disps.get(case, "d.pfm d.pfm\nd.pfm d.pfm\n"))
    (tmp_path / "g.txt").write_text(gts.get(case, "d.pfm d.pfm f.flo\nd.pfm d.pfm f.flo\n"))
    r = _batch(tmp_path, "run_OF_INT", ["--scene-flow", "d.txt", "--gt-scene-flow", "g.txt"], pairs=2)
    assert r.returncode == 2, (case, r.stdout, r.stderr)
    assert not any(p.name.startswith("out") for p in tmp_path.iterdir())


def test_batch_command_accepts_scene_flow_flags(tmp_path):
    (tmp_path / "d.txt").write_text("")
    (tmp_path / "g.txt").write_text("")
    r = _batch(tmp_path, "run_OF_RGB", ["--scene-flow", "d.txt", "--camera", CAMERA, "--gt-scene-flow", "g.txt",
                                        "--kitti", "--bidirectional"])
    assert r.returncode == 0, (r.stdout, r.stderr)
