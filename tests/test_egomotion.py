"""preprocess.egomotion (the restatement of ofdis_egomotion_fullres) against a plain per-correspondence loop written
from the header, with planted degenerate cases; exact recovery of known rig motions on rigid_stereo_clip's exact flows
and disparities; the pose helpers."""
import math

import numpy as np
import pytest

from of_dis_b200 import preprocess, synth

CAM = dict(fx=721.5, fy=707.0, cx=300.25, cy=90.5, baseline=0.54, doffs=0.25)
F32 = np.float32
QNAN = np.uint32(0x7FC00000).view(np.float32)


def params(**kw):
    p = dict(step=2, fb_check=0, alpha=0.01, beta=0.5, edge_diff=1.0, hypotheses=48, threshold=1.0, refine=3, seed=7)
    p.update(kw)
    return p


def motion(w=(0.0, 0.0, 0.0), t=(0.0, 0.0, 0.0)):
    return np.concatenate([synth.axis_angle(w), np.asarray(t, np.float64).reshape(3, 1)], 1)


# ---- a per-correspondence loop written from the header --------------------------------------------------------------
def loop_gather(D1, xs, ys, edge):
    h, w = D1.shape
    x0, y0 = int(math.floor(xs)), int(math.floor(ys))
    x1, y1 = min(x0 + 1, w - 1), min(y0 + 1, h - 1)
    fx, fy = F32(xs - F32(x0)), F32(ys - F32(y0))
    c = [D1[y0, x0], D1[y0, x1], D1[y1, x0], D1[y1, x1]]
    known = all(0 <= v <= F32(1e9) for v in c)
    if known and F32(max(c) - min(c)) <= F32(edge):
        gx, gy = F32(1) - fx, F32(1) - fy
        r0 = F32(F32(c[0] * gx) + F32(c[1] * fx))
        r1 = F32(F32(c[2] * gx) + F32(c[3] * fx))
        return F32(F32(r0 * gy) + F32(r1 * fy))
    return c[3] if (fy >= 0.5 and fx >= 0.5) else c[2] if fy >= 0.5 else c[1] if fx >= 0.5 else c[0]


def loop_pixel(F, D0, D1, cam, edge, x, y):
    """Step 1 at one pixel: (valid, usable0, X, Y, Z, xs, ys, d1, s1)."""
    h, w = D0.shape
    with np.errstate(all="ignore"):
        xs, ys = F32(F32(x) + F[y, x, 0]), F32(F32(y) + F[y, x, 1])
        inside = bool(xs >= 0 and xs <= F32(w - 1) and ys >= 0 and ys <= F32(h - 1))
        d0 = D0[y, x]
        d1 = loop_gather(D1, xs, ys, edge) if inside else QNAN
        s0, s1 = F32(d0 + cam["doffs"]), F32(d1 + cam["doffs"])
        usable0 = bool(0 <= d0 <= F32(1e9) and s0 > 0)
        Z = F32(cam["fb"] / s0)
        X = F32(F32(F32(F32(x) - cam["cx"]) * Z) / cam["fx"])
        Y = F32(F32(F32(F32(y) - cam["cy"]) * Z) / cam["fy"])
    valid = usable0 and inside and bool(0 <= d1 <= F32(1e9)) and bool(s1 > 0)
    return valid, usable0, X, Y, Z, xs, ys, d1, s1


def loop_inlier(g, c, cam, thr):
    X, Y, Z, xs, ys, d1, s1 = c
    with np.errstate(all="ignore"):
        Xp = F32(F32(F32(F32(g[0] * X) + F32(g[1] * Y)) + F32(g[2] * Z)) + g[3])
        Yp = F32(F32(F32(F32(g[4] * X) + F32(g[5] * Y)) + F32(g[6] * Z)) + g[7])
        Zp = F32(F32(F32(F32(g[8] * X) + F32(g[9] * Y)) + F32(g[10] * Z)) + g[11])
        ex = F32(F32(F32(cam["fx"] * Xp) + F32(cam["cx"] * Zp)) - F32(xs * Zp))
        ey = F32(F32(F32(cam["fy"] * Yp) + F32(cam["cy"] * Zp)) - F32(ys * Zp))
        ed = F32(cam["fb"] - F32(s1 * Zp))
        tz = F32(F32(thr) * Zp)
        return bool(Zp > 0) and bool(F32(F32(F32(ex * ex) + F32(ey * ey)) + F32(ed * ed)) <= F32(tz * tz))


def loop_fit3(P, Q):
    def triad(A, B, C):
        u = [B[i] - A[i] for i in range(3)]
        v = [C[i] - A[i] for i in range(3)]
        L = math.sqrt((u[0] * u[0] + u[1] * u[1]) + u[2] * u[2])
        e1 = [ui / L if L > 0 else math.nan for ui in u]

        def cross(a, b):
            return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]
        nn = cross(e1, v)
        Ln = math.sqrt((nn[0] * nn[0] + nn[1] * nn[1]) + nn[2] * nn[2]) if all(map(math.isfinite, nn)) else math.nan
        n = [x / Ln if Ln > 0 else math.nan for x in nn]
        return (e1, cross(n, e1), n), L > 0 and Ln > 0
    (E, okp), (G, okq) = triad(*P), triad(*Q)
    R = [[((G[0][i] * E[0][j]) + (G[1][i] * E[1][j])) + (G[2][i] * E[2][j]) for j in range(3)] for i in range(3)]
    cP = [((P[0][i] + P[1][i]) + P[2][i]) / 3.0 for i in range(3)]
    cQ = [((Q[0][i] + Q[1][i]) + Q[2][i]) / 3.0 for i in range(3)]
    M = []
    for i in range(3):
        M += R[i] + [cQ[i] - (((R[i][0] * cP[0]) + (R[i][1] * cP[1])) + (R[i][2] * cP[2]))]
    return M, okp and okq and all(math.isfinite(x) for x in M)


def loop_q(cam, xs, ys, s1):
    with np.errstate(all="ignore"):
        Z1 = F32(cam["fb"] / s1)
        return F32(F32(F32(xs - cam["cx"]) * Z1) / cam["fx"]), F32(F32(F32(ys - cam["cy"]) * Z1) / cam["fy"]), Z1


def loop_rows(M, c, cam):
    """Step 4's residuals and Jacobian rows of one correspondence c = (X, Y, Z, xs, ys, d1, s1), from the header."""
    X, Y, Z = float(c[0]), float(c[1]), float(c[2])
    Pp = [(((M[4 * i] * X) + (M[4 * i + 1] * Y)) + (M[4 * i + 2] * Z)) + M[4 * i + 3] for i in range(3)]
    fx, fy, cx, cy, fb, doffs = (float(cam[k]) for k in ("fx", "fy", "cx", "cy", "fb", "doffs"))
    iz = 1.0 / Pp[2]
    u, v = Pp[0] * iz, Pp[1] * iz
    grads = [(fx * iz, 0.0, -((fx * iz) * u)), (0.0, fy * iz, -((fy * iz) * v)), (0.0, 0.0, -((fb * iz) * iz))]
    r = [((fx * u) + cx) - float(c[3]), ((fy * v) + cy) - float(c[4]), ((fb * iz) - doffs) - float(c[5])]
    w = [2.0 * Pp[0], 2.0 * Pp[1], 2.0 * Pp[2]]
    J = [[(a[1] * -w[2]) + (a[2] * w[1]), (a[0] * w[2]) + (a[2] * -w[0]), (a[0] * -w[1]) + (a[1] * w[0]),
          a[0], a[1], a[2]] for a in grads]
    return J, r


def loop_update(M, x):
    """[R | t] <- [C R | C t + tau] with the Cayley rotation of the header."""
    w = x[:3]
    q = (w[0] * w[0] + w[1] * w[1]) + w[2] * w[2]
    K = [[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]]
    C = [[(((1.0 - q if i == j else 0.0) + (2.0 * (w[i] * w[j]))) + (2.0 * K[i][j])) / (1.0 + q) for j in range(3)]
         for i in range(3)]
    out = []
    for i in range(3):
        row = [((C[i][0] * M[j]) + (C[i][1] * M[4 + j])) + (C[i][2] * M[8 + j]) for j in range(4)]
        row[3] = row[3] + x[3 + i]
        out += row
    return out


def loop_egomotion(F, D0, D1, camera, p):
    """One pair, scalar code, pose and stats only."""
    cam = {k: F32(camera[k]) for k in preprocess.STEREO_CAMERA_FIELDS}
    cam["fb"] = F32(cam["fx"] * cam["baseline"])
    h, w = D0.shape
    s = p["step"]
    ncx, ncy = (w - 1) // s + 1, (h - 1) // s + 1
    corr = []
    for j in range(ncy):
        for i in range(ncx):
            x, y = min(i * s + s // 2, w - 1), min(j * s + s // 2, h - 1)
            r = loop_pixel(F, D0, D1, cam, p["edge_diff"], x, y)
            if r[0]:
                corr.append(r[2:5] + r[5:7] + (r[7], r[8]))
    m = len(corr)
    if m < 3:
        return [math.nan] * 12, (1, m, -1, 0, 0, 0)
    idx = preprocess.motion_draws(p["seed"], p["hypotheses"], 3, m)
    best, best_key, hyps = -1, -1, []
    for h_ in range(p["hypotheses"]):
        cs = [corr[k] for k in idx[h_]]
        P = [[float(c[0]), float(c[1]), float(c[2])] for c in cs]
        Q = [[float(v) for v in loop_q(cam, c[3], c[4], c[6])] for c in cs]
        with np.errstate(all="ignore"):
            M, ok = loop_fit3(P, Q)
        hyps.append(M)
        if not ok:
            continue
        g = [F32(v) for v in M]
        cnt = sum(loop_inlier(g, c, cam, p["threshold"]) for c in corr)
        key = (cnt << 32) | (0xFFFFFFFF - h_)
        if key > best_key:
            best, best_key = h_, key
    if best < 0:
        return [math.nan] * 12, (2, m, -1, 0, 0, 0)
    M, refits = [float(v) for v in hyps[best]], 0
    for r in range(p["refine"] + 1):
        inl = np.array([loop_inlier([F32(v) for v in M], c, cam, p["threshold"]) for c in corr])
        cnt = int(inl.sum())
        if r == p["refine"] or cnt < 3:
            break
        rows = [loop_rows(M, c, cam) if inl[i] else None for i, c in enumerate(corr)]
        chunks = []
        for c0 in range(0, m, 32):
            acc = [0.0] * 27
            for i in range(c0, min(m, c0 + 32)):
                if not inl[i]:
                    continue
                Ji, ri = rows[i]
                e = 0
                for a in range(6):
                    for b in range(a, 6):
                        acc[e] += ((Ji[0][a] * Ji[0][b]) + (Ji[1][a] * Ji[1][b])) + (Ji[2][a] * Ji[2][b])
                        e += 1
                for a in range(6):
                    acc[e] += -(((Ji[0][a] * ri[0]) + (Ji[1][a] * ri[1])) + (Ji[2][a] * ri[2]))
                    e += 1
            chunks.append(acc)
        while len(chunks) & (len(chunks) - 1):
            chunks.append([0.0] * 27)
        while len(chunks) > 1:
            chunks = [[a + b for a, b in zip(chunks[i], chunks[i + 1])] for i in range(0, len(chunks), 2)]
        v = chunks[0]
        A, e = np.zeros((6, 6)), 0
        for a in range(6):
            for b in range(a, 6):
                A[a, b] = A[b, a] = v[e]
                e += 1
        x, ok = preprocess.motion_solve(A[None], np.array(v[21:])[None])
        if not ok[0]:
            break
        M, refits = loop_update(M, [float(v) for v in x[0]]), refits + 1
    return M, (0, m, best, best_key >> 32, refits, cnt)


def scene(h=24, w=40, seed=0, n=1, rel=None):
    """Random disparities with planted NaN, -0 and out-of-range entries, and flows (some leaving the frame) close to a
    rigid motion, with the t+1 disparity written at the four corners around each target, so that hypotheses find
    inliers."""
    rng = np.random.default_rng(seed)
    cam = dict(CAM, cx=w / 2 - 0.25, cy=h / 2 + 0.5)
    rel = motion((0.0, 0.01, 0.0), (0.05, 0.0, -0.3)) if rel is None else rel
    D0 = rng.uniform(8, 40, (n, h, w)).astype(F32)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    fb = float(F32(F32(cam["fx"]) * F32(cam["baseline"])))
    Z = fb / (D0 + cam["doffs"])
    P = np.stack([(x - cam["cx"]) * Z / cam["fx"], (y - cam["cy"]) * Z / cam["fy"], Z], -1)
    Q = P @ rel[:, :3].T + rel[:, 3]
    xs = cam["fx"] * Q[..., 0] / Q[..., 2] + cam["cx"]
    ys = cam["fy"] * Q[..., 1] / Q[..., 2] + cam["cy"]
    F = np.stack([xs - x, ys - y], -1) + rng.normal(0, 0.05, (n, h, w, 2))
    F[rng.random((n, h, w)) < 0.2] += rng.normal(0, 6, 2)  # outliers
    F = F.astype(F32)
    D1 = np.empty_like(D0)
    for k in range(n):  # the t+1 disparity at the target, splatted to the nearest pixel
        D1[k] = rng.uniform(8, 40, (h, w))
        for dx in (0, 1):
            for dy in (0, 1):
                xi, yi = np.floor(xs[k]).astype(int) + dx, np.floor(ys[k]).astype(int) + dy
                ok = (xi >= 0) & (xi < w) & (yi >= 0) & (yi < h)
                D1[k][yi[ok], xi[ok]] = (fb / Q[k][..., 2] - cam["doffs"])[ok]
    for D in (D0, D1):
        D[rng.random(D.shape) < 0.04] = np.nan
        D[rng.random(D.shape) < 0.02] = -0.0
        D[rng.random(D.shape) < 0.02] = 2e9
        D[rng.random(D.shape) < 0.02] = -0.25  # s = d + doffs = 0: not > 0
    F[:, 0, 0] = (1e3, 0.0)                     # a target outside the frame
    F[:, 1, 1] = (np.nan, 0.0)
    return F, D0, D1, cam


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("edge", [1.0, 0.0, np.inf])
def test_restatement_equals_the_loop(seed, edge):
    F, D0, D1, cam = scene(seed=seed)
    p = params(edge_diff=edge, seed=seed)
    pose, st, _, _, _ = preprocess.egomotion(F, None, D0, D1, cam, p)
    M, ref = loop_egomotion(F[0], D0[0], D1[0], cam, p)
    assert tuple(st[0].tolist()) == ref
    assert st[0]["status"] == 0
    if edge == 1.0:  # the refits ran
        assert st[0]["refits"] > 0
    assert (pose[0].ravel().view(np.uint64) == np.array(M, np.float64).view(np.uint64)).all()


def test_per_pixel_outputs_equal_the_loop():
    F, D0, D1, cam = scene(seed=5)
    p = params()
    pose, st, mask, residual, om = preprocess.egomotion(F, None, D0, D1, cam, p)
    c = {k: F32(cam[k]) for k in preprocess.STEREO_CAMERA_FIELDS}
    c["fb"] = F32(c["fx"] * c["baseline"])
    g = [F32(v) for v in pose[0].ravel()]
    h, w = D0.shape[1:]
    seen = set()
    for y in range(h):
        for x in range(w):
            valid, usable0, X, Y, Z, xs, ys, d1, s1 = loop_pixel(F[0], D0[0], D1[0], c, p["edge_diff"], x, y)
            with np.errstate(all="ignore"):
                Xp = F32(F32(F32(F32(g[0] * X) + F32(g[1] * Y)) + F32(g[2] * Z)) + g[3])
                Yp = F32(F32(F32(F32(g[4] * X) + F32(g[5] * Y)) + F32(g[6] * Z)) + g[7])
                Zp = F32(F32(F32(F32(g[8] * X) + F32(g[9] * Y)) + F32(g[10] * Z)) + g[11])
                live = valid and bool(Zp > 0)
                exp_mask = 2 if not live else 0 if loop_inlier(g, (X, Y, Z, xs, ys, d1, s1), c, p["threshold"]) else 1
                rx = F32(F[0, y, x, 0] - F32(F32(F32(F32(c["fx"] * Xp) / Zp) + c["cx"]) - F32(x)))
                ry = F32(F[0, y, x, 1] - F32(F32(F32(F32(c["fy"] * Yp) / Zp) + c["cy"]) - F32(y)))
                X1, Y1, Z1 = loop_q(c, xs, ys, s1)
                omx = [F32(X1 - Xp), F32(Y1 - Yp), F32(Z1 - Zp)]
            seen.add(exp_mask)
            assert mask[0, y, x] == exp_mask, (x, y)
            exp_r = [rx, ry] if usable0 else [QNAN, QNAN]
            exp_r = [QNAN if np.isnan(v) else v for v in exp_r]
            assert (residual[0, y, x].view(np.uint32) == np.array(exp_r, F32).view(np.uint32)).all(), (x, y)
            exp_o = [QNAN if (not live or np.isnan(v)) else v for v in omx]
            assert (om[0, y, x].view(np.uint32) == np.array(exp_o, F32).view(np.uint32)).all(), (x, y)
    assert seen == {0, 1, 2}


def test_degenerate_draws_are_unsolvable():
    P = np.array([[[0.0, 0.0, 5.0], [1.0, 0.0, 5.0], [2.0, 0.0, 5.0]],   # collinear
                  [[0.0, 0.0, 5.0], [0.0, 0.0, 5.0], [1.0, 1.0, 5.0]],   # repeated
                  [[0.0, 0.0, 5.0], [1.0, 0.0, 5.0], [0.0, 1.0, 6.0]]])  # fine
    M, ok = preprocess.ego_fit3(P, P.copy())
    assert ok.tolist() == [False, False, True]
    assert np.allclose(M[2].reshape(3, 4), np.concatenate([np.eye(3), np.zeros((3, 1))], 1), atol=1e-12)
    for k in range(3):
        assert loop_fit3(P[k].tolist(), P[k].tolist())[1] == bool(ok[k])


def test_points_behind_the_camera_are_never_inliers():
    cam = preprocess._ego_cam(CAM)
    c = np.array([[0.5, 0.25, 4.0, 300.0, 90.0, 50.0, 50.25, 0.0]], F32)
    flip = np.array([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, -1, 0], F32)  # Z' = -Z
    assert not preprocess.ego_inliers(flip[None], c, cam, 1e30)[0, 0]
    assert not loop_inlier(list(flip), tuple(c[0, :7]), cam, 1e30)


def test_too_few_correspondences_and_no_solvable_hypothesis():
    F, D0, D1, cam = scene(seed=3)
    D0[:] = np.nan
    pose, st, mask, residual, om = preprocess.egomotion(F, None, D0, D1, cam, params())
    assert st[0]["status"] == 1 and np.isnan(pose).all() and (mask == 2).all()
    assert (residual.view(np.uint32) == 0x7FC00000).all() and (om.view(np.uint32) == 0x7FC00000).all()
    # every valid cell on one line of P: three draws are always collinear
    F, D0, D1, cam = scene(seed=3)
    D0[:] = np.nan
    D0[0, 5, :] = 20.0  # one row at one depth: the points lie on a line
    _, st, _, _, _ = preprocess.egomotion(F, None, D0, D1, cam, params(step=1))
    assert st[0]["status"] == 2 and st[0]["n_corr"] >= 3
    assert loop_egomotion(F[0], D0[0], D1[0], cam, params(step=1))[1][0] == 2


@pytest.mark.parametrize("kind", ["identity", "rotation", "forward"])
def test_recovers_the_rig_motion_from_exact_flows(kind):
    cam = dict(fx=721.5, fy=721.5, cx=300.0, cy=90.0, baseline=0.54, doffs=0.0)
    rel = {"identity": motion(), "rotation": motion((0.004, -0.012, 0.003)),
           "forward": motion((0.0, 0.002, 0.0), (0.02, 0.01, -0.9))}[kind]
    clip = synth.rigid_stereo_clip(2, 180, 600, 1, 4, cam, [rel, rel])
    pose, st, mask, _, _ = preprocess.egomotion(clip["flow"], None, clip["disp"][:-1], clip["disp"][1:], cam,
                                                params(step=4, hypotheses=128, refine=5))
    for k in range(2):
        assert st[k]["status"] == 0
        R, t = pose[k][:, :3], pose[k][:, 3]
        Rt, tt = clip["poses"][k][:, :3], clip["poses"][k][:, 3]
        ang = math.acos(min(1.0, max(-1.0, 0.5 * (np.trace(R.T @ Rt) - 1.0))))
        assert ang <= 1e-4, (kind, k, ang)
        assert np.linalg.norm(t - tt) <= 1e-4 * max(np.linalg.norm(tt), 1.0), (kind, k, t, tt)


def test_pose_helpers_round_trip(tmp_path):
    rng = np.random.default_rng(1)
    rel = np.stack([motion(rng.normal(0, 0.02, 3), rng.normal(0, 0.5, 3)) for _ in range(5)])
    abs_ = preprocess.chain_poses(rel)
    assert abs_.shape == (6, 3, 4) and np.allclose(abs_[0], np.eye(4)[:3])
    for k in range(5):  # T_(k+1) = T_k inv(rel_k): rel_k maps camera k to camera k+1
        Tk, Tk1 = np.eye(4), np.eye(4)
        Tk[:3], Tk1[:3] = abs_[k], abs_[k + 1]
        M = np.eye(4)
        M[:3] = rel[k]
        assert np.allclose(np.linalg.inv(Tk1) @ Tk, M)
    path = str(tmp_path / "poses.txt")
    preprocess.write_kitti_poses(path, abs_)
    back = preprocess.read_kitti_poses(path)
    assert (back == abs_).all()
    t_err, r_err = preprocess.pose_errors(rel, back)
    assert np.allclose(t_err, 0, atol=1e-9) and np.allclose(r_err, 0, atol=1e-5)
    off = rel.copy()
    off[2, 0, 3] += 0.1
    t_err, r_err = preprocess.pose_errors(off, back)
    assert abs(t_err[2] - 0.1) < 1e-9 and np.allclose(np.delete(t_err, 2), 0, atol=1e-9)
    off = rel.copy()
    off[3, :, :3] = synth.axis_angle((0, math.radians(2.0), 0)) @ rel[3, :, :3]
    _, r_err = preprocess.pose_errors(off, back)
    assert abs(r_err[3] - 2.0) < 1e-6
    with open(path, "a") as f:
        f.write("1 2 3\n")
    with pytest.raises(ValueError):
        preprocess.read_kitti_poses(path)


# ---- batch command: --odometry and --gt-poses are refused where they do not apply (no device needed) ----------------
CAMERA = "721.5,707,16,12,0.54,0.25"


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
    preprocess.write_pfm(str(tmp_path / "d.pfm"), np.zeros((24, 32), np.float32))
    (tmp_path / "d.txt").write_text("d.pfm d.pfm\n" * pairs)
    (tmp_path / "odo").mkdir(exist_ok=True)
    return subprocess.run([str(bindir) + "/" + exe + "_batch", "list.txt"] + args, capture_output=True, text=True,
                          cwd=str(tmp_path))


SF = ["--scene-flow", "d.txt", "--camera", CAMERA]


@pytest.mark.parametrize("exe,args", [
    ("run_DE_INT", ["--odometry", "odo"] + SF), ("run_DE_RGB", ["--odometry", "odo"]),
    ("run_OF_INT", ["--warm-start", "--odometry", "odo"] + SF),
    ("run_OF_INT", ["--odometry", "odo", "--camera", CAMERA]), ("run_OF_RGB", ["--odometry", "odo", "--scene-flow", "d.txt"]),
    ("run_OF_INT", ["--gt-poses", "g.txt"] + SF), ("run_OF_INT", ["--odometry"]),
    ("run_OF_INT", ["--odometry", "missing/dir"] + SF)])
def test_batch_command_refuses_odometry_flags(tmp_path, exe, args):
    (tmp_path / "g.txt").write_text("")
    r = _batch(tmp_path, exe, args)
    assert r.returncode == 2, (args, r.stdout, r.stderr)


@pytest.mark.parametrize("case", ["few_files", "few_lines", "missing_file", "bad_numbers"])
def test_batch_command_refuses_pose_lists_that_do_not_match_the_clips(tmp_path, case):
    """Two unrelated pairs are two clips of one pair each: two poses files of at least two lines."""
    two = "1 0 0 0 0 1 0 0 0 0 1 0\n" * 2
    (tmp_path / "p.txt").write_text(two)
    (tmp_path / "short.txt").write_text(two[:len(two) // 2])
    (tmp_path / "bad.txt").write_text(two + "1 2 3\n")
    lists = {"few_files": "p.txt\n", "few_lines": "p.txt short.txt\n", "missing_file": "p.txt nope.txt\n",
             "bad_numbers": "p.txt bad.txt\n"}
    (tmp_path / "g.txt").write_text(lists[case])
    r = _batch(tmp_path, "run_OF_INT", ["--odometry", "odo", "--gt-poses", "g.txt"] + SF, pairs=2)
    assert r.returncode == 2, (case, r.stdout, r.stderr)
    assert not any(p.name.startswith("out") for p in tmp_path.iterdir())


def test_batch_command_accepts_odometry_flags(tmp_path):
    (tmp_path / "g.txt").write_text("")
    r = _batch(tmp_path, "run_OF_RGB", ["--odometry", "odo", "--gt-poses", "g.txt", "--bidirectional"] + SF)
    assert r.returncode == 0, (r.stdout, r.stderr)
    assert (tmp_path / "odo" / "odometry.txt").read_text() == ""
