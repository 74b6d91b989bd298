"""preprocess.global_motion (the restatement of ofdis_global_motion_fullres) against a plain per-hypothesis,
per-correspondence loop written from the header, on known motions, and on its edge cases.  No GPU needed."""
import numpy as np
import pytest

from of_dis_b200 import preprocess, synth

f32 = np.float32
M64 = (1 << 64) - 1


def params(model, **kw):
    p = dict(model=model, step=2, fb_check=0, alpha=0.01, beta=0.5, hypotheses=24, threshold=1.0, refine=3, seed=7)
    p.update(kw)
    return p


# ---- the loop, from the header -------------------------------------------------------------------------------------
def mix_int(z):
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def rows_loop(model, c):
    x, y, p, q = (float(v) for v in c)
    if model == 1:
        return [x, -y, 1.0, 0.0], [y, x, 0.0, 1.0], p, q
    r1, r2 = [x, y, 1.0, 0.0, 0.0, 0.0], [0.0, 0.0, 0.0, x, y, 1.0]
    if model == 3:
        r1 += [-(x * p), -(y * p)]
        r2 += [-(x * q), -(y * q)]
    return r1, r2, p, q


def solve_loop(A, b):
    A = [list(r) for r in A]
    b = list(b)
    k = len(b)
    for j in range(k):
        piv = j
        for i in range(j + 1, k):
            if abs(A[i][j]) > abs(A[piv][j]):
                piv = i
        if not abs(A[piv][j]) > 0:
            return None
        A[j], A[piv] = A[piv], A[j]
        b[j], b[piv] = b[piv], b[j]
        for i in range(j + 1, k):
            f = A[i][j] / A[j][j]
            for c in range(j + 1, k):
                A[i][c] = A[i][c] - f * A[j][c]
            b[i] = b[i] - f * b[j]
    x = [0.0] * k
    for i in range(k - 1, -1, -1):
        s = b[i]
        for c in range(i + 1, k):
            s = s - A[i][c] * x[c]
        x[i] = s / A[i][i]
    return x if all(np.isfinite(x)) else None


def hmat_loop(model, x):
    if model == 1:
        return [x[0], -x[1], x[2], x[1], x[0], x[3], 0.0, 0.0, 1.0]
    return list(x[:6]) + (list(x[6:8]) if model == 3 else [0.0, 0.0]) + [1.0]


def inlier_loop(H, c, t):
    g = [f32(v) for v in H]
    x, y, p, q = c
    X = (g[0] * x + g[1] * y) + g[2]
    Y = (g[3] * x + g[4] * y) + g[5]
    W = (g[6] * x + g[7] * y) + g[8]
    ex, ey = X - p * W, Y - q * W
    tw = t * W
    return bool(W > 0 and ex * ex + ey * ey <= tw * tw)


def global_motion_loop(F, B, I1, p):
    h, w = F.shape[:2]
    model, s = p["model"], p["step"]
    n_min = model + 1
    cxf, cyf = f32(0.5) * f32(w - 1), f32(0.5) * f32(h - 1)
    sig = f32(2.0) / f32(max(w, h))
    cm = preprocess.consistency_check(F, B, p["alpha"], p["beta"])[0] if p["fb_check"] else None

    def valid(X, Y):
        u, v = F[Y, X]
        if not (abs(u) <= f32(1e9) and abs(v) <= f32(1e9)):
            return False
        xs, ys = f32(X) + u, f32(Y) + v
        if not (xs >= 0 and xs <= f32(w - 1) and ys >= 0 and ys <= f32(h - 1)):
            return False
        return cm is None or cm[Y, X] == 0

    corr = []
    for j in range((h - 1) // s + 1):
        for i in range((w - 1) // s + 1):
            cx, cy = min(i * s + s // 2, w - 1), min(j * s + s // 2, h - 1)
            if valid(cx, cy):
                u, v = F[cy, cx]
                corr.append(((f32(cx) - cxf) * sig, (f32(cy) - cyf) * sig, (f32(cx) + u - cxf) * sig,
                             (f32(cy) + v - cyf) * sig))
    m = len(corr)
    t = f32(p["threshold"]) * sig
    st = dict(status=0, n_corr=m, best_hypothesis=-1, ransac_inliers=0, refits=0, n_inliers=0)
    best_key, best_x = -1, None
    if m < n_min:
        st["status"] = 1
    else:
        for hh in range(p["hypotheses"]):
            A, b = [], []
            for d in range(n_min):
                z = mix_int((p["seed"] + (8 * hh + d + 1) * 0x9E3779B97F4A7C15) & M64)
                r1, r2, b1, b2 = rows_loop(model, corr[((z >> 32) * m) >> 32])
                A += [r1, r2]
                b += [b1, b2]
            x = solve_loop(A, b)
            if x is None:
                continue
            cnt = sum(inlier_loop(hmat_loop(model, x), c, t) for c in corr)
            key = (cnt << 32) | (0xFFFFFFFF - hh)
            if key > best_key:
                best_key, best_x = key, x
        if best_x is None:
            st["status"] = 2
    if st["status"]:
        M = [float("nan")] * 9
    else:
        st["best_hypothesis"] = 0xFFFFFFFF - (best_key & 0xFFFFFFFF)
        st["ransac_inliers"] = best_key >> 32
        x = best_x
        for r in range(p["refine"] + 1):
            inl = [inlier_loop(hmat_loop(model, x), c, t) for c in corr]
            st["n_inliers"] = sum(inl)
            if r == p["refine"] or sum(inl) < n_min:
                break
            k = 2 * n_min
            ne = k * (k + 1) // 2 + k
            chunks = []
            for c0 in range(0, m, 32):
                acc = [0.0] * ne
                for e in range(c0, min(m, c0 + 32)):
                    if not inl[e]:
                        continue
                    r1, r2, b1, b2 = rows_loop(model, corr[e])
                    terms = [(r1[a] * r1[bb]) + (r2[a] * r2[bb]) for a in range(k) for bb in range(a, k)]
                    terms += [(r1[a] * b1) + (r2[a] * b2) for a in range(k)]
                    acc = [a + tt for a, tt in zip(acc, terms)]
                chunks.append(acc)
            while len(chunks) & (len(chunks) - 1):
                chunks.append([0.0] * ne)
            while len(chunks) > 1:
                chunks = [[a + bb for a, bb in zip(chunks[i], chunks[i + 1])] for i in range(0, len(chunks), 2)]
            v = chunks[0]
            A = [[0.0] * k for _ in range(k)]
            e = 0
            for a in range(k):
                for bb in range(a, k):
                    A[a][bb] = A[bb][a] = v[e]
                    e += 1
            xn = solve_loop(A, v[e:])
            if xn is None:
                break
            x = xn
            st["refits"] += 1
        Hm = hmat_loop(model, x)
        S, Cx, Cy = float(sig), float(cxf), float(cyf)
        Am = [0.0] * 9
        for r in range(3):
            Am[3 * r] = Hm[3 * r] * S
            Am[3 * r + 1] = Hm[3 * r + 1] * S
            Am[3 * r + 2] = Hm[3 * r + 2] - (Am[3 * r] * Cx + Am[3 * r + 1] * Cy)
        M = [0.0] * 9
        for c in range(3):
            M[c] = Am[c] / S + Cx * Am[6 + c]
            M[3 + c] = Am[3 + c] / S + Cy * Am[6 + c]
            M[6 + c] = Am[6 + c]
        if model == 3:
            d = M[8]
            M = [v / d for v in M]
    qnan = f32(np.uint32(0x7FC00000).view(f32))
    mask = np.full((h, w), 2, np.uint8)
    res = np.full((h, w, 2), qnan, f32)
    reg = np.zeros(I1.shape, np.uint8)
    I1f = I1.reshape(h, w, -1).astype(f32)
    if st["status"] == 0:
        mm = [f32(v) for v in M]
        for Y in range(h):
            for X in range(w):
                fX, fY = f32(X), f32(Y)
                mx = (mm[0] * fX + mm[1] * fY) + mm[2]
                my = (mm[3] * fX + mm[4] * fY) + mm[5]
                wq = (mm[6] * fX + mm[7] * fY) + mm[8]
                xw, yw = mx / wq, my / wq
                u, v = F[Y, X]
                rx, ry = u - (xw - fX), v - (yw - fY)
                res[Y, X] = rx, ry
                thr = f32(p["threshold"])
                mask[Y, X] = 2 if not valid(X, Y) else 0 if rx * rx + ry * ry <= thr * thr else 1
                if wq > 0 and xw >= 0 and xw <= f32(w - 1) and yw >= 0 and yw <= f32(h - 1):
                    x0, y0 = int(np.floor(xw)), int(np.floor(yw))
                    x1, y1 = min(x0 + 1, w - 1), min(y0 + 1, h - 1)
                    fx, fy = xw - f32(x0), yw - f32(y0)
                    for ch in range(I1f.shape[2]):
                        r0 = I1f[y0, x0, ch] * (f32(1) - fx) + I1f[y0, x1, ch] * fx
                        r1 = I1f[y1, x0, ch] * (f32(1) - fx) + I1f[y1, x1, ch] * fx
                        val = r0 * (f32(1) - fy) + r1 * fy
                        reg.reshape(h, w, -1)[Y, X, ch] = np.uint8(np.fmin(np.fmax(val, f32(0)), f32(255)) + f32(0.5))
    return np.array(M).reshape(3, 3), st, mask, res, reg


# ---- inputs ----------------------------------------------------------------------------------------------------------
def bits64(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def bits32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def model_flow(M, h, w):
    """The flow of the pixel map M at every pixel, float32."""
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    wq = M[2, 0] * x + M[2, 1] * y + M[2, 2]
    u = (M[0, 0] * x + M[0, 1] * y + M[0, 2]) / wq - x
    v = (M[1, 0] * x + M[1, 1] * y + M[1, 2]) / wq - y
    return np.stack([u, v], -1).astype(np.float32)


def scene(h=17, w=23, seed=3, noc=1):
    """A camera flow plus an independently moving block, a few NaN/inf/huge values and pixels that leave the frame,
    its partner (the negated flow, perturbed), and an I1."""
    rng = np.random.default_rng(seed)
    M = synth.similarity_about_centre(h, w, 2.0, 1.02, (0.7, -0.4))
    M[2, :2] = [1e-4, -2e-4]
    F = model_flow(M, h, w)
    F[3:8, 4:10] += np.array([2.5, -1.5], np.float32)
    F += rng.normal(0, 0.05, F.shape).astype(np.float32)
    F[0, 0] = np.nan
    F[1, 2, 0] = np.inf
    F[2, 5, 1] = 3e9
    F[h - 1, w - 1] = [5.0, 5.0]
    B = (-F + rng.normal(0, 0.3, F.shape)).astype(np.float32)
    I1 = rng.integers(0, 256, (h, w) + ((noc,) if noc > 1 else ()), dtype=np.uint8)
    return F, B, I1


def assert_same(got, exp, what):
    gM, gs, gm, gr, greg = got
    eM, es, em, er, ereg = exp
    assert (bits64(gM) == bits64(eM)).all() or (np.isnan(gM).all() and np.isnan(eM).all()), (what, gM, eM)
    assert {k: int(gs[k]) for k in preprocess.MOTION_STATS_DTYPE.names} == es, (what, gs, es)
    assert (gm == em).all(), what
    assert (bits32(gr) == bits32(er)).all(), what
    assert (greg == ereg).all(), what


@pytest.mark.parametrize("fb", [0, 1])
@pytest.mark.parametrize("model", [1, 2, 3])
def test_restatement_equals_the_loop(model, fb):
    for noc, refine in ((1, 3), (3, 0)):
        F, B, I1 = scene(noc=noc)
        p = params(model, fb_check=fb, refine=refine)
        got = preprocess.global_motion(F, B, I1, p)
        exp = global_motion_loop(F, B, I1, p)
        assert exp[1]["status"] == 0 and exp[1]["n_corr"] > 20
        assert_same(got, exp, (model, fb, noc, refine))
        assert set(np.unique(got[2]).tolist()) == {0, 1, 2}


def test_splitmix64_pinned_values():
    # the first outputs of SplitMix64 seeded with 1234567 (the generator's published reference values)
    seed = 1234567
    want = [6457827717110365317, 3203168211198807973, 9817491932198370423, 4593380528125082431,
            16408922859458223821]
    got = preprocess.splitmix64([(seed + n * 0x9E3779B97F4A7C15) & M64 for n in range(1, 6)])
    assert [int(v) for v in got] == want
    for z in (0, 1, M64, 0x9E3779B97F4A7C15, 123456789123456789):
        assert int(preprocess.splitmix64(z)[0]) == mix_int(z)
    idx = preprocess.motion_draws(99, 5, 4, 1000)
    for h in range(5):
        for d in range(4):
            z = mix_int((99 + (8 * h + d + 1) * 0x9E3779B97F4A7C15) & M64)
            assert idx[h, d] == ((z >> 32) * 1000) >> 32


@pytest.mark.parametrize("model", [1, 2, 3])
def test_exact_motions_are_recovered(model):
    h, w = 60, 80
    M = synth.similarity_about_centre(h, w, 1.5, 0.98, (2.25, -1.5))
    if model == 2:
        M[0, 1] += 0.03
        M[1, 0] -= 0.02
    if model == 3:
        M[2, :2] = [2e-4, -1e-4]
    F = model_flow(M, h, w)
    got, st, mask, res, _ = preprocess.global_motion(F, None, None, params(model, step=4, hypotheses=64))
    assert st["status"] == 0 and st["n_inliers"] == st["n_corr"] == st["ransac_inliers"]
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    pt = lambda A: np.stack([(A[0, 0] * x + A[0, 1] * y + A[0, 2]) / (A[2, 0] * x + A[2, 1] * y + A[2, 2]),  # noqa
                             (A[1, 0] * x + A[1, 1] * y + A[1, 2]) / (A[2, 0] * x + A[2, 1] * y + A[2, 2])], -1)
    assert np.abs(pt(got) - pt(M)).max() < 1e-3
    inside = mask != 2
    assert (mask[inside] == 0).all()


def test_repeated_indices_are_unsolvable():
    c = np.array([[0.1, 0.2, 0.15, 0.25], [-0.3, 0.4, -0.2, 0.35], [0.5, -0.1, 0.45, -0.05], [0.2, 0.6, 0.3, 0.6]],
                 np.float32)
    for model in (1, 2, 3):
        n_min = model + 1
        for sel in ([0] * n_min, list(range(n_min - 1)) + [n_min - 2]):
            r1, r2, b1, b2 = preprocess.motion_rows(model, c[sel])
            A = np.stack([r1, r2], 1).reshape(1, 2 * n_min, 2 * n_min)
            b = np.stack([b1, b2], 1).reshape(1, 2 * n_min)
            assert not preprocess.motion_solve(A, b)[1][0]
            assert solve_loop(A[0].tolist(), b[0].tolist()) is None
        r1, r2, b1, b2 = preprocess.motion_rows(model, c[:n_min])
        A = np.stack([r1, r2], 1).reshape(1, 2 * n_min, 2 * n_min)
        assert preprocess.motion_solve(A, np.stack([b1, b2], 1).reshape(1, -1))[1][0]


def test_no_correspondence_gives_status_1():
    h, w = 12, 16
    F = np.full((h, w, 2), np.nan, np.float32)
    I1 = np.full((h, w), 9, np.uint8)
    M, st, mask, res, reg = preprocess.global_motion(F, None, I1, params(3))
    assert st["status"] == 1 and st["n_corr"] == 0 and st["best_hypothesis"] == -1
    assert np.isnan(M).all() and (bits64(M) == 0x7FF8000000000000).all()
    assert (mask == 2).all() and (bits32(res) == 0x7FC00000).all() and (reg == 0).all()
    assert_same((M, st, mask, res, reg), global_motion_loop(F, None, I1, params(3)), "nan")


def test_degenerate_samples_give_status_2():
    """Exactly two valid cells: a similarity hypothesis whose two draws coincide is unsolvable; a seed whose only
    hypothesis draws one cell twice leaves no solvable hypothesis."""
    h, w = 8, 8
    F = np.full((h, w, 2), np.nan, np.float32)
    F[2, 2] = [0.5, 0.25]  # the seed pixels of cells (0, 0) and (1, 1)
    F[6, 6] = [-0.5, 0.75]
    seed = next(s for s in range(100) if len(set(preprocess.motion_draws(s, 1, 2, 2)[0])) == 1)
    I1 = np.zeros((h, w), np.uint8)
    M, st, mask, res, reg = preprocess.global_motion(F, None, I1, params(1, step=4, hypotheses=1, seed=seed))
    assert st["status"] == 2 and st["n_corr"] == 2 and np.isnan(M).all() and (mask == 2).all()
    assert_same((M, st, mask, res, reg), global_motion_loop(F, None, I1, params(1, step=4, hypotheses=1, seed=seed)),
                "degenerate")


def test_ties_take_the_lowest_hypothesis():
    """On an exact translation every solvable hypothesis has every correspondence as an inlier: the lowest solvable
    h wins."""
    h, w = 20, 24
    F = np.zeros((h, w, 2), np.float32)
    F[..., 0], F[..., 1] = 1.5, -0.75
    p = params(1, step=3, hypotheses=40, seed=5)
    _, st, mask, _, _ = preprocess.global_motion(F, None, None, p)
    m = st["n_corr"]
    idx = preprocess.motion_draws(5, 40, 2, int(m))
    first = next(h for h in range(40) if idx[h, 0] != idx[h, 1])
    assert st["best_hypothesis"] == first and st["ransac_inliers"] == m
    assert set(np.unique(mask).tolist()) <= {0, 2}


def test_clip_has_the_known_motion():
    H = synth.similarity_about_centre(48, 64, 0.5, 1.01, (3.0, 0.0))
    frames, models, masks = synth.global_motion_clip(2, 48, 64, 1, seed=1, H=H)
    assert frames.shape == (3, 48, 64) and frames.dtype == np.uint8
    assert models.shape == (2, 3, 3) and (models == H).all()
    assert masks.shape == (2, 48, 64) and 0.1 < masks.mean() < 0.2


@pytest.mark.parametrize("exe,args", [
    ("run_DE_INT", ["--global-motion", "homography", "gm.txt"]),
    ("run_DE_RGB", ["--global-motion", "affine", "gm.txt"]),
    ("run_OF_INT", ["--warm-start", "--global-motion", "homography", "gm.txt"]),
    ("run_OF_RGB", ["--global-motion", "homography", "gm.txt", "--warm-start"]),
    ("run_OF_INT", ["--global-motion", "rotation", "gm.txt"]),
    ("run_OF_INT", ["--global-motion", "affine"]),
])
def test_batch_command_refuses_global_motion(tmp_path, exe, args):
    """The stereo binaries, --warm-start and an unknown model are refused before any work."""
    import subprocess

    from of_dis_b200 import build

    bindir = build.build_host()
    lst = tmp_path / "list.txt"
    lst.write_text("")
    r = subprocess.run([str(bindir) + "/" + exe + "_batch", str(lst)] + args, capture_output=True, text=True,
                       cwd=str(tmp_path))
    assert r.returncode == 2, (args, r.stdout, r.stderr)
    assert not (tmp_path / "gm.txt").exists()


@pytest.mark.parametrize("model", ["similarity", "affine", "homography"])
def test_batch_command_accepts_global_motion(tmp_path, model):
    import subprocess

    from of_dis_b200 import build

    bindir = build.build_host()
    lst = tmp_path / "list.txt"
    lst.write_text("")
    r = subprocess.run([str(bindir) + "/run_OF_RGB_batch", str(lst), "--bidirectional", "--kitti", "--global-motion",
                        model, "gm.txt"], capture_output=True, text=True, cwd=str(tmp_path))
    assert r.returncode == 0, (r.stdout, r.stderr)
    assert (tmp_path / "gm.txt").read_text() == ""
