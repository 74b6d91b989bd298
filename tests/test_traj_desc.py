"""preprocess.traj_descriptors / TrajStream: the float32 restatement of the device's trajectory descriptors
(ofdis_traj_begin / ofdis_traj_advance), which tests/test_traj_desc_gpu.py uses as its checker.  It is checked here
against a per-track, per-pixel loop written from the header, on the binning and segment-test edge cases, across
splits into calls, against the output bound, and for its purpose on a clip with a moving camera."""
import math

import numpy as np
import pytest

from of_dis_b200 import preprocess, synth

f32 = np.float32
TP = dict(capacity=100000, spacing=4, alpha=0.01, beta=0.5, mb_alpha=0.01, mb_beta=0.002, min_eig=4.0)
SMALL = dict(preprocess.TRAJ_DEFAULTS, L=3, nt=3, N=8, ns=2, min_disp=0.3, min_var=0.5)


def smooth_clip(n, h, w, ch, seed):
    return synth.synthetic_sequence(n + 1, h, w, ch, seed=seed, amp=1.5)


def flows(n, h, w, seed, u=0.8, v=-0.5):
    """Smooth forward flows around (u, v) and exact-ish backward partners, float32."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    F = np.empty((n, h, w, 2), f32)
    for k in range(n):
        a, b = rng.normal(0, 0.3, 2)
        F[k, ..., 0] = u + a * np.sin(xx / 7.0 + k)
        F[k, ..., 1] = v + b * np.cos(yy / 5.0 - k)
    return F, -F


# ---- a per-track, per-pixel loop written from the header -------------------------------------------------------------
def ref_bins(a, b):
    a, b = f32(a), f32(b)
    with np.errstate(over="ignore", invalid="ignore"):
        mag = np.sqrt(f32(a * a + b * b))
    if not mag <= np.finfo(f32).max:
        return None
    ang = f32(preprocess.atan2_f32(b, a))
    if ang < 0:
        ang = f32(ang + f32(6.2831855))
    fbin = f32(ang * f32(1.2732395))
    fl = f32(math.floor(float(fbin)))
    b0 = int(fl) % 8 if int(fl) == 8 else int(fl)
    m1 = f32(f32(fbin - fl) * mag)
    return b0, (b0 + 1) % 8, f32(mag - m1), m1


def ref_residual(F, m, x, y):
    """R at pixel (x, y) from the header, or None where it is unknown."""
    u, v = F[y, x]
    fx, fy = f32(x), f32(y)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        mx = f32(f32(m[0] * fx + m[1] * fy) + m[2])
        my = f32(f32(m[3] * fx + m[4] * fy) + m[5])
        wq = f32(f32(m[6] * fx + m[7] * fy) + m[8])
        ru, rv = f32(u - f32(f32(mx / wq) - fx)), f32(v - f32(f32(my / wq) - fy))
    ok = abs(u) <= 1e9 and abs(v) <= 1e9 and wq > 0 and np.isfinite(ru) and np.isfinite(rv)
    return (ru, rv) if ok else None


def ref_segment(pos, disp, p):
    """The tests of a completed segment from the header, scalar float32: (why, (mean_x, mean_y, sd_x, sd_y,
    length), sum of |d_i|); disp entries are None where R is unknown."""
    L = len(disp)
    n = f32(L + 1)
    with np.errstate(over="ignore", invalid="ignore"):
        mean = [f32(0), f32(0)]
        for c in range(2):
            for j in range(L + 1):
                mean[c] = f32(mean[c] + pos[j][c])
            mean[c] = f32(mean[c] / n)
        sd = [f32(0), f32(0)]
        for c in range(2):
            for j in range(L + 1):
                q = f32(pos[j][c] - mean[c])
                sd[c] = f32(sd[c] + f32(q * q))
            sd[c] = np.sqrt(f32(sd[c] / n))
        steps = [np.sqrt(f32(f32(f32(pos[j + 1][0] - pos[j][0]) ** 2) + f32(f32(pos[j + 1][1] - pos[j][1]) ** 2)))
                 for j in range(L)]
        length = f32(0)
        for st in steps:
            length = f32(length + st)
        mags = [np.sqrt(f32(f32(d[0] * d[0]) + f32(d[1] * d[1]))) if d is not None else f32(np.nan) for d in disp]
        dsum = f32(0)
        for a in mags:
            dsum = f32(dsum + a)
    stats = (mean[0], mean[1], sd[0], sd[1], length)
    if sd[0] < f32(p["min_var"]) and sd[1] < f32(p["min_var"]):
        return 1, stats, dsum
    if sd[0] > f32(p["max_var"]) or sd[1] > f32(p["max_var"]):
        return 2, stats, dsum
    smax = max(steps)
    if smax > f32(p["max_dis"]) and smax > f32(f32(0.7) * length):
        return 3, stats, dsum
    if not all(np.isfinite(a) for a in mags) or max(mags) <= f32(p["min_disp"]):
        return 4, stats, dsum
    return 0, stats, dsum


def ref_pixel(I, F, m, X, Y, min_flow):
    """The 33 contributions of pixel (X, Y) of source frame I with flow F and float32 model m, from the header."""
    h, w = F.shape[:2]

    def g(x, y):
        p = I[y, x]
        return f32((f32(p[0]) + f32(p[1]) + f32(p[2])) / f32(3)) if I.ndim == 3 else f32(p)

    def R(x, y):
        return ref_residual(F, m, x, y)

    xl, xr, yu, yd = max(X - 1, 0), min(X + 1, w - 1), max(Y - 1, 0), min(Y + 1, h - 1)
    out = np.zeros(33, f32)

    def put(lo, bins):
        if bins is not None:
            out[lo + bins[0]] += bins[2]
            out[lo + bins[1]] += bins[3]

    put(0, ref_bins(f32(f32(g(xr, Y) - g(xl, Y)) * f32(0.5)), f32(f32(g(X, yd) - g(X, yu)) * f32(0.5))))
    r = R(X, Y)
    if r is not None:
        bins = ref_bins(*r)
        if bins is not None and np.sqrt(f32(r[0] * r[0] + r[1] * r[1])) <= f32(min_flow):
            out[16] += f32(1)
        else:
            put(8, bins)
    nb = [R(xl, Y), R(xr, Y), R(X, yu), R(X, yd)]
    if all(q is not None for q in nb):
        for c, lo in ((0, 17), (1, 25)):
            put(lo, ref_bins(f32(f32(nb[1][c] - nb[0][c]) * f32(0.5)), f32(f32(nb[3][c] - nb[2][c]) * f32(0.5))))
    return out


def ref_hist(I, F, m, x, y, p):
    h, w = F.shape[:2]
    N, ns = p["N"], p["ns"]
    c = N // ns
    xr, yr = int(math.floor(f32(x + f32(0.5)))), int(math.floor(f32(y + f32(0.5))))
    ox, oy = min(max(xr - N // 2, 0), w - N), min(max(yr - N // 2, 0), h - N)
    v = np.zeros((ns * ns, 33), f32)
    for cx in range(ns):
        for cy in range(ns):
            lanes = np.zeros((32, 33), f32)
            for q in range(c * c):
                lanes[q % 32] = lanes[q % 32] + ref_pixel(I, F, m, ox + cx * c + q % c, oy + cy * c + q // c,
                                                          p["min_flow"])
            s = lanes[0].copy()
            for l in range(1, 32):
                s = s + lanes[l]
            v[cx * ns + cy] = s + f32(p["eps"])
    out = np.empty_like(v)
    for lo, nb in ((0, 8), (8, 9), (17, 8), (25, 8)):
        s = f32(0)
        for cell in range(ns * ns):
            for k in range(nb):
                s = f32(s + v[cell, lo + k])
        out[:, lo:lo + nb] = np.sqrt(v[:, lo:lo + nb] / s)
    return out


def ref_descriptors(clip, F, B, models, p):
    """Follows every id through the tracker's lists; emits segments in pair order, then id order."""
    lists, _ = preprocess.track_points(clip, F, B, TP)
    L, nt, tl = p["L"], p["nt"], p["L"] // p["nt"]
    n = len(lists) - 1
    ms = [preprocess.traj_model(None if models is None else models[k]) for k in range(n)]
    where = [{int(t["id"]): (t["x"], t["y"]) for t in l} for l in lists]
    born = {}
    for f, l in enumerate(where):
        for i in l:
            born.setdefault(i, f)
    out = []  # (pair, id, record, desc)
    counts = dict.fromkeys(preprocess.TRAJ_STATS_FIELDS, 0)
    for i, b in born.items():
        s = b
        while s + L <= n and all(i in where[f] for f in range(s, s + L + 1)):
            pos = np.array([where[f][i] for f in range(s, s + L + 1)], f32)
            disp = np.empty((L, 2), f32)
            dref = []
            acc = np.zeros((nt, p["ns"] ** 2, 33), f32)
            for j in range(L):
                f = s + j
                x, y = pos[j]
                xr, yr = int(math.floor(f32(x + f32(0.5)))), int(math.floor(f32(y + f32(0.5))))
                dref.append(ref_residual(F[f], ms[f], xr, yr))
                disp[j] = dref[-1] if dref[-1] is not None else np.nan
                hst = ref_hist(clip[f], F[f], ms[f], x, y, p)
                acc[j // tl] = hst if j % tl == 0 else acc[j // tl] + hst
            why, st, dsum = ref_segment(pos, dref, p)
            if why:
                counts[preprocess.TRAJ_STATS_FIELDS[why]] += 1
            else:
                counts["emitted"] += 1
                rec = np.zeros(1, preprocess.TRAJ_RECORD_DTYPE)
                rec["id"], rec["start"] = i, s
                for k, val in zip(("mean_x", "mean_y", "sd_x", "sd_y", "length"), st):
                    rec[k] = val
                parts = [(disp / dsum).reshape(-1)]
                for lo, nb in ((0, 8), (8, 9), (17, 8), (25, 8)):
                    parts.append((acc[:, :, lo:lo + nb] / f32(tl)).reshape(-1))
                out.append((s + L - 1, i, rec, np.concatenate(parts).astype(f32)))
            s += L
    out.sort(key=lambda e: (e[0], e[1]))
    n_desc = np.bincount([e[0] for e in out], minlength=n).astype(np.int32)
    recs = np.concatenate([e[2] for e in out]) if out else np.zeros(0, preprocess.TRAJ_RECORD_DTYPE)
    desc = np.stack([e[3] for e in out]) if out else np.zeros((0, preprocess.traj_dim(p)), f32)
    return recs, desc, n_desc, counts


def bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint8),
                                                 np.ascontiguousarray(b).view(np.uint8))


@pytest.mark.parametrize("ch,models,p", [
    (1, None, SMALL), (3, "sim", SMALL), (1, "sim", dict(SMALL, L=4, nt=2, N=9, ns=3, min_flow=0.9)),
    (3, "nan", dict(SMALL, L=2, nt=1, N=6, ns=1))], ids=["gray", "rgb-models", "gray-models-odd", "rgb-nan-models"])
def test_restatement_matches_the_header_loop(ch, models, p):
    h, w, n = 14, 18, 7
    clip = smooth_clip(n, h, w, ch, seed=3)
    F, B = flows(n, h, w, seed=4)
    M = None
    if models:
        M = np.stack([synth.similarity_about_centre(h, w, 0.4 * k, 1.0 + 0.002 * k, (0.6, -0.2)).reshape(9)
                      for k in range(n)])
        if models == "nan":
            M[1::2] = np.nan
    exp = ref_descriptors(clip, F, B, M, p)
    lists, recs, desc, n_desc, tst, st = preprocess.traj_descriptors(clip, F, B, M, TP, p)
    assert recs.size > 0
    assert np.array_equal(n_desc, exp[2])
    assert bits_equal(recs, exp[0]) and bits_equal(desc, exp[1])
    assert st == exp[3]
    exp_lists, exp_tst = preprocess.track_points(clip, F, B, TP)
    assert len(lists) == len(exp_lists) and all(bits_equal(a, b) for a, b in zip(lists, exp_lists))
    assert tst == exp_tst


def test_orientation_bins_edge_cases():
    tiny = f32(-1e-30)
    b0, m0, m1 = preprocess.orientation_bins([1.0, 0.0, -1.0, 0.0, 1.0, 0.0, np.nan, 3e38],
                                             [tiny, 0.0, 0.0, 1.0, -1.0, -0.0, 1.0, 3e38])
    # an angle just below 0 goes to 2 pi, whose fbin rounds to 8: bin 0 and the rest of the weight in bin 1
    assert b0[0] == 0 and m0[0] + m1[0] == f32(1)
    # zero vectors: bin 0 with both weights 0; (-1, 0): pi, fbin 4
    assert b0[1] == 0 and m0[1] == 0 and m1[1] == 0
    assert b0[2] in (3, 4) and m0[2] + m1[2] == f32(1)
    assert b0[3] in (1, 2) and b0[4] in (6, 7)
    assert b0[5] == 0 and m0[5] == 0 and m1[5] == 0
    # unknown and non-finite magnitudes give no bin
    assert b0[6] == 255 and b0[7] == 255 and m0[6] == m1[6] == 0
    # every bin index is in range and both weights are non-negative
    rng = np.random.default_rng(1)
    a, b = rng.normal(0, 5, 10000).astype(f32), rng.normal(0, 5, 10000).astype(f32)
    b0, m0, m1 = preprocess.orientation_bins(a, b)
    assert b0.max() <= 7 and (m0 >= 0).all() and (m1 >= 0).all()


def test_hof_zero_bin_unknown_flow_and_nonpositive_w():
    h, w = 6, 7
    I = np.full((h, w), 100, np.uint8)
    F = np.zeros((h, w, 2), f32)
    F[..., 0] = 0.4                 # exactly min_flow: the zero bin
    F[1, 1] = (np.nan, 0.0)         # unknown F
    F[2, 2] = (2e9, 0.0)            # beyond 1e9: unknown
    F[3, 3] = (0.5, 0.0)            # above min_flow: a real bin
    eye = preprocess.traj_model(None)
    c, R, known = preprocess.traj_fields(I, F, eye, 0.4)
    assert c[0, 0, 16] == 1 and c[0, 0, 8:16].sum() == 0
    assert c[1, 1, 8:17].sum() == 0 and not known[1, 1] and not known[2, 2]
    assert c[3, 3, 16] == 0 and c[3, 3, 8] == f32(0.5)
    # MBH of a pixel next to an unknown R is unknown; a flat frame has zero gradients (bin 0, weight 0)
    assert c[1, 2, 17:].sum() == 0 and c[0, 0, :8].sum() == 0
    # a model whose w is not positive makes R unknown there (left half: w = 1 - 0.5 x <= 0 from x = 2)
    m = np.array([1, 0, 0, 0, 1, 0, -0.5, 0, 1], f32)
    _, _, known = preprocess.traj_fields(I, F, m, 0.4)
    assert known[0, :2].all() and not known[0, 2:].any()


def test_patches_clamp_at_all_four_borders():
    h, w = 12, 14
    p = dict(SMALL, N=8, ns=2)
    rng = np.random.default_rng(2)
    contrib = rng.random((h, w, 33)).astype(f32)
    xs = np.array([0.0, 13.0, 0.4, 6.6], f32)
    ys = np.array([0.0, 11.0, 11.0, 0.2], f32)
    got = preprocess.traj_frame_hist(contrib, xs, ys, p)
    # the clamped patches are the ones at the corners and the same as positions a few pixels inside
    inner = preprocess.traj_frame_hist(contrib, np.array([2.0, 11.0, 3.0, 6.6], f32),
                                       np.array([3.0, 8.0, 9.0, 3.0], f32), p)
    assert bits_equal(got, inner)


def seg(xs, ys, d=1.5):
    L = len(xs) - 1
    pos = np.stack([xs, ys], -1).astype(f32)
    disp = np.full((L, 2), f32(d), f32)
    return pos, disp


@pytest.mark.parametrize("case,why", [
    ("static", 1), ("just_moving", 0), ("erratic", 2), ("jump", 3), ("jump_spread", 0), ("camera", 4),
    ("camera_edge", 4), ("camera_beside", 0), ("unknown_d", 4)])
def test_segment_tests(case, why):
    p = dict(preprocess.TRAJ_DEFAULTS, L=4, nt=2)
    line = np.arange(5, dtype=f32)
    if case == "static":
        pos, disp = seg(10 + 0.1 * line, 20 + 0.1 * line)
    elif case == "just_moving":
        pos, disp = seg(10 + 2 * line, 20 + 0 * line)  # sd 2 sqrt(2) > sqrt(3)
    elif case == "erratic":
        pos, disp = seg(10 + 40 * line, 20 + 0 * line)  # sd 40 sqrt(2) > 50
    elif case == "jump":
        pos, disp = seg(np.array([10, 10.5, 11, 40, 40.5], f32), np.full(5, 20, f32))
    elif case == "jump_spread":
        pos, disp = seg(10 + 21 * line, 20 + 0 * line)  # steps of 21 > max_dis, but each < 0.7 length
    elif case == "camera":
        pos, disp = seg(10 + 2 * line, 20 + 0 * line, d=0.5)
    elif case == "camera_edge":
        pos, disp = seg(10 + 2 * line, 20 + 0 * line, d=0.0)
        disp[2] = (1.0, 0.0)  # max |d| == min_disp
    elif case == "camera_beside":
        pos, disp = seg(10 + 2 * line, 20 + 0 * line, d=0.0)
        disp[2] = (np.nextafter(f32(1), f32(2)), 0.0)
    else:
        pos, disp = seg(10 + 2 * line, 20 + 0 * line)
        disp[1] = np.nan
    got, st, _ = preprocess.traj_segment_test(pos, disp, p)
    assert got == why, (case, got, st)


def test_static_and_erratic_thresholds_are_strict():
    p = dict(preprocess.TRAJ_DEFAULTS, L=1, nt=1)
    # two points 2 a apart have sd a: at a = min_var (not below it) the segment is not static
    a = f32(p["min_var"])
    pos = np.array([[0, 0], [2 * a, 2 * a]], f32)
    _, st, _ = preprocess.traj_segment_test(pos, np.full((1, 2), 5, f32), p)
    assert preprocess.traj_segment_test(pos, np.full((1, 2), 5, f32), dict(p, min_var=float(st[2])))[0] != 1
    assert preprocess.traj_segment_test(pos, np.full((1, 2), 5, f32),
                                        dict(p, min_var=float(np.nextafter(st[2], f32(9)))))[0] == 1
    assert preprocess.traj_segment_test(pos, np.full((1, 2), 5, f32), dict(p, max_var=float(st[2])))[0] != 2
    assert preprocess.traj_segment_test(pos, np.full((1, 2), 5, f32),
                                        dict(p, max_var=float(np.nextafter(st[2], f32(0)))))[0] == 2


def test_a_track_of_2L_plus_3_frames_emits_two_segments_sharing_an_endpoint():
    h, w, L = 24, 48, 3
    p = dict(SMALL, L=L, nt=1, N=8, min_var=0.1, min_disp=0.1)
    n = 2 * L + 2  # the track lives 2L + 3 frames
    clip = smooth_clip(n, h, w, 1, seed=5)
    F = np.zeros((n, h, w, 2), f32)
    F[..., 0] = 0.75
    tp = dict(TP, spacing=48, capacity=1)  # one track, seeded at (24, 23)
    lists, recs, desc, n_desc, _, st = preprocess.traj_descriptors(clip, F, -F, None, tp, p)
    assert all(l.size == 1 and l["id"][0] == 0 for l in lists)
    assert recs.size == 2 and list(recs["start"]) == [0, L] and st["emitted"] == 2
    assert list(n_desc) == [0, 0, 1, 0, 0, 1, 0, 0]
    # the second segment starts at the first one's last point
    x = lambda f: f32(24) + f32(0.75) * f  # noqa: E731
    assert recs["mean_x"][0] < x(L) < recs["mean_x"][1]
    assert desc.shape == (2, preprocess.traj_dim(p))


def test_every_split_into_calls_gives_the_same_output():
    h, w, n = 16, 20, 9
    p = SMALL
    clip = smooth_clip(n, h, w, 3, seed=6)
    F, B = flows(n, h, w, seed=7)
    M = np.stack([synth.similarity_about_centre(h, w, 0.3, 1.0, (0.5, -0.3)).reshape(9)] * n)
    one = preprocess.traj_descriptors(clip, F, B, M, TP, p)
    assert one[1].size > 0
    for cuts in ([0, 1, n], [0, 2, 3, 7, n], list(range(n + 1))):
        s = preprocess.TrajStream(TP, p)
        s.begin(clip[0])
        parts = [s.advance(clip[a + 1:b + 1], F[a:b], B[a:b], M[a:b]) for a, b in zip(cuts[:-1], cuts[1:])]
        assert bits_equal(np.concatenate([q[1] for q in parts]), one[1])
        assert bits_equal(np.concatenate([q[2] for q in parts]), one[2])
        assert np.array_equal(np.concatenate([q[3] for q in parts]), one[3])
        assert dict(s.tstats) == one[5]


def test_the_output_bound_is_reached_and_not_exceeded():
    """A full tracker whose tracks never end: every call of n pairs emits at most capacity * ceil((n + L - 1) / L)
    segments, and a call that ends the L - 1 carried steps of every track reaches it."""
    h, w, L = 40, 40, 3
    p = dict(SMALL, L=L, nt=1, N=8, min_var=0.0, min_disp=0.0)
    cap = 9
    tp = dict(TP, spacing=12, capacity=cap, min_eig=-1.0)
    n = 3 * L + 2
    clip = smooth_clip(n, h, w, 1, seed=8)
    F = np.zeros((n, h, w, 2), f32)
    F[..., 0] = -0.25  # to the left: the seeds at x = W-1 stay in the frame
    s = preprocess.TrajStream(tp, p)
    first = s.begin(clip[0])
    assert first.size == cap
    for a, b in ((0, L - 1), (L - 1, L), (L, 2 * L + 1), (2 * L + 1, n)):
        _, recs, _, n_desc, = s.advance(clip[a + 1:b + 1], F[a:b], -F[a:b])
        bound = preprocess.traj_bound(cap, b - a, L)
        assert recs.size <= bound
        if (a, b) == (L - 1, L):  # one pair completes every track's first segment
            assert recs.size == bound == cap


def gm_flows(H, bm, masks, block, h, w):
    """Analytic forward and backward flows of synth.global_motion_clip."""
    n = masks.shape[0]
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    Hi = np.linalg.inv(H)

    def apply(A):
        q = A[2, 0] * xx + A[2, 1] * yy + A[2, 2]
        return (A[0, 0] * xx + A[0, 1] * yy + A[0, 2]) / q - xx, (A[1, 0] * xx + A[1, 1] * yy + A[1, 2]) / q - yy

    fu, fv = apply(H)
    bu, bv = apply(Hi)
    F = np.empty((n, h, w, 2), f32)
    B = np.empty_like(F)
    X0, Y0, X1, Y1 = block[0] * w, block[1] * h, block[2] * w, block[3] * h
    for t in range(n):
        F[t, ..., 0] = np.where(masks[t], bm[0], fu)
        F[t, ..., 1] = np.where(masks[t], bm[1], fv)
        bx, by = xx - (t + 1) * bm[0], yy - (t + 1) * bm[1]
        ins = (bx >= X0) & (bx < X1) & (by >= Y0) & (by < Y1)
        B[t, ..., 0] = np.where(ins, -bm[0], bu)
        B[t, ..., 1] = np.where(ins, -bm[1], bv)
    return F, B


def test_purpose_on_a_camera_motion_clip():
    """Analytic flows and true models of synth.global_motion_clip: compensated, the background's segments all go as
    camera motion and the rectangle's are emitted; without models the background's are emitted."""
    h, w, n = 64, 96, 16
    block, bm = (0.45, 0.25, 0.8, 0.8), (-2.0, 1.5)
    H = synth.similarity_about_centre(h, w, 0.3, 1.0, (1.5, 0.5))
    clip, models, masks = synth.global_motion_clip(n, h, w, 1, seed=3, H=H, block=block, block_motion=bm)
    F, B = gm_flows(H, bm, masks, block, h, w)
    p = dict(preprocess.TRAJ_DEFAULTS, N=16)
    tp = dict(TP, min_eig=1.0)
    figures = {}
    for comp in (True, False):
        _, recs, _, _, _, st = preprocess.traj_descriptors(clip, F, B, models.reshape(n, 9) if comp else None, tp, p)
        inside = sum(bool(masks[int(r["start"]) + 7][min(int(round(float(r["mean_y"]))), h - 1),
                                                     min(int(round(float(r["mean_x"]))), w - 1)]) for r in recs)
        figures[comp] = dict(st, rect=inside, background=int(recs.size) - inside)
    comp, raw = figures[True], figures[False]
    # measured: of the 90 background segments that are emitted without models, all 90 go as camera motion with them;
    # all 48 rectangle segments are emitted either way.  Asserted with a margin of 10 %.
    assert raw["background"] >= 80 and raw["rejected_camera"] == 0, figures
    assert comp["rejected_camera"] >= 0.9 * raw["background"] and comp["background"] <= 0.1 * raw["background"], figures
    assert comp["rect"] >= 0.9 * raw["rect"] and raw["rect"] >= 40, figures


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


@pytest.mark.parametrize("exe,args", [
    ("run_DE_INT", ["--tracks", "t.txt", "--descriptors", "d.txt"]),
    ("run_DE_RGB", ["--tracks", "t.txt", "--descriptors", "d.txt"]),
    ("run_OF_INT", ["--warm-start", "--tracks", "t.txt", "--descriptors", "d.txt"]),
    ("run_OF_INT", ["--warm-start", "--descriptors", "d.txt"]),
    ("run_OF_RGB", ["--descriptors", "d.txt"]),
    ("run_OF_INT", ["--global-motion", "affine", "gm.txt", "--descriptors", "d.txt"]),
    ("run_OF_INT", ["--tracks", "t.txt", "--descriptors"]),
    ("run_OF_INT", ["--tracks", "t.txt", "--descriptors", "d.txt", "small"]),
    ("run_OF_RGB", ["--tracks", "t.txt", "--descriptors", "d.txt", "narrow"]),
    ("run_OF_INT", ["--tracks", "t.txt", "--descriptors", "missing/dir/d.txt"]),
])
def test_batch_command_refuses_descriptors(tmp_path, exe, args):
    """The stereo binaries, --warm-start, a missing --tracks, frames smaller than the 32 x 32 patch and an unwritable
    path are refused before any device work, and no output file is written."""
    import subprocess

    from of_dis_b200 import build

    bindir = build.build_host()
    lst = tmp_path / "list.txt"
    size = {"small": (20, 40), "narrow": (64, 31)}.get(args[-1])
    if size:
        args = args[:-1]
        ch = 3 if exe.endswith("RGB") else 1
        for k in range(2):
            _write_png(str(tmp_path / ("f%d.png" % k)), smooth_clip(0, size[0], size[1], ch, seed=k)[0])
        lst.write_text("f0.png f1.png out.flo\n")
    else:
        lst.write_text("")
    r = subprocess.run([str(bindir) + "/" + exe + "_batch", str(lst)] + args, capture_output=True, text=True,
                       cwd=str(tmp_path))
    expect = 1 if "missing/dir/d.txt" in args else 2
    assert r.returncode == expect, (args, r.stdout, r.stderr)
    assert sorted(q.name for q in tmp_path.iterdir()) == sorted(["list.txt"] + (["f0.png", "f1.png"] if size else []))


def test_batch_command_accepts_descriptors(tmp_path):
    import subprocess

    from of_dis_b200 import build

    bindir = build.build_host()
    lst = tmp_path / "list.txt"
    lst.write_text("")
    r = subprocess.run([str(bindir) + "/run_OF_RGB_batch", str(lst), "--global-motion", "homography", "gm.txt",
                        "--tracks", "t.txt", "--descriptors", "d.txt"], capture_output=True, text=True,
                       cwd=str(tmp_path))
    assert r.returncode == 0, (r.stdout, r.stderr)
    assert (tmp_path / "d.txt").read_text() == "# clip id start mean_x mean_y sd_x sd_y length d0 .. d425\n"
    assert (tmp_path / "t.txt").read_text() == "# clip frame id x y\n"
