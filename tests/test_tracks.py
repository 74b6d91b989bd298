"""preprocess.track_points: the float32 restatement of the device tracker (ofdis_track_begin / ofdis_track_advance),
which tests/test_tracks_gpu.py uses as its checker.  It is checked here against a per-track loop written from the
header, and on flows whose tracks are known."""
import math

import numpy as np

from of_dis_b200 import preprocess

f32 = np.float32
PARAMS = dict(capacity=100000, spacing=4, alpha=0.01, beta=0.5, mb_alpha=0.01, mb_beta=0.002, min_eig=25.0)


def textured(n, h, w, ch=1, seed=0):
    rng = np.random.default_rng(seed)
    shape = (n, h, w) + ((ch,) if ch > 1 else ())
    return rng.integers(0, 256, shape, dtype=np.uint8)


def const_flow(n, h, w, u, v):
    F = np.empty((n, h, w, 2), f32)
    F[..., 0], F[..., 1] = u, v
    return F


def run(clip, F, B, **kw):
    return preprocess.track_points(clip, F, B, dict(PARAMS, **kw))


# ---- a per-track loop written from the header ---------------------------------------------------------------------
def ref_track_points(clip, F, B, p):
    n, h, w = clip.shape[0] - 1, clip.shape[1], clip.shape[2]
    nop = F.shape[-1]
    s = p["spacing"]
    ncx, ncy = (w - 1) // s + 1, (h - 1) // s + 1

    def gray(I, x, y):
        px = I[y, x]
        if I.ndim == 3:
            return (f32(px[0]) + f32(px[1]) + f32(px[2])) / f32(3)
        return f32(px)

    def lam(I, cx, cy):
        a = b = c = f32(0)
        for dy in range(-2, 3):
            py = min(max(cy + dy, 0), h - 1)
            for dx in range(-2, 3):
                px = min(max(cx + dx, 0), w - 1)
                ix = (gray(I, min(px + 1, w - 1), py) - gray(I, max(px - 1, 0), py)) * f32(0.5)
                iy = (gray(I, px, min(py + 1, h - 1)) - gray(I, px, max(py - 1, 0))) * f32(0.5)
                a, b, c = a + ix * ix, b + ix * iy, c + iy * iy
        d = a - c
        return (a + c) * f32(0.5) - np.sqrt(d * d * f32(0.25) + b * b)

    def bil(Fk, x, y):
        x0, y0 = int(math.floor(x)), int(math.floor(y))
        x1, y1 = min(x0 + 1, w - 1), min(y0 + 1, h - 1)
        fx, fy = x - f32(x0), y - f32(y0)
        gx, gy = f32(1) - fx, f32(1) - fy
        return [(Fk[y0, x0, c] * gx + Fk[y0, x1, c] * fx) * gy + (Fk[y1, x0, c] * gx + Fk[y1, x1, c] * fx) * fy
                for c in range(nop)] + [f32(0)] * (2 - nop)

    st = dict.fromkeys(preprocess.TRACK_STATS_FIELDS, 0)
    tracks, next_id = [], 0

    def seed(I):
        nonlocal tracks, next_id
        occ = {(int(x) // s, int(y) // s) for _, x, y in tracks}
        for j in range(ncy):
            for i in range(ncx):
                cx, cy = min(i * s + s // 2, w - 1), min(j * s + s // 2, h - 1)
                if (i, j) in occ or not lam(I, cx, cy) >= f32(p["min_eig"]):
                    continue
                if len(tracks) < p["capacity"] and next_id < 2 ** 31 - 1:
                    tracks.append((next_id, f32(cx), f32(cy)))
                    next_id += 1
                    st["seeded"] += 1
                else:
                    st["dropped"] += 1

    def advance(Fk, Bk):
        nonlocal tracks
        out = []
        for tid, x, y in tracks:
            u, v = bil(Fk, x, y)
            xn, yn = x + u, y + v
            if not (xn >= 0 and xn <= f32(w - 1) and yn >= 0 and yn <= f32(h - 1)):
                st["ended_leaves"] += 1
                continue
            b0, b1 = bil(Bk, xn, yn)
            du, dv = u + b0, v + b1
            err, mag = du * du + dv * dv, (u * u + v * v) + (b0 * b0 + b1 * b1)
            if not err <= f32(p["alpha"]) * mag + f32(p["beta"]):
                st["ended_inconsistent"] += 1
                continue
            xr, yr = int(math.floor(x + f32(0.5))), int(math.floor(y + f32(0.5)))
            l, r = Fk[yr, max(xr - 1, 0)], Fk[yr, min(xr + 1, w - 1)]
            up, dn = Fk[max(yr - 1, 0), xr], Fk[min(yr + 1, h - 1), xr]
            ux, uy = (r[0] - l[0]) * f32(0.5), (dn[0] - up[0]) * f32(0.5)
            g2 = ux * ux + uy * uy
            if nop == 2:
                vx, vy = (r[1] - l[1]) * f32(0.5), (dn[1] - up[1]) * f32(0.5)
                g2 = g2 + (vx * vx + vy * vy)
            if g2 > f32(p["mb_alpha"]) * (u * u + v * v) + f32(p["mb_beta"]):
                st["ended_boundary"] += 1
                continue
            out.append((tid, xn, yn))
        tracks = out

    lists = []
    seed(clip[0])
    lists.append(list(tracks))
    for k in range(n):
        advance(F[k], B[k])
        seed(clip[k + 1])
        lists.append(list(tracks))
    st["alive"], st["next_id"] = len(tracks), next_id
    return lists, st


def assert_lists_equal(got, exp):
    assert len(got) == len(exp)
    for k, (g, e) in enumerate(zip(got, exp)):
        e = np.array(e, preprocess.TRACK_POINT_DTYPE)
        assert g.dtype == preprocess.TRACK_POINT_DTYPE and g.shape == e.shape, (k, g.shape, e.shape)
        assert np.array_equal(g.view(np.uint8), e.view(np.uint8)), "frame %d differs" % k


def smooth_flows(n, h, w, nop, seed):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(f32)
    F = np.empty((n, h, w, nop), f32)
    B = np.empty_like(F)
    for k in range(n):
        for c in range(nop):
            a, fx, fy = rng.uniform(1, 3), rng.uniform(0.02, 0.1), rng.uniform(0.02, 0.1)
            F[k, ..., c] = (a * np.sin(fx * x + k) * np.cos(fy * y)).astype(f32)
        B[k] = -F[k] + rng.normal(0, 0.4, F[k].shape).astype(f32)
    # a step, so that motion boundaries end some tracks
    F[:, :, w // 2:, 0] += f32(2.5)
    B[:, :, w // 2:, 0] -= f32(2.5)
    return F, B


def test_restatement_equals_the_per_track_loop():
    for nop, ch, seed in ((2, 1, 1), (2, 3, 2), (1, 1, 3), (1, 3, 4)):
        h, w, n = 29, 37, 3
        clip = textured(n + 1, h, w, ch, seed)
        clip[:, 10:20, 5:15] = 128  # a flat patch seeds nothing
        F, B = smooth_flows(n, h, w, nop, seed)
        p = dict(PARAMS, spacing=3, min_eig=200.0, capacity=90)
        got, gst = preprocess.track_points(clip, F, B, p)
        exp, est = ref_track_points(clip, F, B, p)
        assert_lists_equal(got, exp)
        assert gst == est
        ended = est["ended_leaves"], est["ended_inconsistent"], est["ended_boundary"]
        assert all(e > 0 for e in ended), ended
        assert est["dropped"] > 0 and est["alive"] > 0


def test_integer_translation_moves_every_track_by_the_flow():
    h, w, n = 40, 56, 4
    clip = textured(n + 1, h, w, seed=5)
    F = const_flow(n, h, w, 3, -2)
    lists, st = run(clip, F, -F)
    assert st["ended_inconsistent"] == 0 and st["ended_boundary"] == 0
    for k in range(n):
        a, b = lists[k], lists[k + 1]
        common, ia, ib = np.intersect1d(a["id"], b["id"], return_indices=True)
        moved = (a["x"][ia] + f32(3) == b["x"][ib]) & (a["y"][ia] - f32(2) == b["y"][ib])
        assert moved.all()
        # the ones that did not survive are exactly those pushed out of the frame
        gone = np.setdiff1d(a["id"], b["id"])
        ga = a[np.isin(a["id"], gone)]
        assert ((ga["x"] + 3 > w - 1) | (ga["y"] - 2 < 0)).all()
        assert len(common) + len(gone) == len(a)


def test_tracks_leave_at_the_border_and_new_seeds_fill_uncovered_cells():
    h, w, n, s = 32, 48, 1, 4
    clip = textured(n + 1, h, w, seed=6)
    F = const_flow(n, h, w, 5, 0)
    lists, st = run(clip, F, -F, spacing=s)
    a, b = lists
    ncx, ncy = (w - 1) // s + 1, (h - 1) // s + 1
    assert len(a) == ncx * ncy  # every cell of a textured frame seeds
    assert st["ended_leaves"] == int((a["x"] + 5 > w - 1).sum()) > 0
    new = b[b["id"] >= len(a)]
    assert len(new) > 0
    # the new seeds are in the cells the moved tracks left empty: seeds at x = 2, 6, ... moved to 7, 11, ..., so the
    # leftmost column of cells, every one of them
    assert np.array_equal(new["x"], np.full(ncy, 2, f32)) and np.array_equal(new["y"], np.arange(2, h, s, dtype=f32))
    assert np.array_equal(new["id"], np.arange(len(a), len(a) + len(new)))
    assert st["alive"] == len(b) and st["next_id"] == len(a) + len(new)


def test_disagreeing_backward_flow_ends_tracks_as_inconsistent():
    h, w, n = 24, 32, 1
    clip = textured(n + 1, h, w, seed=7)
    F = const_flow(n, h, w, 1, 1)
    lists, st = run(clip, F, -F + f32(2))
    assert st["ended_inconsistent"] == len(lists[0]) - st["ended_leaves"] > 0
    assert st["ended_boundary"] == 0
    assert not np.isin(lists[1]["id"], lists[0]["id"]).any()


def test_a_step_in_the_flow_ends_tracks_as_boundary():
    h, w, n = 16, 64, 1
    clip = textured(n + 1, h, w, seed=8)
    F = const_flow(n, h, w, 0, 0)
    F[:, :, 32:, 0] = 1
    B = -F
    B[:, :, 33:, 0] = -1  # B at the targets of the moved half
    lists, st = run(clip, F, B, spacing=1, min_eig=-np.inf)
    a = lists[0]
    assert st["ended_inconsistent"] == 0
    ended = a[~np.isin(a["id"], lists[1]["id"])]
    assert st["ended_boundary"] == len(ended) - st["ended_leaves"] > 0
    # the motion boundary is at columns 31 and 32 (central differences of the step)
    inside = ended[ended["x"] + F[0, 0, ended["x"].astype(int), 0] <= w - 1]
    assert set(np.unique(inside["x"].astype(int))) == {31, 32}


def test_flat_and_striped_frames_seed_nothing():
    h, w = 20, 30
    flat = np.full((2, h, w), 77, np.uint8)
    stripes = np.zeros((2, h, w, 3), np.uint8)
    stripes[:, :, ::2] = 200
    stripes[:, :, 1::3] = 31
    for clip in (flat, stripes):
        _, _, lam = preprocess.track_seed_eigen(clip[0], 4)
        assert (lam == 0).all()
        F = const_flow(1, h, w, 0, 0)
        lists, st = run(clip, F, F, min_eig=1e-6)
        assert len(lists[0]) == len(lists[1]) == 0 and st["seeded"] == 0 and st["dropped"] == 0
    lists, st = run(stripes, const_flow(1, h, w, 0, 0), const_flow(1, h, w, 0, 0), min_eig=0.0)
    assert st["seeded"] > 0  # lambda == 0 passes min_eig 0


def test_capacity_overflow_drops_the_highest_cells():
    h, w, n, s = 32, 40, 2, 4
    clip = textured(n + 1, h, w, seed=9)
    F = const_flow(n, h, w, 4, 0)
    full, fst = run(clip, F, -F, spacing=s)
    cap = 25
    lists, st = run(clip, F, -F, spacing=s, capacity=cap)
    cells = len(full[0])
    assert np.array_equal(lists[0], full[0][:cap])  # the lowest cells
    assert st["dropped"] > 0 and st["dropped"] + st["seeded"] > cap
    assert all(len(l) <= cap for l in lists)
    assert lists[0].size == cap and st["seeded"] + st["dropped"] >= cells


def test_ids_ascend_within_every_frame():
    h, w, n = 48, 64, 6
    clip = textured(n + 1, h, w, 3, seed=10)
    F, B = smooth_flows(n, h, w, 2, 11)
    lists, st = run(clip, F, B)
    for l in lists:
        assert (np.diff(l["id"]) > 0).all()
    assert st["alive"] == len(lists[-1]) and st["seeded"] == st["next_id"]
    ended = st["ended_leaves"] + st["ended_inconsistent"] + st["ended_boundary"]
    assert st["seeded"] - ended == st["alive"]
