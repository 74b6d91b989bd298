"""Seeded synthetic image pairs with known flow (SURVEY.md section 8d).

image : sum over sigma in {1.5,3,6,12,24} of sigma * gaussian_blur(N(0,1), sigma)
        on a (H+64)x(W+64)xC canvas, min-max scaled to [0,255]
flow  : u = A sin(4x/W+.3) cos(3y/H),  v = .6A cos(2.5x/W) sin(5y/H+.7)
        (stereo: u = -(2 + A(.5+.5 sin(3.1x/W + 2y/H))), v = 0)
I0    : centre crop of the canvas;  I1(x) = canvas(x - flow(x)) (cubic), so that
        I0(x) ~= I1(x + flow(x)) (the reference's convention, patch.cpp:217)
clip  : frame t = canvas(x - t flow(x)) (synthetic_sequence; frames 0, 1 are the pair)
Both are quantised to uint8 because the reference CLI reads 8-bit images.
"""
from __future__ import annotations

import numpy as np


def synthetic_flow(h: int, w: int, amp: float = 6.0, stereo: bool = False):
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    if stereo:
        u = -(2.0 + amp * (0.5 + 0.5 * np.sin(3.1 * x / w + 2.0 * y / h)))
        v = np.zeros_like(u)
    else:
        u = amp * np.sin(4.0 * x / w + 0.3) * np.cos(3.0 * y / h)
        v = 0.6 * amp * np.cos(2.5 * x / w) * np.sin(5.0 * y / h + 0.7)
    return u, v


def _canvas(h: int, w: int, channels: int, seed: int):
    """The (h+2m)x(w+2m)xC float64 canvas in [0,255] and its margin m."""
    from scipy import ndimage

    rng = np.random.default_rng(seed)
    m = 32
    hc, wc = h + 2 * m, w + 2 * m
    canv = np.zeros((hc, wc, channels), dtype=np.float64)
    for c in range(channels):
        acc = np.zeros((hc, wc))
        for sigma in (1.5, 3.0, 6.0, 12.0, 24.0):
            acc += sigma * ndimage.gaussian_filter(rng.standard_normal((hc, wc)), sigma, mode="reflect")
        canv[..., c] = acc
    lo, hi = canv.min(), canv.max()
    return (canv - lo) / (hi - lo) * 255.0, m


def _frame(canv, m: int, h: int, w: int, u, v, t: int):
    """Frame t of the canvas' clip, quantised to uint8: frame 0 is the centre crop, frame t >= 1 the canvas
    sampled at x - t*flow(x) (cubic)."""
    from scipy import ndimage

    channels = canv.shape[2]
    if t == 0:
        img = canv[m:m + h, m:m + w]
    else:
        yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
        img = np.empty((h, w, channels))
        for c in range(channels):
            img[..., c] = ndimage.map_coordinates(canv[..., c], [yy + m - t * v, xx + m - t * u], order=3, mode="nearest")
    q = np.clip(np.rint(img), 0, 255).astype(np.uint8)
    return np.ascontiguousarray(q[..., 0] if channels == 1 else q)


def synthetic_pair(h: int, w: int, channels: int = 1, seed: int = 0, amp: float = 6.0, stereo: bool = False):
    """Returns (img0_u8, img1_u8, flow_gt[h,w,2]); images are (h,w) or (h,w,3)."""
    canv, m = _canvas(h, w, channels, seed)
    u, v = synthetic_flow(h, w, amp, stereo)
    # I1(x + f(x)) = I0(x); first-order inverse: I1(x) = canvas(x - f(x))
    i0, i1 = _frame(canv, m, h, w, u, v, 0), _frame(canv, m, h, w, u, v, 1)
    return i0, i1, np.stack([u, v], -1).astype(np.float32)


def synthetic_sequence(n_frames: int, h: int, w: int, channels: int = 1, seed: int = 0, amp: float = 6.0,
                       stereo: bool = False):
    """A clip of n_frames uint8 frames, [n_frames][h][w] or [n_frames][h][w][3]: frame t is the canvas sampled at
    x - t*flow(x), so frames 0 and 1 are synthetic_pair(h, w, channels, seed, amp, stereo)[:2] bit for bit."""
    canv, m = _canvas(h, w, channels, seed)
    u, v = synthetic_flow(h, w, amp, stereo)
    return np.ascontiguousarray(np.stack([_frame(canv, m, h, w, u, v, t) for t in range(n_frames)]))


def layered_stereo(h: int, w: int, channels: int = 1, seed: int = 0, d_bg: int = 8, d_fg: int = 24,
                   block=(0.3, 0.25, 0.7, 0.75)):
    """A two-layer stereo pair with real occlusions: a textured background at the integer disparity d_bg and, in front
    of it, a textured rectangle at the larger integer disparity d_fg covering the fractions `block` = (x0, y0, x1, y1)
    of the left view.  The right view shows at column xr the foreground point xr + d_fg where that lies in the
    rectangle, else the background point xr + d_bg (the library's convention I0(x) = I1(x - d(x)), stereo F = -d).
    Both layers are crops of independent canvases (_canvas), sampled at integer positions, so every visible point has
    exactly the same bytes in both views.  Returns (left_u8, right_u8, gt, occluded): gt the left view's positive
    disparity (h, w) float32, occluded (h, w) bool where the left pixel's match in the right view is hidden by the
    foreground or falls outside the frame."""
    assert 0 <= d_bg < d_fg
    bg, m = _canvas(h, w + d_fg, channels, seed)
    fg, _ = _canvas(h, w + d_fg, channels, seed + 1)
    X0, Y0, X1, Y1 = int(block[0] * w), int(block[1] * h), int(block[2] * w), int(block[3] * h)
    y, x = np.mgrid[0:h, 0:w]
    in_rows = (y >= Y0) & (y < Y1)
    in_fg = in_rows & (x >= X0) & (x < X1)
    left = np.where(in_fg[..., None], fg[m + y, m + x], bg[m + y, m + x])
    xf, xb = x + d_fg, x + d_bg  # the left-view columns that the right view's column x shows
    right_fg = in_rows & (xf >= X0) & (xf < X1)
    right = np.where(right_fg[..., None], fg[m + y, m + xf], bg[m + y, m + xb])
    gt = np.where(in_fg, d_fg, d_bg).astype(np.float32)
    xr = x - gt.astype(np.int64)
    hidden = ~in_fg & in_rows & (xr + d_fg >= X0) & (xr + d_fg < X1)
    occluded = (xr < 0) | hidden

    def q(img):
        img = np.clip(np.rint(img), 0, 255).astype(np.uint8)
        return np.ascontiguousarray(img[..., 0] if channels == 1 else img)

    return q(left), q(right), gt, occluded


def layered_scene_flow(h: int, w: int, channels: int = 1, seed: int = 0, d_bg: int = 8, d_fg=(24, 30), dx: int = 6,
                       block=(0.3, 0.25, 0.6, 0.75)):
    """Two stereo pairs, at t and t+1, of layered_stereo's scene in which the foreground rectangle moves: at t it covers
    the fractions `block` = (x0, y0, x1, y1) of the left view at the integer disparity d_fg[0]; at t+1 it has moved
    sideways by the integer dx pixels and has the disparity d_fg[1] (it came nearer or went away).  The background
    stays at d_bg.  Both layers are crops of independent canvases (_canvas) sampled at integer positions, the
    foreground's texture moving with it, so every visible point has exactly the same bytes in all four views.
    Returns (frames, gt): frames (4, h, w[, 3]) uint8, L_t, R_t, L_t+1, R_t+1; gt a dict of (h, w) arrays in frame-t
    coordinates: "disp0" the positive disparity at t, "disp1" that of the same point at t+1 (KITTI's disp_occ_1),
    "flow" (h, w, 2) the left view's flow, all float32; "occluded" bool where the point's match in R_t, L_t+1 or
    R_t+1 is hidden or outside the frame; and "disp_t1", L_t+1's own disparity map (frame-t+1 coordinates)."""
    assert 0 <= d_bg < min(d_fg)
    pad = max(d_fg) + abs(dx)
    bg, m = _canvas(h, w + pad, channels, seed)
    fg, _ = _canvas(h, w + pad, channels, seed + 1)
    X0, Y0, X1, Y1 = int(block[0] * w), int(block[1] * h), int(block[2] * w), int(block[3] * h)
    y, x = np.mgrid[0:h, 0:w]
    in_rows = (y >= Y0) & (y < Y1)
    wc = bg.shape[1]

    def col(c):
        return np.clip(m + c, 0, wc - 1)

    def view(shift, d_f):
        """The stereo pair with the rectangle moved by `shift`: left, right, the left view's disparity and where its
        match in the right view is hidden or outside, and the rectangle's pixels."""
        bx0, bx1 = X0 + shift, X1 + shift
        in_fg = in_rows & (x >= bx0) & (x < bx1)
        left = np.where(in_fg[..., None], fg[m + y, col(x - shift)], bg[m + y, col(x)])
        xf = x + d_f
        right_fg = in_rows & (xf >= bx0) & (xf < bx1)
        right = np.where(right_fg[..., None], fg[m + y, col(xf - shift)], bg[m + y, col(x + d_bg)])
        disp = np.where(in_fg, d_f, d_bg)
        xr = x - disp
        hidden = ~in_fg & in_rows & (xr + d_f >= bx0) & (xr + d_f < bx1)
        return left, right, disp, (xr < 0) | hidden, in_fg

    l0, r0, disp_t, occ0, fg0 = view(0, d_fg[0])
    l1, r1, disp_t1, occ1, fg1 = view(dx, d_fg[1])
    u = np.where(fg0, dx, 0)
    xt = x + u
    out = (xt < 0) | (xt > w - 1)
    xtc = np.clip(xt, 0, w - 1)
    covered = ~fg0 & fg1[y, xtc]  # a background point behind the rectangle at t+1
    occluded = occ0 | out | covered | occ1[y, xtc]

    def q(img):
        img = np.clip(np.rint(img), 0, 255).astype(np.uint8)
        return np.ascontiguousarray(img[..., 0] if channels == 1 else img)

    frames = np.stack([q(l0), q(r0), q(l1), q(r1)])
    gt = {"disp0": disp_t.astype(np.float32), "disp1": np.where(fg0, d_fg[1], d_bg).astype(np.float32),
          "flow": np.stack([u, np.zeros_like(u)], -1).astype(np.float32), "occluded": occluded,
          "disp_t1": disp_t1.astype(np.float32)}
    return frames, gt


def similarity_about_centre(h: int, w: int, angle_deg: float = 0.0, zoom: float = 1.0, shift=(0.0, 0.0)):
    """The 3 x 3 float64 map of pixel positions that rotates by angle_deg and scales by zoom about the frame's centre
    ((w-1)/2, (h-1)/2), then shifts by (dx, dy)."""
    c, s = zoom * np.cos(np.deg2rad(angle_deg)), zoom * np.sin(np.deg2rad(angle_deg))
    ox, oy = 0.5 * (w - 1), 0.5 * (h - 1)
    return np.array([[c, -s, ox - c * ox + s * oy + shift[0]], [s, c, oy - s * ox - c * oy + shift[1]], [0, 0, 1.0]])


def global_motion_clip(n: int, h: int, w: int, channels: int = 1, seed: int = 0, H=None,
                       block=(0.55, 0.3, 0.85, 0.8), block_motion=(-4.0, 2.5)):
    """A clip of n + 1 uint8 frames under one camera motion: frame t + 1 maps the pixel x of frame t to H x (H a 3 x 3
    map of pixel positions, default the identity), i.e. frame t is the canvas of _canvas sampled at H^-t x (cubic).  In
    front of it a textured rectangle of an independent canvas covers the fractions `block` = (x0, y0, x1, y1) of frame
    0 and moves on its own by the translation block_motion = (dx, dy) per frame.  Returns (frames, models, masks):
    frames (n + 1, h, w[, 3]), models (n, 3, 3) float64 (H for every pair) and masks (n, h, w) bool, the rectangle's
    pixels in frame t of pair t."""
    from scipy import ndimage

    H = np.eye(3) if H is None else np.asarray(H, np.float64)
    bg, m = _canvas(h, w, channels, seed)
    fg, _ = _canvas(h, w, channels, seed + 1)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    X0, Y0, X1, Y1 = block[0] * w, block[1] * h, block[2] * w, block[3] * h
    frames, masks = [], []
    Hinv = np.eye(3)
    Hi = np.linalg.inv(H)
    for t in range(n + 1):
        sx = Hinv[0, 0] * xx + Hinv[0, 1] * yy + Hinv[0, 2]
        sy = Hinv[1, 0] * xx + Hinv[1, 1] * yy + Hinv[1, 2]
        sw = Hinv[2, 0] * xx + Hinv[2, 1] * yy + Hinv[2, 2]
        bx, by = xx - t * block_motion[0], yy - t * block_motion[1]
        inside = (bx >= X0) & (bx < X1) & (by >= Y0) & (by < Y1)
        img = np.empty((h, w, channels))
        for c in range(channels):
            back = ndimage.map_coordinates(bg[..., c], [sy / sw + m, sx / sw + m], order=3, mode="nearest")
            front = ndimage.map_coordinates(fg[..., c], [by + m, bx + m], order=3, mode="nearest")
            img[..., c] = np.where(inside, front, back)
        q = np.clip(np.rint(img), 0, 255).astype(np.uint8)
        frames.append(q[..., 0] if channels == 1 else q)
        masks.append(inside)
        Hinv = Hinv @ Hi
    return np.ascontiguousarray(np.stack(frames)), np.repeat(H[None], n, 0), np.stack(masks[:n])


def shaky_clip(n: int, h: int, w: int, channels: int = 1, seed: int = 0, pan=(1.0, 0.0), jitter: float = 2.0):
    """A clip of n uint8 frames filmed by a camera that pans by `pan` = (dx, dy) pixels per frame and shakes at random
    about that path: frame t shows the canvas of _canvas through the pose C_t = J_t P_t, P_t the shift by t * pan and
    J_t a random rotation (up to jitter / 4 degrees) about the frame's centre plus a random shift of up to `jitter`
    pixels in x and y, i.e. frame t is the canvas sampled at C_t^-1 x (cubic).  Returns (frames, models, smooth):
    frames (n, h, w[, 3]), models (n - 1, 3, 3) float64, model t = C_{t+1} C_t^-1 mapping a pixel of frame t to its
    position in frame t + 1, and smooth (n, 3, 3) the corrections P_t C_t^-1 = J_t^-1 that move frame t onto the
    shake-free path."""
    from scipy import ndimage

    rng = np.random.default_rng(seed + 7)
    bg, m = _canvas(h, w, channels, seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    poses, frames = [], []
    for t in range(n):
        J = similarity_about_centre(h, w, rng.uniform(-0.25, 0.25) * jitter, 1.0,
                                    (rng.uniform(-1, 1) * jitter, rng.uniform(-1, 1) * jitter))
        P = np.array([[1.0, 0.0, t * pan[0]], [0.0, 1.0, t * pan[1]], [0.0, 0.0, 1.0]])
        C = J @ P
        Ci = np.linalg.inv(C)
        sx = Ci[0, 0] * xx + Ci[0, 1] * yy + Ci[0, 2]
        sy = Ci[1, 0] * xx + Ci[1, 1] * yy + Ci[1, 2]
        img = np.empty((h, w, channels))
        for c in range(channels):
            img[..., c] = ndimage.map_coordinates(bg[..., c], [sy + m, sx + m], order=3, mode="nearest")
        q = np.clip(np.rint(img), 0, 255).astype(np.uint8)
        frames.append(q[..., 0] if channels == 1 else q)
        poses.append((C, J))
    models = np.stack([poses[t + 1][0] @ np.linalg.inv(poses[t][0]) for t in range(n - 1)])
    smooth = np.stack([np.linalg.inv(J) for _, J in poses])
    return np.ascontiguousarray(np.stack(frames)), models, smooth


def axis_angle(w) -> np.ndarray:
    """The rotation matrix (3, 3) float64 of the rotation vector w (radians, Rodrigues' formula)."""
    w = np.asarray(w, np.float64)
    th = float(np.linalg.norm(w))
    if th == 0.0:
        return np.eye(3)
    k = w / th
    K = np.array([[0.0, -k[2], k[1]], [k[2], 0.0, -k[0]], [-k[1], k[0], 0.0]])
    return np.eye(3) + np.sin(th) * K + (1.0 - np.cos(th)) * (K @ K)


def _value_noise(table: np.ndarray, u: np.ndarray, v: np.ndarray) -> np.ndarray:
    """Bilinear value noise of a periodic random table at lattice coordinates (u, v)."""
    n = table.shape[0]
    u0, v0 = np.floor(u), np.floor(v)
    fu, fv = u - u0, v - v0
    i0, j0 = u0.astype(np.int64) % n, v0.astype(np.int64) % n
    i1, j1 = (i0 + 1) % n, (j0 + 1) % n
    return ((table[j0, i0] * (1 - fu) + table[j0, i1] * fu) * (1 - fv) +
            (table[j1, i0] * (1 - fu) + table[j1, i1] * fu) * fv)


def rigid_stereo_clip(n: int, h: int, w: int, channels: int, seed: int, camera, motions, block=None):
    """A stereo clip of a piecewise-planar textured scene seen by a moving rig: a ground plane 1.65 m below the first
    camera and a back wall 40 m ahead, plus a box on the ground that moves on its own between frames.  camera: a
    mapping with fx, fy, cx, cy, baseline, doffs; motions: n relative poses (3, 4) (or (R, t) pairs), each mapping a
    point in camera-t coordinates to camera-t+1 coordinates.  block: None for the default box, or a mapping with
    "centre" (world, metres, at frame 0), "half" (half sizes) and "velocity" (metres per frame).
    Returns a dict: "left", "right" (n+1, h, w[, channels]) uint8 frames; "disp" (n+1, h, w) float32, the analytic
    left disparity fb / Z - doffs of every frame; "flow" (n, h, w, 2) float32, the exact flow of every pair (a pixel's
    surface point carried by the rig's motion, or by the box's); "poses" (n, 3, 4) float64, the true relative poses;
    "abs" (n+1, 3, 4) camera-to-world poses; "box" (n, h, w) bool, the box's pixels in frame t."""
    rng = np.random.default_rng(seed)
    tables = [rng.uniform(0, 1, (256, 256)) for _ in range(3 * channels)]
    fx, fy, cx, cy = (float(camera[k]) for k in ("fx", "fy", "cx", "cy"))
    base, doffs = float(camera["baseline"]), float(camera["doffs"])
    fb = float(np.float32(np.float32(fx) * np.float32(base)))
    blk = {"centre": (-1.2, 0.85, 9.0), "half": (0.9, 0.8, 0.9), "velocity": (0.25, 0.0, -0.15)}
    blk.update(block or {})
    bc0, bh, bv = (np.asarray(blk[k], np.float64) for k in ("centre", "half", "velocity"))
    ground, wall = 1.65, 40.0
    rel = []
    for mo in motions:
        if isinstance(mo, (tuple, list)) and len(mo) == 2:
            P = np.concatenate([np.asarray(mo[0], np.float64), np.asarray(mo[1], np.float64).reshape(3, 1)], 1)
        else:
            P = np.asarray(mo, np.float64).reshape(3, 4)
        rel.append(P)
    assert len(rel) == n
    T = [np.eye(4)]
    for P in rel:
        M = np.eye(4)
        M[:3] = P
        T.append(T[-1] @ np.linalg.inv(M))
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    dcam = np.stack([(x - cx) / fx, (y - cy) / fy, np.ones_like(x)], -1)

    def cast(Tk, k, right):
        Rc, tc = Tk[:3, :3], Tk[:3, 3]
        d = dcam @ Rc.T
        o = tc + (Rc @ np.array([base, 0.0, 0.0]) if right else 0.0)
        inf = np.full((h, w), np.inf)
        with np.errstate(divide="ignore", invalid="ignore"):
            tg = np.where(d[..., 1] > 0, (ground - o[1]) / d[..., 1], inf)
            tw = np.where(d[..., 2] > 0, (wall - o[2]) / d[..., 2], inf)
            lo, hi = bc0 + k * bv - bh, bc0 + k * bv + bh
            t0 = (lo - o) / d
            t1 = (hi - o) / d
            tmin = np.max(np.minimum(t0, t1), -1)
            tmax = np.min(np.maximum(t0, t1), -1)
        tb = np.where((tmax >= tmin) & (tmin > 0), tmin, inf)
        t = np.minimum(np.minimum(tg, tw), tb)
        p = o + d * t[..., None]
        return t, p, tb <= np.minimum(tg, tw), tg <= tw

    def shade(p, isbox, isground, k):
        loc = p - (bc0 + k * bv)
        su = np.where(isbox, loc[..., 0] + 0.7 * loc[..., 2], p[..., 0])
        sv = np.where(isbox, loc[..., 1] + 0.3 * loc[..., 2], np.where(isground, p[..., 2], p[..., 1]))
        img = np.zeros((h, w, channels))
        for c in range(channels):
            acc = 0.0
            for o, scale in enumerate((0.04, 0.15, 0.6)):
                acc = acc + (0.5 ** o) * _value_noise(tables[3 * c + o], su / scale, sv / scale)
            img[..., c] = 30.0 + 190.0 * acc / 1.75 + np.where(isbox, 20.0, 0.0)
        img = np.clip(np.round(img), 0, 255).astype(np.uint8)
        return img if channels > 1 else img[..., 0]

    left, right, disp, pts, boxes = [], [], [], [], []
    for k in range(n + 1):
        t, p, isbox, isground = cast(T[k], k, False)
        left.append(shade(p, isbox, isground, k))
        tr, pr, isbox_r, isground_r = cast(T[k], k, True)
        right.append(shade(pr, isbox_r, isground_r, k))
        disp.append((fb / t - doffs).astype(np.float32))
        pts.append(p)
        boxes.append(isbox)
    flows = []
    for k in range(n):
        p = pts[k] + np.where(boxes[k][..., None], bv, 0.0)
        Ti = np.linalg.inv(T[k + 1])
        q = p @ Ti[:3, :3].T + Ti[:3, 3]
        flows.append(np.stack([fx * q[..., 0] / q[..., 2] + cx - x, fy * q[..., 1] / q[..., 2] + cy - y], -1))
    return {"left": np.stack(left), "right": np.stack(right), "disp": np.stack(disp),
            "flow": np.stack(flows).astype(np.float32) if n else np.zeros((0, h, w, 2), np.float32),
            "poses": np.stack(rel) if n else np.zeros((0, 3, 4)), "abs": np.stack([Tk[:3] for Tk in T]),
            "box": np.stack(boxes[:n]) if n else np.zeros((0, h, w), bool)}
