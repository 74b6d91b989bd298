"""Host-side pre/post-processing around the hot path (numpy).

This is the arithmetic of run_dense.cpp:298-344 (pad to
2^lv_f, float conversion, x0.5 pyramid, Sobel/8 gradients, border padding) and
run_dense.cpp:407-414 (x2^lv_l upsampling, crop).  It is OUTSIDE the hot path
(SURVEY.md section 8f rank 1-2): the hot path's input is the padded pyramid.

For 8-bit input images every value of every pyramid level is a dyadic rational
that float32 holds exactly (8 integer bits + 2 fraction bits per level), so the
box mean and the Sobel/8 sums below are exact and therefore bit-identical to
OpenCV's evaluation order; tests/test_preprocess.py checks that against cv2
when it is importable.
"""
from __future__ import annotations

import functools
import math

import numpy as np


def pad_to_multiple(img: np.ndarray, lv_f: int, div_level: int | None = None):
    """run_dense.cpp:299-311: replicate-pad so width, height are divisible by 2^div_level (default lv_f; lv_f + 1 for
    a run with an init flow, run_dense.cpp:301).  Returns (padded, padw, padh)."""
    scfct = 2 ** (lv_f if div_level is None else div_level)
    h, w = img.shape[:2]
    padw = (scfct - w % scfct) % scfct
    padh = (scfct - h % scfct) % scfct
    if padw or padh:
        t, b = int(math.floor(padh / 2.0)), int(math.ceil(padh / 2.0))
        l, r = int(math.floor(padw / 2.0)), int(math.ceil(padw / 2.0))
        pads = ((t, b), (l, r)) + (((0, 0),) if img.ndim == 3 else ())
        img = np.pad(img, pads, mode="edge")
    return img, padw, padh


def half_size(img: np.ndarray) -> np.ndarray:
    """cv::resize(.5,.5,INTER_LINEAR) on even-sized float32 images == 2x2 box mean
    (run_dense.cpp:150)."""
    a = img[0::2, 0::2]
    b = img[0::2, 1::2]
    c = img[1::2, 0::2]
    d = img[1::2, 1::2]
    return (((a + b) + (c + d)) * np.float32(0.25)).astype(np.float32)


def sobel8(img: np.ndarray):
    """cv::Sobel(CV_32F, 3x3, scale 1/8, BORDER_DEFAULT=reflect101), run_dense.cpp:156-157.
    Returns (dx, dy)."""
    pads = ((1, 1), (1, 1)) + (((0, 0),) if img.ndim == 3 else ())
    p = np.pad(img, pads, mode="reflect")
    # dx: row filter [-1 0 1], column filter [1 2 1]/8
    t = p[:, 2:] - p[:, :-2]
    dx = (t[:-2] * np.float32(0.125) + t[1:-1] * np.float32(0.25)) + t[2:] * np.float32(0.125)
    # dy: row filter [1 2 1]/8 ... applied as column [-1 0 1] of the row-smoothed image
    s = (p[:, :-2] * np.float32(0.125) + p[:, 1:-1] * np.float32(0.25)) + p[:, 2:] * np.float32(0.125)
    dy = s[2:] - s[:-2]
    return dx.astype(np.float32), dy.astype(np.float32)


def build_pyramid(img_f32: np.ndarray, lv_f: int, imgpadding: int):
    """ConstructImgPyramide (run_dense.cpp:130-178): returns three lists indexed by
    level 0..lv_f of C-contiguous float32 arrays padded by `imgpadding` on all
    sides (image: replicate, gradients: zero)."""
    imgs, dxs, dys = [], [], []
    cur = np.ascontiguousarray(img_f32, dtype=np.float32)
    for i in range(lv_f + 1):
        if i > 0:
            cur = half_size(cur)
        dx, dy = sobel8(cur)
        pads = ((imgpadding, imgpadding), (imgpadding, imgpadding)) + (((0, 0),) if cur.ndim == 3 else ())
        imgs.append(np.ascontiguousarray(np.pad(cur, pads, mode="edge")))
        dxs.append(np.ascontiguousarray(np.pad(dx, pads, mode="constant")))
        dys.append(np.ascontiguousarray(np.pad(dy, pads, mode="constant")))
    return imgs, dxs, dys


class PairPyramids:
    """Everything OFClass's constructor takes for one image pair (oflow.h:84-111)."""

    def __init__(self, img0_u8: np.ndarray, img1_u8: np.ndarray, lv_f: int, imgpadding: int,
                 div_level: int | None = None):
        """div_level: the frames are padded to multiples of 2^div_level (default lv_f; lv_f + 1 for a run with an
        init flow, run_dense.cpp:301)."""
        assert img0_u8.shape == img1_u8.shape
        self.height_org, self.width_org = img0_u8.shape[:2]
        a, self.padw, self.padh = pad_to_multiple(img0_u8, lv_f, div_level)
        b, _, _ = pad_to_multiple(img1_u8, lv_f, div_level)
        self.height, self.width = a.shape[:2]
        self.noc = 1 if a.ndim == 2 else a.shape[2]
        self.lv_f = lv_f
        self.imgpadding = imgpadding
        self.i0, self.i0x, self.i0y = build_pyramid(a.astype(np.float32), lv_f, imgpadding)
        self.i1, self.i1x, self.i1y = build_pyramid(b.astype(np.float32), lv_f, imgpadding)

    def level_shape(self, lv: int):
        return self.height >> lv, self.width >> lv


def initflow_from_fullres(flow: np.ndarray, lv_f: int) -> np.ndarray:
    """The reference's disabled init-flow input (run_dense.cpp:355-378): a flow of the original frame size
    ((h, w, nop) or (h, w)) -> the `initflow` of OFClass, level lv_f + 1, (h', w', nop) float32.

    Replicate padding to multiples of s = 2^(lv_f+1) (floor(pad/2) left/top), every value times 2^-(lv_f+1) (exact),
    then cv::resize(INTER_AREA) by the integer factor s.  That is OpenCV's area-fast path, whose order is restated
    here: sum = 0, then for the s^2 terms of the block in row-major order, groups of four add as
    sum += ((t0 + t1) + t2) + t3, and the result is sum * (1/s^2) -- the 0 start turns a block that sums to -0 into
    +0.  For s = 2 with one channel OpenCV's SIMD body computes ((a + b) + (c + d)) * 0.25 instead, while its scalar
    tail (the last destination columns, depending on the build's SIMD width) keeps the order above; this
    restatement, and the device, use the SIMD body's formula for every column."""
    fl = np.asarray(flow, np.float32)
    if fl.ndim == 2:
        fl = fl[..., None]
    s = 2 ** (lv_f + 1)
    v, _, _ = pad_to_multiple(fl, lv_f + 1)
    v = v * np.float32(2.0 ** -(lv_f + 1))
    H, W, nop = v.shape[0] // s, v.shape[1] // s, v.shape[2]
    t = v.reshape(H, s, W, s, nop).transpose(0, 2, 1, 3, 4).reshape(H, W, s * s, nop)  # row-major block terms
    if s == 2 and nop == 1:
        return ((((t[:, :, 0] + t[:, :, 1]) + (t[:, :, 2] + t[:, :, 3])) * np.float32(0.25))).astype(np.float32)
    g = t.reshape(H, W, s * s // 4, 4, nop)
    part = ((g[:, :, :, 0] + g[:, :, :, 1]) + g[:, :, :, 2]) + g[:, :, :, 3]
    acc = np.zeros((H, W, nop), np.float32)
    for i in range(part.shape[2]):
        acc = acc + part[:, :, i]
    return (acc * np.float32(1.0 / (s * s))).astype(np.float32)


def upsample_linear(flow: np.ndarray, s: int) -> np.ndarray:
    """cv::resize(fx=fy=s, INTER_LINEAR) for integer s: src = (dst+.5)/s-.5, edge clamped
    (run_dense.cpp:410)."""
    h, w = flow.shape[:2]

    def taps(n_src, n_dst):
        x = (np.arange(n_dst, dtype=np.float32) + np.float32(0.5)) / np.float32(s) - np.float32(0.5)
        x0 = np.floor(x).astype(np.int64)
        f = (x - x0).astype(np.float32)
        f[x0 < 0] = 0
        i0 = np.clip(x0, 0, n_src - 1)
        i1 = np.clip(x0 + 1, 0, n_src - 1)
        return i0, i1, f

    x0, x1, fx = taps(w, w * s)
    y0, y1, fy = taps(h, h * s)
    fl = flow.reshape(h, w, -1)
    fxb = fx[None, :, None]
    fyb = fy[:, None, None]
    rows = fl[:, x0] * (np.float32(1) - fxb) + fl[:, x1] * fxb
    out = rows[y0] * (np.float32(1) - fyb) + rows[y1] * fyb
    return out.astype(np.float32).reshape((h * s, w * s) + flow.shape[2:])


def postprocess(flow_level: np.ndarray, lv_l: int, padw: int, padh: int, width_org: int, height_org: int):
    """run_dense.cpp:407-414: scale by 2^lv_l, upsample, crop the divisibility padding."""
    out = flow_level
    if lv_l != 0:
        sc = 2 ** lv_l
        out = upsample_linear(out * np.float32(sc), sc)
    x0, y0 = int(math.floor(padw / 2.0)), int(math.floor(padh / 2.0))
    return np.ascontiguousarray(out[y0:y0 + height_org, x0:x0 + width_org])


def consistency_check(fw: np.ndarray, bw: np.ndarray, alpha: float, beta: float):
    """Forward-backward (flow) / left-right (stereo) consistency (Sundaram, Brox, Keutzer, ECCV 2010) of the
    full-resolution flow `fw` against its partner `bw`, both (h, w, nop) or (h, w) float32; the restatement of
    ofdis_consistency_fullres, float32 throughout, evaluated in this order without contraction:

        (xs, ys) = (x, y) + F(x, y)                    (stereo: ys = y)
        outside [0, w-1] x [0, h-1], or NaN:  mask 2, err +inf
        x0 = floor(xs), x1 = min(x0 + 1, w - 1), fx = xs - x0 (and y); b = bilinear B at (xs, ys), rows first:
            r0 = B(x0,y0) (1-fx) + B(x1,y0) fx,  r1 = B(x0,y1) (1-fx) + B(x1,y1) fx,  b = r0 (1-fy) + r1 fy
        err = du^2 + dv^2 with (du, dv) = F + b;  mag = (u^2 + v^2) + (b0^2 + b1^2)
        mask = 0 if err <= alpha mag + beta else 1

    Returns (mask uint8 (h, w), err float32 (h, w))."""
    f32 = np.float32
    F = np.asarray(fw, f32)
    B = np.asarray(bw, f32)
    F = F.reshape(F.shape[:2] + (-1,))
    B = B.reshape(B.shape[:2] + (-1,))
    h, w, nop = F.shape
    assert B.shape == F.shape
    u = F[..., 0]
    v = F[..., 1] if nop == 2 else np.zeros_like(u)
    with np.errstate(invalid="ignore", over="ignore"):
        xs = np.arange(w, dtype=f32)[None, :] + u
        ys = np.arange(h, dtype=f32)[:, None] + v
        inside = (xs >= 0) & (xs <= f32(w - 1)) & (ys >= 0) & (ys <= f32(h - 1))
        xc = np.where(inside, xs, f32(0))
        yc = np.where(inside, ys, f32(0))
        x0 = np.floor(xc).astype(np.int64)
        y0 = np.floor(yc).astype(np.int64)
        x1 = np.minimum(x0 + 1, w - 1)
        y1 = np.minimum(y0 + 1, h - 1)
        fx = (xc - x0.astype(f32)).astype(f32)
        fy = (yc - y0.astype(f32)).astype(f32)
        gx, gy = f32(1) - fx, f32(1) - fy
        b = []
        for c in range(nop):
            Bc = B[..., c]
            r0 = Bc[y0, x0] * gx + Bc[y0, x1] * fx
            r1 = Bc[y1, x0] * gx + Bc[y1, x1] * fx
            b.append(r0 * gy + r1 * fy)
        b0 = b[0]
        b1 = b[1] if nop == 2 else np.zeros_like(u)
        du = u + b0
        dv = v + b1 if nop == 2 else np.zeros_like(u)
        err = du * du + dv * dv
        mag = (u * u + v * v) + (b0 * b0 + b1 * b1)
        mask = np.where(err <= f32(alpha) * mag + f32(beta), 0, 1).astype(np.uint8)
    mask[~inside] = 2
    err = np.where(inside, err, f32(np.inf)).astype(f32)
    return mask, err


UNKNOWN_FLOW_THRESH = 1e9  # Middlebury's flow-io: a ground-truth component above this (or NaN) is unknown
_QNAN = np.uint32(0x7FC00000).view(np.float32)


def flow_error(flow: np.ndarray, gt: np.ndarray, classes: np.ndarray | None = None, nclasses: int = 1):
    """End-point error of full-resolution flows against ground truth, per pixel and per class; the restatement of
    ofdis_flow_error_fullres, float32 without contraction:

        known      flow: G_u, G_v not NaN and |G_u|, |G_v| <= 1e9;  stereo: G not NaN and |G| <= 1e9
        e, g       flow: e = sqrt(du^2 + dv^2) with (du, dv) = F - G, g = sqrt(G_u^2 + G_v^2);  stereo: |F - G|, |G|
        map        e where known, else the quiet NaN 0x7fc00000
        counted    for class c: known and classes == c (classes None: every pixel is class 0), c < nclasses
        counts     n, e > 1, e > 3, e > 5, outliers e > 3 and e > 0.05 g
        sum_err    per row a float64 sum from +0.0 adds (double) e of the row's counted pixels with x ascending (+0.0
                   for the others); the total from +0.0 adds the row sums with y ascending

    flow and gt: one pair (h, w, nop) or (h, w) (stereo), or a batch (n, h, w, nop); classes uint8 of the same shape
    without nop.  Returns (stats, err): stats of api.ERROR_STATS_DTYPE, (nclasses,) for one pair or (n, nclasses) for a
    batch, and the float32 map (h, w) or (n, h, w)."""
    from .api import ERROR_STATS_DTYPE

    f32 = np.float32
    F = np.asarray(flow, f32)
    G = np.asarray(gt, f32)
    assert F.shape == G.shape, (F.shape, G.shape)
    single = F.ndim in (2, 3)
    if F.ndim == 2:
        F, G = F[..., None], G[..., None]
    if single:
        F, G = F[None], G[None]
    n, h, w, nop = F.shape
    assert nop in (1, 2) and 1 <= nclasses
    cls = np.zeros((n, h, w), np.uint8) if classes is None else np.asarray(classes, np.uint8).reshape(n, h, w)
    assert classes is not None or nclasses == 1
    with np.errstate(invalid="ignore", over="ignore"):
        lim = f32(UNKNOWN_FLOW_THRESH)
        if nop == 2:
            known = (np.abs(G[..., 0]) <= lim) & (np.abs(G[..., 1]) <= lim)
            du, dv = F[..., 0] - G[..., 0], F[..., 1] - G[..., 1]
            e = np.sqrt(du * du + dv * dv)
            g = np.sqrt(G[..., 0] * G[..., 0] + G[..., 1] * G[..., 1])
        else:
            known = np.abs(G[..., 0]) <= lim
            e = np.abs(F[..., 0] - G[..., 0])
            g = np.abs(G[..., 0])
        tests = (e > f32(1), e > f32(3), e > f32(5), (e > f32(3)) & (e > f32(0.05) * g))
    err = np.where(known, e, _QNAN).astype(f32)
    stats = np.zeros((n, nclasses), ERROR_STATS_DTYPE)
    for p in range(n):
        for c in range(nclasses):
            counted = known[p] & (cls[p] == c)
            st = stats[p, c]
            st["n"] = int(counted.sum())
            st["n_over"] = [int((counted & t[p]).sum()) for t in tests[:3]]
            st["n_outlier"] = int((counted & tests[3][p]).sum())
            terms = np.where(counted, e[p].astype(np.float64), 0.0)
            rows = np.zeros(h, np.float64)
            for x in range(w):  # x ascending, every row at once
                rows = rows + terms[:, x]
            total = 0.0
            for y in range(h):
                total += float(rows[y])
            st["sum_err"] = total
    if single:
        return stats[0], err[0]
    return stats, err


def write_pgm(path: str, img: np.ndarray) -> None:
    """Binary PGM (P5), maxval 255: an (h, w) uint8 image, rows top-down."""
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape[:2]
    with open(path, "wb") as f:
        f.write(b"P5\n%d %d\n255\n" % (w, h))
        f.write(img.reshape(h, w).tobytes())


def write_flo(path: str, flow: np.ndarray) -> None:
    """SaveFlowFile (run_dense.cpp:16-57): 'PIEH', int32 w, int32 h, float32 row-major."""
    h, w = flow.shape[:2]
    with open(path, "wb") as f:
        f.write(b"PIEH")
        np.array([w, h], dtype="<i4").tofile(f)
        np.ascontiguousarray(flow, dtype="<f4").tofile(f)


def read_flo(path: str) -> np.ndarray:
    with open(path, "rb") as f:
        tag = f.read(4)
        if tag != b"PIEH":
            raise ValueError("not a .flo file")
        w, h = np.fromfile(f, dtype="<i4", count=2)
        data = np.fromfile(f, dtype="<f4")
    return data.reshape(h, w, -1)


def write_pfm(path: str, disp: np.ndarray) -> None:
    """SavePFMFile (run_dense.cpp:60-81): 'Pf', scale -1 (little endian), rows bottom-up, negated."""
    h, w = disp.shape[:2]
    with open(path, "wb") as f:
        f.write(("Pf\n%d %d\n%f\n" % (w, h, -1.0)).encode())
        np.ascontiguousarray(-disp.reshape(h, w)[::-1], dtype="<f4").tofile(f)


def read_pfm(path: str) -> np.ndarray:
    """The exact inverse of write_pfm: (h, w, 1) float32 (rows top-down, values negated back)."""
    with open(path, "rb") as f:
        data = f.read()
    parts = data.split(b"\n", 3)
    if len(parts) != 4 or parts[0] != b"Pf":
        raise ValueError("not a one-channel .pfm file")
    w, h = (int(x) for x in parts[1].split())
    if float(parts[2]) >= 0:
        raise ValueError("big-endian .pfm (scale >= 0) is not what SavePFMFile writes")
    body = np.frombuffer(parts[3], dtype="<f4")
    if body.size != w * h or len(parts[3]) != 4 * w * h:
        raise ValueError("truncated .pfm file")
    return np.ascontiguousarray(-body.reshape(h, w)[::-1]).astype(np.float32).reshape(h, w, 1)


# ---- encoded flows (ofdis_get_flow_fullres_encoded) and KITTI's 16-bit PNGs ------------------------------------------
F16_NAN = 0x7E00  # the one NaN of the binary16 encoding: numpy's astype(float16) of the quiet NaN 0x7fc00000


def encode_f16(flow: np.ndarray) -> np.ndarray:
    """OFDIS_ENC_F16: every value rounded to the nearest binary16, ties to even (magnitudes of 65520 and more become
    +-inf); every NaN, whatever its sign and payload, becomes 0x7e00.  Returns float16 of the same shape."""
    F = np.asarray(flow, np.float32)
    with np.errstate(over="ignore"):
        h = F.astype(np.float16).view(np.uint16)
    return np.where(np.isnan(F), np.uint16(F16_NAN), h).astype(np.uint16).view(np.float16)


def encode_kitti(flow: np.ndarray, swapped: bool = False) -> np.ndarray:
    """OFDIS_ENC_KITTI in float32 without contraction.  flow: (..., 2) or stereo (..., 1), in this library's
    convention (what get_flow_fullres returns).
        flow    (..., 3) uint16 (R, G, B): where u and v are not NaN,
                (clamp(u * 64 + 32768, 0, 65535), the same of v, 1) truncated to uint16, else (0, 0, 0)
        stereo  (...) uint16: d = -F (F when `swapped`, the right view of a swapped slot); where d >= 0 (NaN fails,
                -0 passes) clamp(d * 256, 1, 65535) truncated to uint16, else 0"""
    f32 = np.float32
    F = np.asarray(flow, f32)
    assert F.shape[-1] in (1, 2), F.shape
    if F.shape[-1] == 2:
        u, v = F[..., 0], F[..., 1]
        valid = ~np.isnan(u) & ~np.isnan(v)
        out = np.zeros(F.shape[:-1] + (3,), np.uint16)
        with np.errstate(over="ignore", invalid="ignore"):
            for c, x in enumerate((u, v)):
                q = np.fmin(np.fmax(np.where(valid, x, f32(0)) * f32(64) + f32(32768), f32(0)), f32(65535))
                out[..., c] = np.where(valid, q, f32(0)).astype(np.uint16)
        out[..., 2] = valid
        return out
    d = F[..., 0] if swapped else -F[..., 0]
    with np.errstate(invalid="ignore"):
        valid = d >= f32(0)
    with np.errstate(over="ignore"):
        q = np.fmin(np.fmax(np.where(valid, d, f32(0)) * f32(256), f32(1)), f32(65535))
    return np.where(valid, q, f32(0)).astype(np.uint16)


def kitti_to_flow(enc: np.ndarray, nop: int) -> np.ndarray:
    """A KITTI 16-bit array in this library's convention, float32, NaN where it is invalid (flow_error treats NaN
    ground truth as unknown).  Flow (nop 2): (..., 3) -> (..., 2), (R - 32768.0f) / 64.0f, valid where B > 0.
    Stereo (nop 1): (...) -> (..., 1), -(val / 256.0f), the sign get_flow_fullres and .pfm use, valid where val > 0."""
    f32 = np.float32
    E = np.asarray(enc, np.uint16)
    if nop == 2:
        assert E.shape[-1] == 3, E.shape
        F = (E[..., :2].astype(f32) - f32(32768)) / f32(64)
        F[E[..., 2] == 0] = np.nan
        return F
    F = -(E.astype(f32) / f32(256))
    F[E == 0] = np.nan
    return F[..., None]


_PNG_SIG = b"\x89PNG\r\n\x1a\n"


def write_kitti_png(path: str, enc: np.ndarray) -> None:
    """KITTI's 16-bit PNG: (h, w, 3) uint16 as colour type 2 (flow), (h, w) as colour type 0 (stereo); big-endian
    samples, non-interlaced, every row filter 0."""
    import struct
    import zlib

    E = np.asarray(enc)
    assert E.dtype == np.uint16 and (E.ndim == 2 or (E.ndim == 3 and E.shape[2] == 3)), (E.dtype, E.shape)
    h, w = E.shape[:2]
    rows = np.ascontiguousarray(E, ">u2").reshape(h, -1).view(np.uint8)
    raw = np.concatenate([np.zeros((h, 1), np.uint8), rows], axis=1).tobytes()

    def chunk(t, d):
        return struct.pack(">I", len(d)) + t + d + struct.pack(">I", zlib.crc32(t + d) & 0xFFFFFFFF)

    with open(path, "wb") as f:
        f.write(_PNG_SIG + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 16, 2 if E.ndim == 3 else 0, 0, 0, 0)))
        f.write(chunk(b"IDAT", zlib.compress(raw, 1)) + chunk(b"IEND", b""))


def _unfilter(ft: int, line: np.ndarray, up: np.ndarray, bpp: int) -> np.ndarray:
    """One PNG row of filter type ft (0 None, 1 Sub, 2 Up, 3 Average, 4 Paeth), with `bpp` bytes per pixel."""
    if ft == 0:
        return line
    if ft == 2:
        return (line.astype(np.uint16) + up).astype(np.uint8)
    if ft == 1:  # out[x] = in[x] + out[x - bpp]: running sums mod 256 per byte position of a pixel
        return (np.cumsum(line.reshape(-1, bpp).astype(np.int64), axis=0) % 256).astype(np.uint8).reshape(-1)
    out = bytearray(line.tobytes())
    prior = up.tobytes()
    for x in range(len(out)):
        a = out[x - bpp] if x >= bpp else 0
        b = prior[x]
        if ft == 3:
            pred = (a + b) >> 1
        elif ft == 4:
            c = prior[x - bpp] if x >= bpp else 0
            p = a + b - c
            pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
            pred = a if (pa <= pb and pa <= pc) else (b if pb <= pc else c)
        else:
            raise ValueError("PNG filter type %d" % ft)
        out[x] = (out[x] + pred) & 0xFF
    return np.frombuffer(bytes(out), np.uint8)


def read_kitti_png(path: str) -> np.ndarray:
    """The 16-bit PNGs of write_kitti_png, from any writer: (h, w, 3) uint16 for colour type 2, (h, w) for colour type
    0.  Bit depth 16 and no interlacing are required; every row may use any of the five filter types."""
    import struct
    import zlib

    with open(path, "rb") as f:
        b = f.read()
    if b[:8] != _PNG_SIG:
        raise ValueError("%s: not a PNG file" % path)
    pos, idat, hdr = 8, [], None
    while pos + 8 <= len(b):
        n, t = struct.unpack(">I", b[pos:pos + 4])[0], b[pos + 4:pos + 8]
        data = b[pos + 8:pos + 8 + n]
        if t == b"IHDR":
            hdr = struct.unpack(">IIBBBBB", data[:13])
        elif t == b"IDAT":
            idat.append(data)
        elif t == b"IEND":
            break
        pos += 12 + n
    if hdr is None:
        raise ValueError("%s: no IHDR" % path)
    w, h, depth, ctype, _, _, interlace = hdr
    if depth != 16 or ctype not in (0, 2) or interlace != 0:
        raise ValueError("%s: not a 16-bit non-interlaced gray or RGB PNG" % path)
    ch = 3 if ctype == 2 else 1
    stride = w * ch * 2
    raw = np.frombuffer(zlib.decompress(b"".join(idat)), np.uint8)
    if raw.size != h * (stride + 1):
        raise ValueError("%s: image data of the wrong length" % path)
    raw = raw.reshape(h, stride + 1)
    img = np.zeros((h, stride), np.uint8)
    up = np.zeros(stride, np.uint8)
    for y in range(h):
        img[y] = _unfilter(int(raw[y, 0]), raw[y, 1:], up, 2 * ch)
        up = img[y]
    out = img.view(">u2").astype(np.uint16)
    return out.reshape(h, w, 3) if ch == 3 else out.reshape(h, w)


# ---- color-coded flows (ofdis_flow_color_fullres) -------------------------------------------------------------------
PI_F = np.float32(np.pi)
# the odd polynomial of atan2_f32: atan(t) ~ t * (C0 + s * (C1 + ... + s * C7)), s = t * t, fitted on [0, 1]
ATAN_C = np.array([0.99999934, -0.3332986, 0.19946565, -0.13908629, 0.09642195, -0.055912293, 0.021862935,
                   -0.0040545613], np.float32)
COLOR_UNKNOWN_THRESH = np.float32(1e9)  # |u|, |v| (flow) or d (stereo) above this, or NaN, is not colored


def make_color_wheel() -> np.ndarray:
    """Middlebury's makecolorwheel: 55 (R, G, B) int entries, integer division; segments RY 15, YG 6, GC 4, CB 11,
    BM 13, MR 6."""
    w = []
    for i in range(15):
        w.append((255, 255 * i // 15, 0))
    for i in range(6):
        w.append((255 - 255 * i // 6, 255, 0))
    for i in range(4):
        w.append((0, 255, 255 * i // 4))
    for i in range(11):
        w.append((0, 255 - 255 * i // 11, 255))
    for i in range(13):
        w.append((255 * i // 13, 0, 255))
    for i in range(6):
        w.append((255, 0, 255 - 255 * i // 6))
    return np.array(w, np.int32)


COLOR_WHEEL = make_color_wheel()
# KITTI's stereo devkit (disp_to_color): (R, G, B, bin width in 1/1000 of the scale)
DISP_COLOR_MAP = np.array([[0, 0, 0, 114], [0, 0, 1, 185], [1, 0, 0, 114], [1, 0, 1, 174], [0, 1, 0, 114],
                           [0, 1, 1, 185], [1, 1, 0, 114], [1, 1, 1, 0]], np.int32)


def disp_color_bins():
    """(wt[0..6], cum[0..7]) in float32: wt[i] = 1000.0f / M[i][3], cum[i+1] = cum[i] + M[i][3] / 1000.0f in order."""
    f32 = np.float32
    wt = np.array([f32(1000) / f32(DISP_COLOR_MAP[i, 3]) for i in range(7)], f32)
    cum = [f32(0)]
    for i in range(7):
        cum.append(f32(cum[i] + f32(DISP_COLOR_MAP[i, 3]) / f32(1000)))
    return wt, np.array(cum, f32)


def atan2_f32(y, x) -> np.ndarray:
    """The library's float32 atan2, the same expressions as the device's: t = min(|x|, |y|) / max(|x|, |y|) (0 where
    both are 0), p = t * poly(t * t) by Horner with ATAN_C, then pi/2 - p where |y| > |x|, pi - p where x's sign bit
    is set, and y's sign.  Within 1e-6 of float64 arctan2, in [-PI_F, PI_F] for finite input; C's signed zeros."""
    f32 = np.float32
    y, x = np.asarray(y, f32), np.asarray(x, f32)
    ax, ay = np.abs(x), np.abs(y)
    mx, mn = np.maximum(ax, ay), np.minimum(ax, ay)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore", under="ignore"):
        t = np.where(mx > 0, mn / np.where(mx > 0, mx, f32(1)), f32(0)).astype(f32)
        s = t * t
        q = np.full_like(s, ATAN_C[7])
        for k in range(6, -1, -1):
            q = q * s + ATAN_C[k]
        p = t * q
        p = np.where(ay > ax, PI_F * f32(0.5) - p, p)
        p = np.where(np.signbit(x), PI_F - p, p)
        return np.where(np.signbit(y), -p, p).astype(f32)


def _slots(flow: np.ndarray, nop: int) -> np.ndarray:
    F = np.asarray(flow, np.float32)
    assert F.ndim in (3, 4) and F.shape[-1] == nop, (F.shape, nop)
    return F


def flow_to_color(flow: np.ndarray, max_value: float = 0.0):
    """ofdis_flow_color_fullres for flow, bit for bit: Middlebury's MotionToColor / computeColor in float32 without
    contraction.  flow: one slot (h, w, 2) or a batch (n, h, w, 2).  Returns (rgb, scale): (..., 3) uint8 and the
    scale of every slot (float32 scalar for one slot, (n,) for a batch)."""
    f32 = np.float32
    F = _slots(flow, 2)
    one = F.ndim == 3
    F = F[None] if one else F
    u, v = F[..., 0], F[..., 1]
    known = (np.abs(u) <= COLOR_UNKNOWN_THRESH) & (np.abs(v) <= COLOR_UNKNOWN_THRESH)  # NaN fails both
    uk, vk = np.where(known, u, f32(0)), np.where(known, v, f32(0))
    with np.errstate(over="ignore", under="ignore", invalid="ignore"):  # inf * 0 only in the branch not taken
        rad0 = np.sqrt(uk * uk + vk * vk).astype(f32)
        if max_value > 0:
            scale = np.full(F.shape[0], max_value, f32)
        else:
            m = rad0.reshape(F.shape[0], -1).max(axis=1, initial=f32(0)).astype(f32)
            scale = np.where(m == 0, f32(1), m).astype(f32)
        sc = scale[:, None, None]
        fx, fy = uk / sc, vk / sc
        rad = np.sqrt(fx * fx + fy * fy).astype(f32)
        a = atan2_f32(-vk, -uk) / PI_F
        fk = (a + f32(1)) / f32(2) * f32(54)
        k0 = fk.astype(np.int32)
        k1 = (k0 + 1) % 55
        fr = fk - k0.astype(f32)
        rgb = np.zeros(F.shape[:-1] + (3,), np.uint8)
        for b in range(3):
            w0 = COLOR_WHEEL[k0, b].astype(f32) / f32(255)
            w1 = COLOR_WHEEL[k1, b].astype(f32) / f32(255)
            col = (f32(1) - fr) * w0 + fr * w1
            col = np.where(rad <= f32(1), f32(1) - rad * (f32(1) - col), col * f32(0.75))
            rgb[..., b] = np.where(known, (f32(255) * col).astype(np.uint8), np.uint8(0))
    return (rgb[0], scale[0]) if one else (rgb, scale)


def disp_to_color(flow: np.ndarray, max_value: float = 0.0, swapped=False):
    """ofdis_flow_color_fullres for stereo, bit for bit: KITTI's disp_to_color in float32 without contraction.
    flow: one slot (h, w, 1) or a batch (n, h, w, 1) in this library's sign; d = -F, or +F where `swapped` (a bool, or
    one per slot of a batch).  Returns (rgb, scale) as flow_to_color does."""
    f32 = np.float32
    F = _slots(flow, 1)
    one = F.ndim == 3
    F = F[None] if one else F
    sw = np.broadcast_to(np.asarray(swapped, bool), (F.shape[0],))
    d = np.where(sw[:, None, None], F[..., 0], -F[..., 0])
    with np.errstate(invalid="ignore"):
        valid = (d >= 0) & (d <= COLOR_UNKNOWN_THRESH)
    dv = np.where(valid, d, f32(0))
    if max_value > 0:
        scale = np.full(F.shape[0], max_value, f32)
    else:
        m = dv.reshape(F.shape[0], -1).max(axis=1, initial=f32(0)).astype(f32)
        scale = np.fmax(m, f32(1)).astype(f32)
    wt, cum = disp_color_bins()
    with np.errstate(over="ignore", under="ignore"):
        val = np.fmin(np.fmax(dv / scale[:, None, None], f32(0)), f32(1))
        i = np.full(val.shape, 6, np.int32)
        for k in range(6, -1, -1):
            i = np.where(val < cum[k + 1], k, i)
        w = f32(1) - (val - cum[i]) * np.concatenate([wt, [f32(0)]])[i]
        rgb = np.zeros(F.shape[:-1] + (3,), np.uint8)
        for c in range(3):
            m0 = DISP_COLOR_MAP[i, c].astype(f32)
            m1 = DISP_COLOR_MAP[i + 1, c].astype(f32)
            x = np.fmin(np.fmax((w * m0 + (f32(1) - w) * m1) * f32(255), f32(0)), f32(255))
            rgb[..., c] = np.where(valid, x.astype(np.uint8), np.uint8(0))
    return (rgb[0], scale[0]) if one else (rgb, scale)


def _bilinear_frame(img: np.ndarray, xs: np.ndarray, ys: np.ndarray) -> np.ndarray:
    """bil(I, xs, ys) of ofdis_interpolate_fullres: img (h, w, C) float32 of the bytes, (xs, ys) float32 positions in
    the frame; corners floor and min(floor + 1, size - 1), horizontal pass first.  Returns (..., C) float32."""
    f32 = np.float32
    h, w = img.shape[:2]
    x0 = np.floor(xs).astype(np.int64)
    y0 = np.floor(ys).astype(np.int64)
    x1 = np.minimum(x0 + 1, w - 1)
    y1 = np.minimum(y0 + 1, h - 1)
    fx = (xs - x0.astype(f32)).astype(f32)[..., None]
    fy = (ys - y0.astype(f32)).astype(f32)[..., None]
    gx, gy = f32(1) - fx, f32(1) - fy
    r0 = img[y0, x0] * gx + img[y0, x1] * fx
    r1 = img[y1, x0] * gx + img[y1, x1] * fx
    return r0 * gy + r1 * fy


def _fill_holes(ut: np.ndarray, filled: np.ndarray):
    """Step 4 of ofdis_interpolate_fullres in place: Jacobi rounds in which a hole with a neighbour (left, right, up,
    down) filled before the round takes s / k, s = 0 plus those neighbours in that order.  Returns the rounds run."""
    f32 = np.float32
    h, w, nop = ut.shape
    rounds = 0
    while not filled.all():
        rounds += 1
        s = np.zeros_like(ut)
        k = np.zeros((h, w), np.int32)
        for dy, dx in ((0, -1), (0, 1), (-1, 0), (1, 0)):  # left, right, up, down
            nf = np.zeros((h, w), bool)
            nv = np.zeros_like(ut)
            ys, yd = (slice(0, h - 1), slice(1, h)) if dy < 0 else (slice(1, h), slice(0, h - 1)) if dy > 0 else \
                (slice(0, h), slice(0, h))
            xs, xd = (slice(0, w - 1), slice(1, w)) if dx < 0 else (slice(1, w), slice(0, w - 1)) if dx > 0 else \
                (slice(0, w), slice(0, w))
            nf[yd, xd] = filled[ys, xs]
            nv[yd, xd] = ut[ys, xs]
            s = s + np.where(nf[..., None], nv, f32(0))
            k += nf
        new = ~filled & (k > 0)
        ut[new] = s[new] / k[new].astype(f32)[:, None]
        filled |= new
    return rounds


def _interpolate_pair(i0: np.ndarray, i1: np.ndarray, F: np.ndarray, B: np.ndarray, t: float, alpha: float,
                      beta: float):
    f32 = np.float32
    h, w, nop = F.shape
    I0 = i0.reshape(h, w, -1).astype(f32)
    I1 = i1.reshape(h, w, -1).astype(f32)
    tt = f32(t)
    m0, _ = consistency_check(F, B, alpha, beta)
    m1, _ = consistency_check(B, F, alpha, beta)
    X = np.arange(w, dtype=f32)[None, :]
    Y = np.arange(h, dtype=f32)[:, None]
    u = F[..., 0]
    v = F[..., 1] if nop == 2 else np.zeros_like(u)
    with np.errstate(invalid="ignore", over="ignore"):
        # 2. match cost
        xs, ys = X + u, Y + v
        inside = (xs >= 0) & (xs <= f32(w - 1)) & (ys >= 0) & (ys <= f32(h - 1))
        b = _bilinear_frame(I1, np.where(inside, xs, f32(0)), np.where(inside, ys, f32(0)))
        c = np.zeros((h, w), f32)
        for ch in range(I0.shape[2]):
            c = c + np.abs(I0[..., ch] - b[..., ch])
        c = np.where(inside, c, f32(np.inf)).astype(f32)
        # 3. forward splat: the smallest key (cost bits, source index) per target
        known = (np.abs(u) <= f32(INTERP_UNKNOWN_THRESH)) & (np.abs(v) <= f32(INTERP_UNKNOWN_THRESH))
        px, py = X + tt * u, Y + tt * v
        ok = known & (px > f32(-1)) & (px < f32(w)) & (py > f32(-1)) & (py < f32(h))
    src = np.flatnonzero(ok)
    pxs, pys = px.reshape(-1)[src], py.reshape(-1)[src]
    flx, fly = np.floor(pxs), np.floor(pys)
    tx, ty = flx.astype(np.int64), fly.astype(np.int64)
    key = (c.reshape(-1)[src].view(np.uint32).astype(np.uint64) << np.uint64(32)) | src.astype(np.uint64)
    keys = np.full(h * w, _NO_SOURCE, np.uint64)
    for dy in (0, 1):
        for dx in (0, 1):
            xx, yy = tx + dx, ty + dy
            sel = ((dx == 0) | (pxs > flx)) & ((dy == 0) | (pys > fly)) & (xx >= 0) & (xx < w) & (yy >= 0) & (yy < h)
            np.minimum.at(keys, yy[sel] * w + xx[sel], key[sel])
    filled = keys != _NO_SOURCE
    ut = np.zeros((h * w, nop), f32)
    ut[filled] = F.reshape(-1, nop)[(keys[filled] & np.uint64(0xFFFFFFFF)).astype(np.int64)]
    ut = ut.reshape(h, w, nop)
    # 4. hole filling (a pair that no source reached keeps u_t = 0)
    rounds = _fill_holes(ut, filled.reshape(h, w)) if filled.any() else 0
    # 5. color
    uu = ut[..., 0]
    vv = ut[..., 1] if nop == 2 else np.zeros_like(uu)
    x0, y0 = X - tt * uu, Y - tt * vv
    x1, y1 = X + (f32(1) - tt) * uu, Y + (f32(1) - tt) * vv
    in0 = (x0 >= 0) & (x0 <= f32(w - 1)) & (y0 >= 0) & (y0 <= f32(h - 1))
    in1 = (x1 >= 0) & (x1 <= f32(w - 1)) & (y1 >= 0) & (y1 <= f32(h - 1))
    clampx = lambda a: np.fmin(np.fmax(a, f32(0)), f32(w - 1))  # noqa: E731
    clampy = lambda a: np.fmin(np.fmax(a, f32(0)), f32(h - 1))  # noqa: E731
    s0 = _bilinear_frame(I0, clampx(x0), clampy(y0))
    s1 = _bilinear_frame(I1, clampx(x1), clampy(y1))
    rnd = lambda a, ins: np.floor(np.where(ins, a, f32(0)) + f32(0.5)).astype(np.int64)  # noqa: E731
    o0 = in0 & (m0[rnd(y0, in0), rnd(x0, in0)] != 0)
    o1 = in1 & (m1[rnd(y1, in1), rnd(x1, in1)] != 0)
    only0 = ((in0 & ~in1) | (o0 & ~o1))[..., None]
    only1 = ((in1 & ~in0) | (o1 & ~o0))[..., None]
    val = np.where(only0, s0, np.where(only1, s1, (f32(1) - tt) * s0 + tt * s1))
    out = (np.fmin(np.fmax(val, f32(0)), f32(255)) + f32(0.5)).astype(np.uint8)
    return out, ut, rounds


INTERP_UNKNOWN_THRESH = 1e9  # a source splats only when |u|, |v| <= this (NaN fails), the rule of flow_error
_NO_SOURCE = np.uint64(0xFFFFFFFFFFFFFFFF)


def interpolate_frames(frames0: np.ndarray, frames1: np.ndarray, fw: np.ndarray, bw: np.ndarray, t: float,
                       alpha: float, beta: float, with_rounds: bool = False):
    """ofdis_interpolate_fullres bit for bit: the frame at time t between frames0 and frames1 from the forward flow
    fw (frames0 -> frames1) and its backward partner bw, float32 without contraction.  One pair: frames (h, w[, noc])
    uint8 and flows (h, w, nop); a batch: a leading axis on all four.  The masks are consistency_check's, the splat is
    np.minimum.at on the 64-bit keys, the hole filling restates the Jacobi rounds.  Returns (out, flow_t): out uint8
    of the frames' shape, flow_t float32 of the flows' shape (u_t); with_rounds also the most hole-filling rounds any
    pair needed."""
    F = np.asarray(fw, np.float32)
    B = np.asarray(bw, np.float32)
    a0 = np.asarray(frames0, np.uint8)
    a1 = np.asarray(frames1, np.uint8)
    one = F.ndim == 3
    if one:
        F, B, a0, a1 = F[None], B[None], a0[None], a1[None]
    assert F.ndim == 4 and B.shape == F.shape and a0.shape == a1.shape and a0.shape[:3] == F.shape[:3], \
        (F.shape, B.shape, a0.shape, a1.shape)
    out = np.empty(a0.shape, np.uint8)
    flow_t = np.empty(F.shape, np.float32)
    rounds = 0
    for k in range(F.shape[0]):
        o, ut, r = _interpolate_pair(a0[k], a1[k], F[k], B[k], t, alpha, beta)
        out[k] = o.reshape(a0.shape[1:])
        flow_t[k] = ut
        rounds = max(rounds, r)
    if one:
        out, flow_t = out[0], flow_t[0]
    return (out, flow_t, rounds) if with_rounds else (out, flow_t)


# ofdis_track_point (include/ofdis_b200.h), field for field
TRACK_POINT_DTYPE = np.dtype([("id", "<i4"), ("x", "<f4"), ("y", "<f4")])
# ofdis_track_params, field for field
TRACK_PARAM_FIELDS = ("capacity", "spacing", "alpha", "beta", "mb_alpha", "mb_beta", "min_eig")
TRACK_STATS_FIELDS = ("seeded", "ended_leaves", "ended_inconsistent", "ended_boundary", "dropped", "alive", "next_id")
_TRACK_ID_END = 2 ** 31 - 1  # next_id never exceeds this


def _flow_bilinear(F: np.ndarray, xs: np.ndarray, ys: np.ndarray):
    """Channels of the full-resolution flow F (h, w, nop) at in-frame positions: the rule of consistency_check."""
    f32 = np.float32
    h, w, nop = F.shape
    x0 = np.floor(xs).astype(np.int64)
    y0 = np.floor(ys).astype(np.int64)
    x1 = np.minimum(x0 + 1, w - 1)
    y1 = np.minimum(y0 + 1, h - 1)
    fx = (xs - x0.astype(f32)).astype(f32)
    fy = (ys - y0.astype(f32)).astype(f32)
    gx, gy = f32(1) - fx, f32(1) - fy
    out = []
    for c in range(nop):
        Fc = F[..., c]
        r0 = Fc[y0, x0] * gx + Fc[y0, x1] * fx
        r1 = Fc[y1, x0] * gx + Fc[y1, x1] * fx
        out.append(r0 * gy + r1 * fy)
    return out


def track_seed_eigen(frame: np.ndarray, spacing: int):
    """The seed pixels (cx, cy) of every cell, row-major, and the smaller eigenvalue of the structure tensor over the
    5 x 5 window around each (ofdis_track_begin's header), float32."""
    f32 = np.float32
    I = np.asarray(frame, np.uint8)
    h, w = I.shape[:2]
    if I.ndim == 3 and I.shape[2] == 3:
        g = (I[..., 0].astype(f32) + I[..., 1].astype(f32) + I[..., 2].astype(f32)) / f32(3)
    else:
        g = I.reshape(h, w).astype(f32)
    xs = np.arange(w)
    ys = np.arange(h)
    Ix = (g[:, np.minimum(xs + 1, w - 1)] - g[:, np.maximum(xs - 1, 0)]) * f32(0.5)
    Iy = (g[np.minimum(ys + 1, h - 1), :] - g[np.maximum(ys - 1, 0), :]) * f32(0.5)
    s = int(spacing)
    ncx, ncy = (w - 1) // s + 1, (h - 1) // s + 1
    c = np.arange(ncx * ncy)
    cx = np.minimum((c % ncx) * s + s // 2, w - 1)
    cy = np.minimum((c // ncx) * s + s // 2, h - 1)
    a = np.zeros(c.size, f32)
    b = np.zeros(c.size, f32)
    d2 = np.zeros(c.size, f32)
    for dy in range(-2, 3):
        py = np.clip(cy + dy, 0, h - 1)
        for dx in range(-2, 3):
            px = np.clip(cx + dx, 0, w - 1)
            ix, iy = Ix[py, px], Iy[py, px]
            a = a + ix * ix
            b = b + ix * iy
            d2 = d2 + iy * iy
    d = a - d2
    lam = (a + d2) * f32(0.5) - np.sqrt(d * d * f32(0.25) + b * b)
    return cx, cy, lam


# ---- per-pixel confidence (ofdis_confidence_fullres) -----------------------------------------------------------
CONF_PARAM_FIELDS = ("radius", "s_fb", "s_tex", "min_count")
_QNAN32 = np.uint32(0x7FC00000).view(np.float32)


def confidence(frame0: np.ndarray, frame1: np.ndarray, F: np.ndarray, B: np.ndarray | None, params):
    """Restates ofdis_confidence_fullres for one pair: frame0, frame1 (H, W[, 3]) uint8, F and its partner B (H, W, nop)
    or (H, W) float32 full-resolution flows (B None: no forward-backward term), params a mapping with
    CONF_PARAM_FIELDS.  Returns (conf (H, W), terms (H, W, 3): z, e, lambda), float32, in the header's order."""
    r, min_count = int(params["radius"]), int(params["min_count"])
    s_fb, s_tex = f32(params["s_fb"]), f32(params["s_tex"])
    g0, g1 = _brightness(np.asarray(frame0, np.uint8)), _brightness(np.asarray(frame1, np.uint8))
    H, W = g0.shape
    Fa = np.asarray(F, f32).reshape(H, W, -1)
    xs_, ys_ = np.arange(W), np.arange(H)
    Ix = (g0[:, np.minimum(xs_ + 1, W - 1)] - g0[:, np.maximum(xs_ - 1, 0)]) * f32(0.5)
    Iy = (g0[np.minimum(ys_ + 1, H - 1), :] - g0[np.maximum(ys_ - 1, 0), :]) * f32(0.5)
    with np.errstate(invalid="ignore", over="ignore"):
        xs = np.arange(W, dtype=f32)[None, :] + Fa[..., 0]
        ys = np.arange(H, dtype=f32)[:, None] + (Fa[..., 1] if Fa.shape[2] == 2 else f32(0))
        inside = (xs >= 0) & (xs <= f32(W - 1)) & (ys >= 0) & (ys <= f32(H - 1))
        Iw = _bilinear_frame(g1[..., None], np.where(inside, xs, f32(0)), np.where(inside, ys, f32(0)))[..., 0]
    Iw = np.where(inside, Iw, _QNAN32).astype(f32)
    win = [(np.clip(ys_ + dy, 0, H - 1)[:, None], np.clip(xs_ + dx, 0, W - 1)[None, :])
           for dy in range(-r, r + 1) for dx in range(-r, r + 1)]
    zero = np.zeros((H, W), f32)
    n = np.zeros((H, W), np.int64)
    s0, s1, a, b, c = zero.copy(), zero.copy(), zero.copy(), zero.copy(), zero.copy()
    for q in win:
        v = inside[q]
        n += v
        s0 = s0 + np.where(v, g0[q], f32(0))  # adding +0.0 to these sums leaves them as they are
        s1 = s1 + np.where(v, Iw[q], f32(0))
        ix, iy = Ix[q], Iy[q]
        a = a + ix * ix
        b = b + ix * iy
        c = c + iy * iy
    d = a - c
    lam = (a + c) * f32(0.5) - np.sqrt(d * d * f32(0.25) + b * b)
    with np.errstate(invalid="ignore", divide="ignore"):
        nf = n.astype(f32)
        m0, m1 = s0 / nf, s1 / nf
        c00, c11, c01 = zero.copy(), zero.copy(), zero.copy()
        for q in win:
            v = inside[q]
            p0, p1 = g0[q] - m0, Iw[q] - m1
            c00 = c00 + np.where(v, p0 * p0, f32(0))
            c11 = c11 + np.where(v, p1 * p1, f32(0))
            c01 = c01 + np.where(v, p0 * p1, f32(0))
        den = c00 * c11
        z = np.where((n >= min_count) & (den > 0), c01 / np.sqrt(den), _QNAN32).astype(f32)
    if B is None:
        e = np.full((H, W), _QNAN32, f32)
        ce = np.ones((H, W), f32)
    else:
        e = consistency_check(Fa, np.asarray(B, f32).reshape(H, W, -1), 0.0, 0.0)[1]
        with np.errstate(invalid="ignore", over="ignore"):
            ce = np.where(e >= 0, s_fb / (s_fb + e), f32(0)).astype(f32)
    with np.errstate(invalid="ignore"):
        cz = np.where(z > 0, z, f32(0)).astype(f32)
        cl = np.where(lam > 0, lam / (lam + s_tex), f32(0)).astype(f32)
    conf = ((cz * ce) * cl).astype(f32)
    return conf, np.stack([z, e, lam.astype(f32)], -1)


def _track_seed(frame, tracks, next_id, stats, p):
    s = int(p["spacing"])
    h, w = frame.shape[:2]
    cx, cy, lam = track_seed_eigen(frame, s)
    ncx = (w - 1) // s + 1
    occ = np.zeros(cx.size, bool)
    occ[(tracks["y"].astype(np.int64) // s) * ncx + tracks["x"].astype(np.int64) // s] = True
    cells = np.flatnonzero(~occ & (lam >= np.float32(p["min_eig"])))
    adm = max(min(cells.size, int(p["capacity"]) - tracks.size, _TRACK_ID_END - next_id), 0)
    new = np.empty(adm, TRACK_POINT_DTYPE)
    new["id"] = next_id + np.arange(adm)
    new["x"] = cx[cells[:adm]]
    new["y"] = cy[cells[:adm]]
    stats["seeded"] += adm
    stats["dropped"] += cells.size - adm
    return np.concatenate([tracks, new]), next_id + adm


def _track_advance(tracks, F, B, stats, p):
    f32 = np.float32
    h, w, nop = F.shape
    x, y = tracks["x"], tracks["y"]
    with np.errstate(invalid="ignore", over="ignore"):
        f = _flow_bilinear(F, x, y)
        u = f[0]
        v = f[1] if nop == 2 else np.zeros_like(u)
        xn, yn = x + u, y + v
        inside = (xn >= 0) & (xn <= f32(w - 1)) & (yn >= 0) & (yn <= f32(h - 1))
        b = _flow_bilinear(B, np.where(inside, xn, f32(0)), np.where(inside, yn, f32(0)))
        b0 = b[0]
        b1 = b[1] if nop == 2 else np.zeros_like(u)
        du = u + b0
        dv = v + b1 if nop == 2 else np.zeros_like(u)
        err = du * du + dv * dv
        mag = (u * u + v * v) + (b0 * b0 + b1 * b1)
        consistent = inside & (err <= f32(p["alpha"]) * mag + f32(p["beta"]))
        xr = np.floor(x + f32(0.5)).astype(np.int64)
        yr = np.floor(y + f32(0.5)).astype(np.int64)
        l, r = F[yr, np.maximum(xr - 1, 0)], F[yr, np.minimum(xr + 1, w - 1)]
        up, dn = F[np.maximum(yr - 1, 0), xr], F[np.minimum(yr + 1, h - 1), xr]
        ux = (r[:, 0] - l[:, 0]) * f32(0.5)
        uy = (dn[:, 0] - up[:, 0]) * f32(0.5)
        g2 = ux * ux + uy * uy
        if nop == 2:
            vx = (r[:, 1] - l[:, 1]) * f32(0.5)
            vy = (dn[:, 1] - up[:, 1]) * f32(0.5)
            g2 = g2 + (vx * vx + vy * vy)
        boundary = consistent & (g2 > f32(p["mb_alpha"]) * (u * u + v * v) + f32(p["mb_beta"]))
    keep = consistent & ~boundary
    stats["ended_leaves"] += int((~inside).sum())
    stats["ended_inconsistent"] += int((inside & ~consistent).sum())
    stats["ended_boundary"] += int(boundary.sum())
    out = tracks[keep].copy()
    out["x"] = xn[keep]
    out["y"] = yn[keep]
    return out


def track_points(frames: np.ndarray, fw: np.ndarray, bw: np.ndarray, params):
    """ofdis_track_begin on frames[0] followed by ofdis_track_advance through the n pairs, bit for bit, float32
    without contraction.  frames: the clip, (n + 1, h, w[, noc]) uint8; fw, bw: the full-resolution forward flows
    (frame k -> k + 1) and their backward partners, (n, h, w, nop) float32 (stereo also without the last axis);
    params: a mapping with the keys of TRACK_PARAM_FIELDS.  Returns (lists, stats): n + 1 arrays of
    TRACK_POINT_DTYPE, the live tracks after each frame sorted by id, and a dict of TRACK_STATS_FIELDS."""
    p = {k: params[k] for k in TRACK_PARAM_FIELDS}
    clip = np.asarray(frames, np.uint8)
    F = np.asarray(fw, np.float32)
    B = np.asarray(bw, np.float32)
    n = clip.shape[0] - 1
    F = F.reshape(F.shape[:3] + (-1,))
    B = B.reshape(B.shape[:3] + (-1,))
    assert F.shape[0] == n and B.shape == F.shape and F.shape[1:3] == clip.shape[1:3], (clip.shape, F.shape, B.shape)
    stats = dict.fromkeys(TRACK_STATS_FIELDS, 0)
    tracks, next_id = _track_seed(clip[0], np.empty(0, TRACK_POINT_DTYPE), 0, stats, p)
    lists = [tracks]
    for k in range(n):
        tracks = _track_advance(tracks, F[k], B[k], stats, p)
        tracks, next_id = _track_seed(clip[k + 1], tracks, next_id, stats, p)
        lists.append(tracks)
    stats["alive"], stats["next_id"] = int(tracks.size), int(next_id)
    return lists, stats


DISP_FILTER_FIELDS = ("lr_check", "alpha", "beta", "speckle_size", "speckle_diff", "fill")
STEREO_CAMERA_FIELDS = ("fx", "fy", "cx", "cy", "baseline", "doffs")


def _smaller(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """(b < a) ? b : a elementwise: of two equal values (+0 and -0 among them) the first one."""
    return np.where(b < a, b, a)


def _fill_lines(v: np.ndarray, has: np.ndarray) -> np.ndarray:
    """The fill rule along axis 1 of v (lines x positions) where `has` marks the values: a run without a value between
    two values takes the smaller of them (the earlier one where equal), runs at either end the one value next to them;
    a line without a value stays qNaN."""
    n = v.shape[1]
    pos = np.arange(n)[None, :]
    left = np.maximum.accumulate(np.where(has, pos, -1), axis=1)
    right = np.minimum.accumulate(np.where(has, pos, n)[:, ::-1], axis=1)[:, ::-1]
    rows = np.arange(v.shape[0])[:, None]
    vl = np.where(left >= 0, v[rows, np.clip(left, 0, n - 1)], _QNAN)
    vr = np.where(right < n, v[rows, np.clip(right, 0, n - 1)], _QNAN)
    out = np.where(left < 0, vr, np.where(right >= n, vl, _smaller(vl, vr)))
    return np.where(has, v, out).astype(np.float32)


def speckle_components(d: np.ndarray, valid: np.ndarray, diff: float):
    """Connected components of the `valid` pixels of one frame, 4-neighbours joined when fabsf(d_p - d_q) <= diff in
    float32 (scipy.sparse.csgraph.connected_components over the joined edges).  Returns (labels, sizes): a label per
    pixel and each pixel's component size (0 where not valid)."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components

    h, w = d.shape
    f32 = np.float32
    idx = np.arange(h * w).reshape(h, w)
    edges = []
    with np.errstate(invalid="ignore", over="ignore"):
        for a, b, da, db in ((idx[:, :-1], idx[:, 1:], d[:, :-1], d[:, 1:]), (idx[:-1], idx[1:], d[:-1], d[1:])):
            va = valid.reshape(-1)[a]
            vb = valid.reshape(-1)[b]
            ok = va & vb & (np.abs((da - db).astype(f32)) <= f32(diff))
            edges.append((a[ok], b[ok]))
    r = np.concatenate([e[0] for e in edges])
    c = np.concatenate([e[1] for e in edges])
    g = coo_matrix((np.ones(r.size, np.int8), (r, c)), shape=(h * w, h * w))
    _, labels = connected_components(g, directed=False)
    counts = np.bincount(labels[valid.reshape(-1)], minlength=labels.max() + 1 if labels.size else 0)
    sizes = np.where(valid.reshape(-1), counts[labels], 0).reshape(h, w)
    return labels.reshape(h, w), sizes


def disparity_filter(F: np.ndarray, B: np.ndarray | None = None, swapped: bool = False, lr_check: int = 0,
                     alpha: float = 0.0, beta: float = 1.0, speckle_size: int = 0, speckle_diff: float = 1.0,
                     fill: int = 0, camera=None):
    """One pair of ofdis_disparity_fullres, bit for bit, float32 without contraction.  F: slot a's full-resolution
    stereo flow, (h, w) or (h, w, 1) float32, exactly what ofdis_get_flow_fullres returns; B: its partner slot's (read
    only with lr_check); swapped: slot a is marked swapped.  camera: None or a mapping with STEREO_CAMERA_FIELDS.
    Returns (disp, status, depth, xyz): (h, w) float32, (h, w) uint8, and with a camera (h, w) and (h, w, 3) float32
    (else None).

        d = -F (+F when swapped); status 3 where d is not in [0, 1e9], else with lr_check consistency_check's mask of F
        against B, else 0.
        speckle_size > 0: components of status-0 pixels (4-neighbours, fabsf(d_p - d_q) <= speckle_diff) of at most
        speckle_size pixels get status 4.
        fill: the row pass (_fill_lines on the rows, values where the status is 0), then the same along the columns.
        disp: d where the status is 0, the filled value, else qNaN.
        depth: Z = (fx * baseline) / (D + doffs) where D + doffs > 0, else qNaN; xyz: ((x - cx) Z / fx,
        (y - cy) Z / fy, Z); every NaN of depth and xyz is qNaN."""
    f32 = np.float32
    Fa = np.asarray(F, f32)
    Fa = Fa.reshape(Fa.shape[:2] + (-1,))
    h, w = Fa.shape[:2]
    d = Fa[..., 0] if swapped else -Fa[..., 0]
    status = np.where((d >= 0) & (d <= f32(1e9)), 0, 3).astype(np.uint8)
    if lr_check:
        mask, _ = consistency_check(Fa, B, alpha, beta)
        status = np.where(status == 0, mask, status).astype(np.uint8)
    if speckle_size > 0:
        _, sizes = speckle_components(d, status == 0, speckle_diff)
        status[(status == 0) & (sizes <= speckle_size)] = 4
    valid = status == 0
    disp = np.where(valid, d, _QNAN).astype(f32)
    if fill:
        rows = _fill_lines(disp, valid)
        full = valid.any(axis=1)
        disp = _fill_lines(rows.T, np.broadcast_to(full[None, :], (w, h))).T.copy()
    depth = xyz = None
    if camera is not None:
        cam = {k: f32(camera[k]) for k in STEREO_CAMERA_FIELDS}
        fb = f32(cam["fx"] * cam["baseline"])
        with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
            s = (disp + cam["doffs"]).astype(f32)
            Z = np.where(s > 0, fb / np.where(s > 0, s, f32(1)), _QNAN).astype(f32)
            Z = np.where(np.isnan(Z), _QNAN, Z).astype(f32)
            X = ((np.arange(w, dtype=f32)[None, :] - cam["cx"]) * Z / cam["fx"]).astype(f32)
            Y = ((np.arange(h, dtype=f32)[:, None] - cam["cy"]) * Z / cam["fy"]).astype(f32)
        canon = lambda a: np.where(np.isnan(a), _QNAN, a).astype(f32)  # noqa: E731
        depth = Z
        xyz = np.stack([canon(X), canon(Y), Z], axis=-1)
    return disp, status, depth, xyz


# ofdis_sf_stats (include/ofdis_b200.h), field for field
SF_STATS_FIELDS = ("n_d1", "n_d2", "n_fl", "n_sf", "out_d1", "out_d2", "out_fl", "out_sf")
SF_STATS_DTYPE = np.dtype([(k, "<i8") for k in SF_STATS_FIELDS])


def _known_disp(d: np.ndarray) -> np.ndarray:
    """0 <= d <= 1e9: NaN fails, -0 passes."""
    return (d >= 0) & (d <= np.float32(1e9))


def sf_gather_d1(D1: np.ndarray, xs: np.ndarray, ys: np.ndarray, inside: np.ndarray, edge_diff) -> np.ndarray:
    """Step 2 of ofdis_scene_flow_fullres: the second disparity D1 (n, h, w) gathered at the targets (xs, ys) (float32,
    (n, ...)) that lie in the frame (`inside`; the value elsewhere is meaningless).  Four known corners spread by at
    most edge_diff blend bilinearly, rows first; otherwise the nearest corner."""
    f32 = np.float32
    n, h, w = D1.shape
    with np.errstate(invalid="ignore", over="ignore"):
        xc = np.where(inside, xs, f32(0))
        yc = np.where(inside, ys, f32(0))
        x0 = np.floor(xc).astype(np.int64)
        y0 = np.floor(yc).astype(np.int64)
        x1 = np.minimum(x0 + 1, w - 1)
        y1 = np.minimum(y0 + 1, h - 1)
        fx = (xc - x0.astype(f32)).astype(f32)
        fy = (yc - y0.astype(f32)).astype(f32)
        k = np.arange(n).reshape((n,) + (1,) * (xs.ndim - 1))
        c00, c10, c01, c11 = D1[k, y0, x0], D1[k, y0, x1], D1[k, y1, x0], D1[k, y1, x1]
        corners_known = _known_disp(c00) & _known_disp(c10) & _known_disp(c01) & _known_disp(c11)
        hi = np.maximum(np.maximum(c00, c10), np.maximum(c01, c11))
        lo = np.minimum(np.minimum(c00, c10), np.minimum(c01, c11))
        blend = corners_known & ((hi - lo) <= f32(edge_diff))
        gx, gy = f32(1) - fx, f32(1) - fy
        r0 = c00 * gx + c10 * fx
        r1 = c01 * gx + c11 * fx
        near = np.where(fy >= f32(0.5), np.where(fx >= f32(0.5), c11, c01), np.where(fx >= f32(0.5), c10, c00))
        return np.where(blend, r0 * gy + r1 * fy, near).astype(f32)


def scene_flow(F: np.ndarray, disp0: np.ndarray, disp1: np.ndarray, edge_diff: float = 1.0, camera=None, gt=None,
               classes: np.ndarray | None = None, nclasses: int = 1):
    """ofdis_scene_flow_fullres bit for bit, float32 without contraction.  F: full-resolution flows, (h, w, 2) for one
    pair or (n, h, w, 2), exactly what ofdis_get_flow_fullres returns; disp0, disp1: the positive disparities at t and
    t+1, (h, w) or (n, h, w) float32 with NaN for unknown; camera: None or a mapping with STEREO_CAMERA_FIELDS; gt: None
    or (disp0, disp1, flow) of the same shapes, with classes (uint8, the shape of disp0; None: class 0) and nclasses.
    Returns (disp1_warped, status, motion, stats): float32 and uint8 of disp0's shape, motion (..., 3) float32 (None
    without a camera), stats of SF_STATS_DTYPE, (nclasses,) for one pair or (n, nclasses) (None without gt).

        target       (xs, ys) = (x + u, y + v); fails outside [0, w-1] x [0, h-1] or NaN
        d1           corners x0 = floor(xs), x1 = min(x0 + 1, w - 1) (and y); four known corners with max - min <=
                     edge_diff: bilinear, rows first; else the corner (fx >= 0.5 ? x1 : x0, fy >= 0.5 ? y1 : y0)
        status       bit 0 d0 unknown, bit 1 the target fails, bit 2 d1 unknown (bit 1 clear)
        disp1_warped d1 where bits 1 and 2 are clear, else qNaN
        motion       P1 - P0 where status = 0 and d + doffs > 0 for both, P = (((x - cx) Z) / fx, ((y - cy) Z) / fy, Z)
                     with Z = (fx * baseline) / (d + doffs) and P1 at (xs, ys); else qNaN
        outliers     e > 3 and e > 0.05 g; D1 |d0 - G|, D2 |disp1_warped - G|, Fl |F - G|; an unknown estimate has
                     e = +inf; each counts where its ground truth is known, SF where all three are, as any of them"""
    f32 = np.float32
    Fa = np.asarray(F, f32)
    single = Fa.ndim == 3
    if single:
        Fa = Fa[None]
    n, h, w, _ = Fa.shape
    D0 = np.asarray(disp0, f32).reshape(n, h, w)
    D1 = np.asarray(disp1, f32).reshape(n, h, w)
    u, v = Fa[..., 0], Fa[..., 1]
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        xs = np.arange(w, dtype=f32)[None, None, :] + u
        ys = np.arange(h, dtype=f32)[None, :, None] + v
        inside = (xs >= 0) & (xs <= f32(w - 1)) & (ys >= 0) & (ys <= f32(h - 1))
        d1 = sf_gather_d1(D1, xs, ys, inside, edge_diff)
        k0 = _known_disp(D0)
        k1 = inside & _known_disp(d1)
        status = (np.where(k0, 0, 1) | np.where(inside, 0, 2) | np.where(inside & ~k1, 4, 0)).astype(np.uint8)
        d1w = np.where(k1, d1, _QNAN).astype(f32)
        motion = None
        if camera is not None:
            cam = {key: f32(camera[key]) for key in STEREO_CAMERA_FIELDS}
            fb = f32(cam["fx"] * cam["baseline"])
            s0 = (D0 + cam["doffs"]).astype(f32)
            s1 = (d1 + cam["doffs"]).astype(f32)
            ok = (status == 0) & (s0 > 0) & (s1 > 0)
            Z0 = fb / np.where(ok, s0, f32(1))
            Z1 = fb / np.where(ok, s1, f32(1))
            X0 = ((np.arange(w, dtype=f32)[None, None, :] - cam["cx"]) * Z0) / cam["fx"]
            Y0 = ((np.arange(h, dtype=f32)[None, :, None] - cam["cy"]) * Z0) / cam["fy"]
            X1 = ((xs - cam["cx"]) * Z1) / cam["fx"]
            Y1 = ((ys - cam["cy"]) * Z1) / cam["fy"]
            motion = np.stack([X1 - X0, Y1 - Y0, Z1 - Z0], axis=-1).astype(f32)
            motion = np.where(ok[..., None] & ~np.isnan(motion), motion, _QNAN).astype(f32)
        stats = None
        if gt is not None:
            G0, G1, GF = (np.asarray(a, f32) for a in gt)
            G0, G1, GF = G0.reshape(n, h, w), G1.reshape(n, h, w), GF.reshape(n, h, w, 2)
            cls = np.zeros((n, h, w), np.uint8) if classes is None else np.asarray(classes, np.uint8).reshape(n, h, w)
            assert classes is not None or nclasses == 1
            lim, inf = f32(1e9), f32(np.inf)
            kg0, kg1 = _known_disp(G0), _known_disp(G1)
            Gu, Gv = GF[..., 0], GF[..., 1]
            kgf = (np.abs(Gu) <= lim) & (np.abs(Gv) <= lim)
            kf = (np.abs(u) <= lim) & (np.abs(v) <= lim)
            du, dv = u - Gu, v - Gv
            e0 = np.where(k0, np.abs(D0 - G0), inf)
            e1 = np.where(k1, np.abs(d1w - G1), inf)
            ef = np.where(kf, np.sqrt(du * du + dv * dv), inf)
            gf = np.sqrt(Gu * Gu + Gv * Gv)

            def out(e, g):
                return (e > f32(3)) & (e > f32(0.05) * g)

            o0, o1, of = out(e0, np.abs(G0)), out(e1, np.abs(G1)), out(ef, gf)
            ksf = kg0 & kg1 & kgf
            masks = (kg0, kg1, kgf, ksf, kg0 & o0, kg1 & o1, kgf & of, ksf & (o0 | o1 | of))
            stats = np.zeros((n, nclasses), SF_STATS_DTYPE)
            for p in range(n):
                for c in range(nclasses):
                    sel = cls[p] == c
                    for name, m in zip(SF_STATS_FIELDS, masks):
                        stats[p, c][name] = int((m[p] & sel).sum())
    if single:
        return d1w[0], status[0], None if motion is None else motion[0], None if stats is None else stats[0]
    return d1w, status, motion, stats


# ofdis_motion_params / ofdis_motion_stats (include/ofdis_b200.h), field for field
MOTION_MODELS = {"similarity": 1, "affine": 2, "homography": 3}
MOTION_PARAM_FIELDS = ("model", "step", "fb_check", "alpha", "beta", "hypotheses", "threshold", "refine", "seed")
MOTION_STATS_DTYPE = np.dtype([("status", "<i4"), ("n_corr", "<i4"), ("best_hypothesis", "<i4"),
                               ("ransac_inliers", "<i4"), ("refits", "<i4"), ("n_inliers", "<i4")])
MOTION_UNKNOWN_THRESH = 1e9  # a flow component above this (or NaN) is unknown, the rule of flow_error
_SPLITMIX_GAMMA = 0x9E3779B97F4A7C15
_QNAN64 = np.uint64(0x7FF8000000000000).view(np.float64)


def splitmix64(z) -> np.ndarray:
    """SplitMix64's finalizer on uint64 values (mod 2^64): the n-th output of the generator seeded with s is
    splitmix64(s + n * 0x9E3779B97F4A7C15)."""
    z = np.array(z, dtype=np.uint64, ndmin=1)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def motion_draws(seed: int, hypotheses: int, n_min: int, m: int) -> np.ndarray:
    """The correspondence indices (hypotheses, n_min) of ofdis_global_motion_fullres's draws."""
    n = (8 * np.arange(hypotheses, dtype=np.uint64)[:, None] + np.arange(n_min, dtype=np.uint64)[None, :]
         + np.uint64(1))
    with np.errstate(over="ignore"):
        z = splitmix64(np.uint64(seed % 2 ** 64) + n * np.uint64(_SPLITMIX_GAMMA)).reshape(n.shape)
    return (((z >> np.uint64(32)) * np.uint64(m)) >> np.uint64(32)).astype(np.int64)


def motion_rows(model: int, c: np.ndarray):
    """The two rows of every correspondence c = (x, y, p, q) float32 (..., 4): (r1, r2, b1, b2), float64, r1 and r2
    (..., k)."""
    x, y, p, q = (c[..., i].astype(np.float64) for i in range(4))
    one, zero = np.ones_like(x), np.zeros_like(x)
    if model == 1:
        r1 = [x, -y, one, zero]
        r2 = [y, x, zero, one]
    else:
        r1 = [x, y, one, zero, zero, zero]
        r2 = [zero, zero, zero, x, y, one]
        if model == 3:
            r1 += [-(x * p), -(y * p)]
            r2 += [-(x * q), -(y * q)]
    return np.stack(r1, -1), np.stack(r2, -1), p, q


def motion_solve(A: np.ndarray, b: np.ndarray):
    """The elimination of ofdis_global_motion_fullres on a batch of systems A (s, k, k), b (s, k) float64: partial
    pivoting on the first row of the largest |a_ij|, then back substitution.  Returns (x (s, k), ok (s,))."""
    A = np.array(A, np.float64)
    b = np.array(b, np.float64)
    s, k = b.shape
    ar = np.arange(s)
    ok = np.ones(s, bool)
    with np.errstate(all="ignore"):
        for j in range(k):
            best = np.abs(A[:, j, j])
            piv = np.full(s, j)
            for i in range(j + 1, k):
                a = np.abs(A[:, i, j])
                upd = a > best
                best = np.where(upd, a, best)
                piv = np.where(upd, i, piv)
            ok &= best > 0
            rj, rp = A[ar, j].copy(), A[ar, piv].copy()
            A[ar, piv], A[ar, j] = rj, rp
            bj, bp = b[ar, j].copy(), b[ar, piv].copy()
            b[ar, piv], b[ar, j] = bj, bp
            for i in range(j + 1, k):
                f = A[:, i, j] / A[:, j, j]
                A[:, i, j + 1:] = A[:, i, j + 1:] - f[:, None] * A[:, j, j + 1:]
                b[:, i] = b[:, i] - f * b[:, j]
        x = np.zeros((s, k))
        for i in range(k - 1, -1, -1):
            xi = b[:, i]
            for c in range(i + 1, k):
                xi = xi - A[:, i, c] * x[:, c]
            x[:, i] = xi / A[:, i, i]
    return x, ok & np.isfinite(x).all(axis=1)


def motion_hmat(model: int, x: np.ndarray) -> np.ndarray:
    """H^ (..., 9) float64, row-major, of the parameters x (..., k)."""
    z, o = np.zeros(x.shape[:-1]), np.ones(x.shape[:-1])
    if model == 1:
        h = [x[..., 0], -x[..., 1], x[..., 2], x[..., 1], x[..., 0], x[..., 3], z, z, o]
    else:
        h = [x[..., i] for i in range(6)] + ([x[..., 6], x[..., 7]] if model == 3 else [z, z]) + [o]
    return np.stack(h, -1)


def motion_inliers(g: np.ndarray, c: np.ndarray, t) -> np.ndarray:
    """The inlier test of ofdis_global_motion_fullres, float32: g (..., 9) against the correspondences c (m, 4);
    returns (..., m) bool."""
    f32 = np.float32
    g = np.asarray(g, f32)[..., None, :]
    x, y, p, q = c[:, 0], c[:, 1], c[:, 2], c[:, 3]
    with np.errstate(all="ignore"):
        X = (g[..., 0] * x + g[..., 1] * y) + g[..., 2]
        Y = (g[..., 3] * x + g[..., 4] * y) + g[..., 5]
        W = (g[..., 6] * x + g[..., 7] * y) + g[..., 8]
        ex, ey = X - p * W, Y - q * W
        tw = f32(t) * W
        return (W > 0) & (ex * ex + ey * ey <= tw * tw)


def motion_normal_sums(model: int, c: np.ndarray, inl: np.ndarray):
    """The refit's normal equations (A (k, k), b (k,)) from the inliers `inl` of c (m, 4), summed in chunks of 32 from
    +0.0 and a pairwise tree over the chunk sums padded with +0.0 to a power of two."""
    r1, r2, b1, b2 = motion_rows(model, c)
    k = r1.shape[1]
    terms = [(r1[:, a] * r1[:, b]) + (r2[:, a] * r2[:, b]) for a in range(k) for b in range(a, k)]
    terms += [(r1[:, a] * b1) + (r2[:, a] * b2) for a in range(k)]
    T = np.where(inl[:, None], np.stack(terms, -1), 0.0)
    m, ne = T.shape
    nc = (m + 31) // 32
    T = np.concatenate([T, np.zeros((nc * 32 - m, ne))]).reshape(nc, 32, ne)
    v = np.zeros((nc, ne))
    for e in range(32):
        v = v + T[:, e]
    P = 1
    while P < nc:
        P *= 2
    v = np.concatenate([v, np.zeros((P - nc, ne))])
    while v.shape[0] > 1:
        v = v[0::2] + v[1::2]
    A = np.zeros((k, k))
    e = 0
    for a in range(k):
        for b in range(a, k):
            A[a, b] = A[b, a] = v[0, e]
            e += 1
    return A, v[0, e:]


def motion_to_pixels(model: int, H: np.ndarray, cx, cy, sigma) -> np.ndarray:
    """M = T^-1 H^ T (9,) float64 in the expression order of the header."""
    S, Cx, Cy = float(sigma), float(cx), float(cy)
    A = [0.0] * 9
    for r in range(3):
        A[3 * r] = float(H[3 * r]) * S
        A[3 * r + 1] = float(H[3 * r + 1]) * S
        A[3 * r + 2] = float(H[3 * r + 2]) - (A[3 * r] * Cx + A[3 * r + 1] * Cy)
    M = [0.0] * 9
    for c in range(3):
        M[c] = A[c] / S + Cx * A[6 + c]
        M[3 + c] = A[3 + c] / S + Cy * A[6 + c]
        M[6 + c] = A[6 + c]
    M = np.array(M)
    if model == 3:
        with np.errstate(all="ignore"):
            M = M / M[8]
    return np.where(np.isnan(M), _QNAN64, M)


def motion_params(params) -> dict:
    """The params mapping with the model as its number (names of MOTION_MODELS are accepted)."""
    p = {k: params[k] for k in MOTION_PARAM_FIELDS}
    p["model"] = MOTION_MODELS.get(p["model"], p["model"])
    return p


def _motion_pair(F, B, I1, p):
    f32 = np.float32
    h, w = F.shape[:2]
    model, s = int(p["model"]), int(p["step"])
    n_min, k = model + 1, 2 * (model + 1)
    u, v = F[..., 0], F[..., 1]
    X = np.arange(w, dtype=f32)[None, :]
    Y = np.arange(h, dtype=f32)[:, None]
    with np.errstate(invalid="ignore", over="ignore"):
        xs, ys = X + u, Y + v
        lim = f32(MOTION_UNKNOWN_THRESH)
        valid = (np.abs(u) <= lim) & (np.abs(v) <= lim) & (xs >= 0) & (xs <= f32(w - 1)) & (ys >= 0) & \
            (ys <= f32(h - 1))
    if p["fb_check"]:
        valid &= consistency_check(F, B, p["alpha"], p["beta"])[0] == 0
    # 1. correspondences
    ncx, ncy = (w - 1) // s + 1, (h - 1) // s + 1
    cell = np.arange(ncx * ncy)
    cxs = np.minimum((cell % ncx) * s + s // 2, w - 1)
    cys = np.minimum((cell // ncx) * s + s // 2, h - 1)
    sel = valid[cys, cxs]
    cxs, cys = cxs[sel], cys[sel]
    c_x, c_y = f32(0.5) * f32(w - 1), f32(0.5) * f32(h - 1)
    sigma = f32(2.0) / f32(max(w, h))
    corr = np.stack([(cxs.astype(f32) - c_x) * sigma, (cys.astype(f32) - c_y) * sigma,
                     (xs[cys, cxs] - c_x) * sigma, (ys[cys, cxs] - c_y) * sigma], -1).astype(f32)
    m = corr.shape[0]
    t = f32(p["threshold"]) * sigma
    st = np.zeros((), MOTION_STATS_DTYPE)
    st["n_corr"], st["best_hypothesis"] = m, -1
    status = 1 if m < n_min else 0
    if not status:
        # 2. hypotheses
        idx = motion_draws(int(p["seed"]), int(p["hypotheses"]), n_min, m)
        r1, r2, b1, b2 = motion_rows(model, corr[idx])  # (nh, n_min, k)
        A = np.stack([r1, r2], 2).reshape(idx.shape[0], k, k)
        b = np.stack([b1, b2], 2).reshape(idx.shape[0], k)
        x, ok = motion_solve(A, b)
        # 3. scoring
        g = motion_hmat(model, x).astype(f32)
        counts = np.zeros(idx.shape[0], np.int64)
        for h0 in range(0, idx.shape[0], 256):
            counts[h0:h0 + 256] = motion_inliers(g[h0:h0 + 256], corr, t).sum(axis=1)
        if not ok.any():
            status = 2
    if status:
        M = np.full(9, _QNAN64)
    else:
        keys = np.where(ok, (counts << 32) | (0xFFFFFFFF - np.arange(idx.shape[0])), -1)
        best = int(np.argmax(keys))
        st["best_hypothesis"], st["ransac_inliers"] = best, counts[best]
        xm = x[best]
        refits = 0
        # 4. refits
        for r in range(int(p["refine"]) + 1):
            inl = motion_inliers(motion_hmat(model, xm).astype(f32), corr, t)
            cnt = int(inl.sum())
            if r == int(p["refine"]) or cnt < n_min:
                break
            An, bn = motion_normal_sums(model, corr, inl)
            xn, okn = motion_solve(An[None], bn[None])
            if not okn[0]:
                break
            xm, refits = xn[0], refits + 1
        st["refits"], st["n_inliers"] = refits, cnt
        # 5. the model in pixel coordinates
        M = motion_to_pixels(model, motion_hmat(model, xm), c_x, c_y, sigma)
    st["status"] = status
    # 6. per pixel
    if status:
        residual = np.full((h, w, 2), _QNAN, f32)
        mask = np.full((h, w), 2, np.uint8)
        reg = None if I1 is None else np.zeros(I1.shape, np.uint8)
        return M, st, mask, residual, reg
    mm = M.astype(f32)
    with np.errstate(all="ignore"):
        mx = (mm[0] * X + mm[1] * Y) + mm[2]
        my = (mm[3] * X + mm[4] * Y) + mm[5]
        wq = (mm[6] * X + mm[7] * Y) + mm[8]
        xw, yw = mx / wq, my / wq
        rx, ry = u - (xw - X), v - (yw - Y)
        close = rx * rx + ry * ry <= f32(p["threshold"]) * f32(p["threshold"])
    residual = np.stack([rx, ry], -1).astype(f32)
    residual = np.where(np.isnan(residual), _QNAN, residual).astype(f32)
    mask = np.where(valid, np.where(close, 0, 1), 2).astype(np.uint8)
    reg = None if I1 is None else _sample_u8(I1, wq, xw, yw)
    return M, st, mask, residual, reg


def _sample_u8(I: np.ndarray, wq: np.ndarray, xw: np.ndarray, yw: np.ndarray) -> np.ndarray:
    """The registered frames' rule: the 8-bit frame I (h, w[, noc]) at (xw, yw) (float32 (h, w)) by the bilinear byte
    rule and its rounding where wq > 0 and the position lies in the frame, else 0."""
    f32 = np.float32
    h, w = wq.shape
    img = I.reshape(h, w, -1).astype(f32)
    with np.errstate(invalid="ignore"):
        ins = (wq > 0) & (xw >= 0) & (xw <= f32(w - 1)) & (yw >= 0) & (yw <= f32(h - 1))
    val = _bilinear_frame(img, np.where(ins, xw, f32(0)), np.where(ins, yw, f32(0)))
    out = (np.fmin(np.fmax(val, f32(0)), f32(255)) + f32(0.5)).astype(np.uint8)
    return np.where(ins[..., None], out, np.uint8(0)).reshape(I.shape)


# ---- stereo ego-motion (ofdis_egomotion_fullres) ---------------------------------------------------------------------
# ofdis_egomotion_params, field for field; the stats are MOTION_STATS_DTYPE
EGO_PARAM_FIELDS = ("step", "fb_check", "alpha", "beta", "edge_diff", "hypotheses", "threshold", "refine", "seed")


def _ego_cam(camera) -> dict:
    cam = {key: np.float32(camera[key]) for key in STEREO_CAMERA_FIELDS}
    cam["fb"] = np.float32(cam["fx"] * cam["baseline"])
    return cam


def ego_pixels(F: np.ndarray, D0: np.ndarray, D1: np.ndarray, cam: dict, edge_diff, valid_fb=None) -> dict:
    """Step 1 of ofdis_egomotion_fullres at every pixel of one pair: F (h, w, 2), D0 and D1 (h, w) float32.  Returns
    float32 arrays xs, ys, d0, d1, s0, s1, X, Y, Z (P), the bool arrays usable0 (d0 known, s0 > 0) and valid (the pixel
    would be a correspondence; valid_fb, the consistency mask == 0, joins it where given)."""
    f32 = np.float32
    h, w = D0.shape
    u, v = F[..., 0], F[..., 1]
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        xs = np.arange(w, dtype=f32)[None, :] + u
        ys = np.arange(h, dtype=f32)[:, None] + v
        inside = (xs >= 0) & (xs <= f32(w - 1)) & (ys >= 0) & (ys <= f32(h - 1))
        d1 = sf_gather_d1(D1[None], xs[None], ys[None], inside[None], edge_diff)[0]
        d1 = np.where(inside, d1, _QNAN).astype(f32)
        s0 = (D0 + cam["doffs"]).astype(f32)
        s1 = (d1 + cam["doffs"]).astype(f32)
        usable0 = _known_disp(D0) & (s0 > 0)
        Z = (cam["fb"] / s0).astype(f32)
        X = (((np.arange(w, dtype=f32)[None, :] - cam["cx"]) * Z) / cam["fx"]).astype(f32)
        Y = (((np.arange(h, dtype=f32)[:, None] - cam["cy"]) * Z) / cam["fy"]).astype(f32)
        valid = usable0 & inside & _known_disp(d1) & (s1 > 0)
    if valid_fb is not None:
        valid &= valid_fb
    return dict(xs=xs, ys=ys, d0=D0, d1=d1, s0=s0, s1=s1, X=X, Y=Y, Z=Z, usable0=usable0, valid=valid)


def ego_q(cam: dict, xs, ys, s1):
    """Q, the t+1 point of observations (xs, ys, s1 = d1 + doffs): scene flow's (X1, Y1, Z1), float32."""
    with np.errstate(all="ignore"):
        Z1 = (cam["fb"] / np.asarray(s1, np.float32)).astype(np.float32)
        X1 = (((np.asarray(xs, np.float32) - cam["cx"]) * Z1) / cam["fx"]).astype(np.float32)
        Y1 = (((np.asarray(ys, np.float32) - cam["cy"]) * Z1) / cam["fy"]).astype(np.float32)
    return X1, Y1, Z1


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def _triad(A, B, C):
    """The triads (e1, e2, n) of point triples A, B, C (..., 3) float64: (..., 3 rows, 3) and whether both lengths are
    > 0."""
    with np.errstate(all="ignore"):
        u, v = B - A, C - A
        L = np.sqrt((u[..., 0] * u[..., 0] + u[..., 1] * u[..., 1]) + u[..., 2] * u[..., 2])
        e1 = u / L[..., None]
        nn = _cross(e1, v)
        Ln = np.sqrt((nn[..., 0] * nn[..., 0] + nn[..., 1] * nn[..., 1]) + nn[..., 2] * nn[..., 2])
        n = nn / Ln[..., None]
        e2 = _cross(n, e1)
    return np.stack([e1, e2, n], -2), (L > 0) & (Ln > 0)


def ego_fit3(P: np.ndarray, Q: np.ndarray):
    """The closed-form rigid fit of ofdis_egomotion_fullres's step 2 from three point pairs P, Q (..., 3, 3) float64:
    returns ([R | t] (..., 12) float64, ok (...,))."""
    E, okp = _triad(P[..., 0, :], P[..., 1, :], P[..., 2, :])
    G, okq = _triad(Q[..., 0, :], Q[..., 1, :], Q[..., 2, :])
    with np.errstate(all="ignore"):
        R = ((G[..., 0, :, None] * E[..., 0, None, :]) + (G[..., 1, :, None] * E[..., 1, None, :])) + \
            (G[..., 2, :, None] * E[..., 2, None, :])
        cP = ((P[..., 0, :] + P[..., 1, :]) + P[..., 2, :]) / 3.0
        cQ = ((Q[..., 0, :] + Q[..., 1, :]) + Q[..., 2, :]) / 3.0
        t = cQ - (((R[..., 0] * cP[..., 0, None]) + (R[..., 1] * cP[..., 1, None])) + (R[..., 2] * cP[..., 2, None]))
    M = np.concatenate([R, t[..., None]], -1).reshape(P.shape[:-2] + (12,))
    return M, okp & okq & np.isfinite(M).all(axis=-1)


def ego_transform(g: np.ndarray, X, Y, Z):
    """P' = g P in float32 for g (..., 12) against points (m,): (X', Y', Z') each (..., m)."""
    g = np.asarray(g, np.float32)[..., None, :]
    with np.errstate(all="ignore"):
        Xp = ((g[..., 0] * X + g[..., 1] * Y) + g[..., 2] * Z) + g[..., 3]
        Yp = ((g[..., 4] * X + g[..., 5] * Y) + g[..., 6] * Z) + g[..., 7]
        Zp = ((g[..., 8] * X + g[..., 9] * Y) + g[..., 10] * Z) + g[..., 11]
    return Xp, Yp, Zp


def ego_inliers(g: np.ndarray, c: np.ndarray, cam: dict, threshold) -> np.ndarray:
    """The inlier test of ofdis_egomotion_fullres, float32: g (..., 12) against the correspondences c (m, 8) (X, Y, Z,
    xs, ys, d1, s1, 0); returns (..., m) bool."""
    f32 = np.float32
    Xp, Yp, Zp = ego_transform(g, c[:, 0], c[:, 1], c[:, 2])
    with np.errstate(all="ignore"):
        ex = (cam["fx"] * Xp + cam["cx"] * Zp) - c[:, 3] * Zp
        ey = (cam["fy"] * Yp + cam["cy"] * Zp) - c[:, 4] * Zp
        ed = cam["fb"] - c[:, 6] * Zp
        tz = f32(threshold) * Zp
        return (Zp > 0) & ((ex * ex + ey * ey) + ed * ed <= tz * tz)


def _chunk_tree(T: np.ndarray) -> np.ndarray:
    """Sums of the rows of T (m, ne) float64 in chunks of 32 from +0.0, then a pairwise tree over the chunk sums padded
    with +0.0 to a power of two."""
    m, ne = T.shape
    nc = (m + 31) // 32
    T = np.concatenate([T, np.zeros((nc * 32 - m, ne))]).reshape(nc, 32, ne)
    v = np.zeros((nc, ne))
    for e in range(32):
        v = v + T[:, e]
    P = 1
    while P < nc:
        P *= 2
    v = np.concatenate([v, np.zeros((P - nc, ne))])
    while v.shape[0] > 1:
        v = v[0::2] + v[1::2]
    return v[0]


def ego_rows(M: np.ndarray, c: np.ndarray, cam: dict):
    """The refit's Jacobian rows J (m, 3, 6) and residuals r (m, 3) (x, y, disparity) of the correspondences c at the
    float64 model M (12,), in the header's expression order."""
    X, Y, Z = (c[:, i].astype(np.float64) for i in range(3))
    Pp = [(((M[4 * i] * X) + (M[4 * i + 1] * Y)) + (M[4 * i + 2] * Z)) + M[4 * i + 3] for i in range(3)]
    fx, fy, cx, cy, fb, doffs = (float(cam[k]) for k in ("fx", "fy", "cx", "cy", "fb", "doffs"))
    zero = np.zeros_like(X)
    with np.errstate(all="ignore"):
        iz = 1.0 / Pp[2]
        u, v = Pp[0] * iz, Pp[1] * iz
        ax = (fx * iz, zero, -((fx * iz) * u))
        ay = (zero, fy * iz, -((fy * iz) * v))
        ad = (zero, zero, -((fb * iz) * iz))
        r = np.stack([((fx * u) + cx) - c[:, 3].astype(np.float64), ((fy * v) + cy) - c[:, 4].astype(np.float64),
                      ((fb * iz) - doffs) - c[:, 5].astype(np.float64)], -1)
        w0, w1, w2 = 2.0 * Pp[0], 2.0 * Pp[1], 2.0 * Pp[2]
        J = np.stack([np.stack([(a[1] * -w2) + (a[2] * w1), (a[0] * w2) + (a[2] * -w0), (a[0] * -w1) + (a[1] * w0),
                                a[0], a[1], a[2]], -1) for a in (ax, ay, ad)], 1)
    return J, r


def ego_normal_sums(M: np.ndarray, c: np.ndarray, inl: np.ndarray, cam: dict):
    """The refit's normal equations (A (6, 6), b (6,)) from the inliers `inl` of c (m, 8) at the model M."""
    J, r = ego_rows(M, c, cam)
    with np.errstate(all="ignore"):
        terms = [((J[:, 0, a] * J[:, 0, b]) + (J[:, 1, a] * J[:, 1, b])) + (J[:, 2, a] * J[:, 2, b])
                 for a in range(6) for b in range(a, 6)]
        terms += [-(((J[:, 0, a] * r[:, 0]) + (J[:, 1, a] * r[:, 1])) + (J[:, 2, a] * r[:, 2])) for a in range(6)]
    T = np.where(inl[:, None], np.stack(terms, -1), 0.0)
    v = _chunk_tree(T)
    A = np.zeros((6, 6))
    e = 0
    for a in range(6):
        for b in range(a, 6):
            A[a, b] = A[b, a] = v[e]
            e += 1
    return A, v[e:]


def ego_update(M: np.ndarray, x: np.ndarray) -> np.ndarray:
    """[R | t] <- [C R | C t + tau] with the Cayley rotation C of omega = x[:3] and tau = x[3:]."""
    w = x[:3]
    q = (w[0] * w[0] + w[1] * w[1]) + w[2] * w[2]
    dg, dn = 1.0 - q, 1.0 + q
    K = ((0.0, -w[2], w[1]), (w[2], 0.0, -w[0]), (-w[1], w[0], 0.0))
    C = [[(((dg if i == j else 0.0) + (2.0 * (w[i] * w[j]))) + (2.0 * K[i][j])) / dn for j in range(3)]
         for i in range(3)]
    Mn = np.zeros(12)
    for i in range(3):
        for j in range(4):
            Mn[4 * i + j] = ((C[i][0] * M[j]) + (C[i][1] * M[4 + j])) + (C[i][2] * M[8 + j])
        Mn[4 * i + 3] = Mn[4 * i + 3] + x[3 + i]
    return Mn


def ego_correspondences(px: dict, step: int) -> np.ndarray:
    """The compacted correspondences (m, 8) float32 (X, Y, Z, xs, ys, d1, s1, 0) of step 1 from ego_pixels' arrays."""
    h, w = px["valid"].shape
    s = int(step)
    ncx, ncy = (w - 1) // s + 1, (h - 1) // s + 1
    cell = np.arange(ncx * ncy)
    cxs = np.minimum((cell % ncx) * s + s // 2, w - 1)
    cys = np.minimum((cell // ncx) * s + s // 2, h - 1)
    sel = px["valid"][cys, cxs]
    cxs, cys = cxs[sel], cys[sel]
    cols = [px[k][cys, cxs] for k in ("X", "Y", "Z", "xs", "ys", "d1", "s1")]
    return np.stack(cols + [np.zeros(cxs.shape[0], np.float32)], -1).astype(np.float32)


def _ego_pair(F, B, D0, D1, cam, p):
    f32 = np.float32
    h, w = D0.shape
    fbm = consistency_check(F, B, p["alpha"], p["beta"])[0] == 0 if p["fb_check"] else None
    px = ego_pixels(F, D0, D1, cam, p["edge_diff"], fbm)
    corr = ego_correspondences(px, p["step"])
    m = corr.shape[0]
    st = np.zeros((), MOTION_STATS_DTYPE)
    st["n_corr"], st["best_hypothesis"] = m, -1
    status = 1 if m < 3 else 0
    thr = p["threshold"]
    if not status:
        idx = motion_draws(int(p["seed"]), int(p["hypotheses"]), 3, m)
        c = corr[idx]  # (nh, 3, 8)
        P = c[..., 0:3].astype(np.float64)
        Q = np.stack(ego_q(cam, c[..., 3], c[..., 4], c[..., 6]), -1).astype(np.float64)
        Ms, ok = ego_fit3(P, Q)
        g = Ms.astype(f32)
        counts = np.zeros(idx.shape[0], np.int64)
        for h0 in range(0, idx.shape[0], 256):
            counts[h0:h0 + 256] = ego_inliers(g[h0:h0 + 256], corr, cam, thr).sum(axis=1)
        if not ok.any():
            status = 2
    if status:
        pose = np.full(12, _QNAN64)
    else:
        keys = np.where(ok, (counts << 32) | (0xFFFFFFFF - np.arange(idx.shape[0])), -1)
        best = int(np.argmax(keys))
        st["best_hypothesis"], st["ransac_inliers"] = best, counts[best]
        M = Ms[best]
        refits = 0
        for r in range(int(p["refine"]) + 1):
            inl = ego_inliers(M.astype(f32), corr, cam, thr)
            cnt = int(inl.sum())
            if r == int(p["refine"]) or cnt < 3:
                break
            A, b = ego_normal_sums(M, corr, inl, cam)
            x, okn = motion_solve(A[None], b[None])
            if not okn[0]:
                break
            M, refits = ego_update(M, x[0]), refits + 1
        st["refits"], st["n_inliers"] = refits, cnt
        pose = np.where(np.isnan(M), _QNAN64, M)
    st["status"] = status
    # per pixel
    mask = np.full((h, w), 2, np.uint8)
    residual = np.full((h, w, 2), _QNAN, f32)
    objm = np.full((h, w, 3), _QNAN, f32)
    if status:
        return pose, st, mask, residual, objm
    g = pose.astype(f32)
    X, Y, Z = px["X"].ravel(), px["Y"].ravel(), px["Z"].ravel()
    Xp, Yp, Zp = (a.reshape(h, w) for a in ego_transform(g, X, Y, Z))
    with np.errstate(all="ignore"):
        xi = (cam["fx"] * Xp) / Zp + cam["cx"]
        yi = (cam["fy"] * Yp) / Zp + cam["cy"]
        rx = F[..., 0] - (xi - np.arange(w, dtype=f32)[None, :])
        ry = F[..., 1] - (yi - np.arange(h, dtype=f32)[:, None])
    res = np.stack([rx, ry], -1).astype(f32)
    res = np.where(np.isnan(res), _QNAN, res)
    residual = np.where(px["usable0"][..., None], res, _QNAN).astype(f32)
    cflat = np.stack([px[k].ravel() for k in ("X", "Y", "Z", "xs", "ys", "d1", "s1")] +
                     [np.zeros(h * w, f32)], -1).astype(f32)
    inl = ego_inliers(g, cflat, cam, thr).reshape(h, w)
    with np.errstate(invalid="ignore"):
        live = px["valid"] & (Zp > 0)
    mask = np.where(live, np.where(inl, 0, 1), 2).astype(np.uint8)
    X1, Y1, Z1 = ego_q(cam, px["xs"], px["ys"], px["s1"])
    with np.errstate(all="ignore"):
        om = np.stack([X1 - Xp, Y1 - Yp, Z1 - Zp], -1).astype(f32)
    om = np.where(np.isnan(om), _QNAN, om)
    objm = np.where(live[..., None], om, _QNAN).astype(f32)
    return pose, st, mask, residual, objm


def egomotion_params(params) -> dict:
    return {k: params[k] for k in EGO_PARAM_FIELDS}


def egomotion(F: np.ndarray, B: np.ndarray | None, disp0: np.ndarray, disp1: np.ndarray, camera, params):
    """ofdis_egomotion_fullres bit for bit.  F: the forward flows (n, h, w, 2) exactly as ofdis_get_flow_fullres
    returns them, B the partner flows of fb_check (else None); disp0, disp1 (n, h, w) float32 positive disparities
    with NaN for unknown; camera a mapping with STEREO_CAMERA_FIELDS; params a mapping with EGO_PARAM_FIELDS.  Returns
    (pose (n, 3, 4) float64, stats (n,) MOTION_STATS_DTYPE, mask (n, h, w) uint8, residual (n, h, w, 2) and
    object_motion (n, h, w, 3) float32)."""
    p = egomotion_params(params)
    cam = _ego_cam(camera)
    F = np.asarray(F, np.float32)
    n, h, w = F.shape[:3]
    D0 = np.asarray(disp0, np.float32).reshape(n, h, w)
    D1 = np.asarray(disp1, np.float32).reshape(n, h, w)
    out = [_ego_pair(F[k], None if B is None else np.asarray(B[k], np.float32), D0[k], D1[k], cam, p)
           for k in range(n)]
    pose = np.stack([o[0] for o in out]).reshape(n, 3, 4) if n else np.zeros((0, 3, 4))
    stats = np.array([o[1] for o in out], MOTION_STATS_DTYPE).reshape(n)
    return (pose, stats, np.stack([o[2] for o in out]), np.stack([o[3] for o in out]),
            np.stack([o[4] for o in out]))


# ---- monocular relative pose (ofdis_relpose_fullres) -----------------------------------------------------------------
# ofdis_relpose_params, field for field; the stats are MOTION_STATS_DTYPE (status 3: too little parallax)
RELPOSE_PARAM_FIELDS = ("fx", "fy", "cx", "cy", "step", "fb_check", "alpha", "beta", "hypotheses", "threshold",
                        "refine", "min_parallax", "seed")
RELPOSE_JACOBI_SWEEPS = 8


def relpose_null(A: np.ndarray):
    """The full-pivot null vector of ofdis_relpose_fullres's step 2 on a batch of systems A (s, 8, 9) float64: returns
    (e (s, 9) unit vectors, ok (s,))."""
    A = np.array(A, np.float64)
    s = A.shape[0]
    ar = np.arange(s)
    perm = np.tile(np.arange(9), (s, 1))
    ok = np.ones(s, bool)
    with np.errstate(all="ignore"):
        for j in range(8):
            best = np.full(s, -1.0)
            pr = np.full(s, j)
            pc = np.full(s, j)
            for i in range(j, 8):
                for c in range(j, 9):
                    a = np.abs(A[:, i, c])
                    upd = a > best
                    best = np.where(upd, a, best)
                    pr = np.where(upd, i, pr)
                    pc = np.where(upd, c, pc)
            ok &= best > 0
            rj, rp = A[ar, j].copy(), A[ar, pr].copy()
            A[ar, pr], A[ar, j] = rj, rp
            cj, cp = A[ar, :, j].copy(), A[ar, :, pc].copy()
            A[ar, :, pc], A[ar, :, j] = cj, cp
            qj, qp = perm[ar, j].copy(), perm[ar, pc].copy()
            perm[ar, pc], perm[ar, j] = qj, qp
            for i in range(j + 1, 8):
                f = A[:, i, j] / A[:, j, j]
                A[:, i, j + 1:] = A[:, i, j + 1:] - f[:, None] * A[:, j, j + 1:]
        y = np.zeros((s, 9))
        y[:, 8] = 1.0
        for i in range(7, -1, -1):
            v = -A[:, i, 8]
            for c in range(i + 1, 8):
                v = v - A[:, i, c] * y[:, c]
            y[:, i] = v / A[:, i, i]
        e = np.zeros((s, 9))
        e[ar[:, None], perm] = y
        n2 = np.zeros(s)
        for d in range(9):
            n2 = n2 + e[:, d] * e[:, d]
        e = e / np.sqrt(n2)[:, None]
    return e, ok & np.isfinite(e).all(axis=1)


def relpose_fmat(E: np.ndarray, fx, fy, cx, cy) -> np.ndarray:
    """F = K^-T E K^-1 of E (..., 9) float64 in the header's expression order, rounded to float32."""
    ifx, ify = 1.0 / float(np.float32(fx)), 1.0 / float(np.float32(fy))
    ux, uy = -(float(np.float32(cx)) * ifx), -(float(np.float32(cy)) * ify)
    E = np.asarray(E, np.float64)
    G = [None] * 9
    for i in range(3):
        G[3 * i] = E[..., 3 * i] * ifx
        G[3 * i + 1] = E[..., 3 * i + 1] * ify
        G[3 * i + 2] = ((E[..., 3 * i] * ux) + (E[..., 3 * i + 1] * uy)) + E[..., 3 * i + 2]
    F = [None] * 9
    for j in range(3):
        F[j] = ifx * G[j]
        F[3 + j] = ify * G[3 + j]
        F[6 + j] = ((ux * G[j]) + (uy * G[3 + j])) + G[6 + j]
    return np.stack(F, -1).astype(np.float32)


def relpose_sampson(g: np.ndarray, c: np.ndarray, threshold):
    """Step 3's test, float32: g (..., 9) against pixel correspondences c (m, 4) (px, py, xs, ys).  Returns (inlier,
    e, den), each (..., m)."""
    f32 = np.float32
    g = np.asarray(g, f32)[..., None, :]
    x, y, xs, ys = c[:, 0], c[:, 1], c[:, 2], c[:, 3]
    with np.errstate(all="ignore"):
        a0 = (g[..., 0] * x + g[..., 1] * y) + g[..., 2]
        a1 = (g[..., 3] * x + g[..., 4] * y) + g[..., 5]
        a2 = (g[..., 6] * x + g[..., 7] * y) + g[..., 8]
        b0 = (g[..., 0] * xs + g[..., 3] * ys) + g[..., 6]
        b1 = (g[..., 1] * xs + g[..., 4] * ys) + g[..., 7]
        e = (xs * a0 + ys * a1) + a2
        den = (a0 * a0 + a1 * a1) + (b0 * b0 + b1 * b1)
        t = f32(threshold)
        return e * e <= (t * t) * den, e, den


def _relpose_norm(c: np.ndarray, p: dict):
    f32 = np.float32
    fx, fy, cx, cy = (f32(p[k]) for k in ("fx", "fy", "cx", "cy"))
    return (c[..., 0] - cx) / fx, (c[..., 1] - cy) / fy, (c[..., 2] - cx) / fx, (c[..., 3] - cy) / fy


def _unit3(a):
    """a / |a| in float64 scalars: a zero or non-finite a gives NaN or inf as on the device."""
    a = [np.float64(v) for v in a]
    with np.errstate(all="ignore"):
        L = np.sqrt((a[0] * a[0] + a[1] * a[1]) + a[2] * a[2])
        return [a[0] / L, a[1] / L, a[2] / L]


def relpose_decompose(E) -> tuple:
    """The four (R (9,), t (3,)) candidates of E (9,) float64 by step 4's Jacobi decomposition, in the header's
    order (R1, u3), (R1, -u3), (R2, u3), (R2, -u3)."""
    E = [float(v) for v in E]
    S = [[((E[i] * E[j]) + (E[3 + i] * E[3 + j])) + (E[6 + i] * E[6 + j]) for j in range(3)] for i in range(3)]
    V = [[1.0 if i == j else 0.0 for j in range(3)] for i in range(3)]
    with np.errstate(all="ignore"):
        for _ in range(RELPOSE_JACOBI_SWEEPS):
            for p, q in ((0, 1), (0, 2), (1, 2)):
                apq = S[p][q]
                if apq == 0.0:
                    continue
                th = (S[q][q] - S[p][p]) / (2.0 * apq)
                t = 1.0 / (abs(th) + _sqrt(th * th + 1.0))
                if th < 0.0:
                    t = -t
                c = 1.0 / _sqrt(t * t + 1.0)
                s = t * c
                for M, rows in ((S, False), (S, True), (V, False)):
                    for r in range(3):
                        if rows:
                            a, b = M[p][r], M[q][r]
                            M[p][r], M[q][r] = c * a - s * b, s * a + c * b
                        else:
                            a, b = M[r][p], M[r][q]
                            M[r][p], M[r][q] = c * a - s * b, s * a + c * b
    d0, d1, d2 = S[0][0], S[1][1], S[2][2]
    i1 = (2 if d2 > d1 else 1) if d1 > d0 else (2 if d2 > d0 else 0)
    i2 = (2 if d2 > d1 else 1) if i1 == 0 else (2 if d2 > d0 else 0) if i1 == 1 else (1 if d1 > d0 else 0)
    v1 = _unit3([V[i][i1] for i in range(3)])
    v2 = [V[i][i2] for i in range(3)]
    v3 = _unit3(_vcross(v1, v2))
    v2 = _vcross(v3, v1)
    u1 = _unit3([((E[3 * i] * v1[0]) + (E[3 * i + 1] * v1[1])) + (E[3 * i + 2] * v1[2]) for i in range(3)])
    w = [((E[3 * i] * v2[0]) + (E[3 * i + 1] * v2[1])) + (E[3 * i + 2] * v2[2]) for i in range(3)]
    u3 = _unit3(_vcross(u1, w))
    u2 = _vcross(u3, u1)
    R1 = np.array([((u2[i] * v1[j]) - (u1[i] * v2[j])) + (u3[i] * v3[j]) for i in range(3) for j in range(3)])
    R2 = np.array([((u1[i] * v2[j]) - (u2[i] * v1[j])) + (u3[i] * v3[j]) for i in range(3) for j in range(3)])
    t = np.array(u3)
    return [(R1, t), (R1, -t), (R2, t), (R2, -t)]


def _sqrt(v: float) -> float:
    return math.sqrt(v) if v >= 0 else float("nan")


def _relpose_rot(R, x, y):
    return [((R[3 * i] * x) + (R[3 * i + 1] * y)) + R[3 * i + 2] for i in range(3)]


def _vcross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _vdot(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def relpose_front(R, t, x, y, xp, yp) -> np.ndarray:
    """Step 4's cheirality test in float64 of (R (9,), t (3,)) on normalized correspondences (arrays)."""
    Y = _relpose_rot(R, x, y)
    r1 = [xp, yp, np.ones_like(xp)]
    tt = [np.full_like(x, t[i]) for i in range(3)]
    with np.errstate(all="ignore"):
        c1, c2 = _vcross(r1, Y), _vcross(r1, tt)
        lam = -_vdot(c1, c2) / _vdot(c1, c1)
        return (lam > 0) & (lam * Y[2] + t[2] > 0)


def relpose_refit_terms(R, t, b1, b2, E, x, y, xp, yp, fx, fy) -> np.ndarray:
    """Step 4's accumulators (m, 22) of normalized correspondences (float64 arrays) at the model (R, t)."""
    ifx, ify = 1.0 / fx, 1.0 / fy
    one = np.ones_like(x)
    with np.errstate(all="ignore"):
        Y = _relpose_rot(R, x, y)
        a = [((E[3 * q] * x) + (E[3 * q + 1] * y)) + E[3 * q + 2] for q in range(3)]
        b = [((E[q] * xp) + (E[3 + q] * yp)) + E[6 + q] for q in range(3)]
        res = ((xp * a[0]) + (yp * a[1])) + a[2]
        s0, s1, s2, s3 = a[0] * ifx, a[1] * ify, b[0] * ifx, b[1] * ify
        wt = 1.0 / np.sqrt(((s0 * s0 + s1 * s1) + s2 * s2) + s3 * s3)
        rr = wt * res
        z = [xp, yp, one]
        zt = _vcross(z, [t[0] * one, t[1] * one, t[2] * one])
        gw = _vcross(Y, zt)
        yz = _vcross(Y, z)
        J = [wt * (2.0 * gw[q]) for q in range(3)]
        J += [wt * _vdot([b1[0] * one, b1[1] * one, b1[2] * one], yz), wt * _vdot([b2[0] * one, b2[1] * one,
                                                                                     b2[2] * one], yz)]
        terms = [J[p] * J[q] for p in range(5) for q in range(p, 5)] + [-(J[p] * rr) for p in range(5)]
        dx, dy = fx * (xp - Y[0] / Y[2]), fy * (yp - Y[1] / Y[2])
        terms.append(np.sqrt(dx * dx + dy * dy))
        Rw = [sum_(((2.0 * (t[i] * t[k])) - (1.0 if i == k else 0.0)) * R[3 * k + j] for k in range(3))
              for i in range(3) for j in range(3)]
        Yw = _relpose_rot(Rw, x, y)
        wx, wy = fx * (xp - Yw[0] / Yw[2]), fy * (yp - Yw[1] / Yw[2])
        terms.append(np.sqrt(wx * wx + wy * wy))
    return np.stack(terms, -1)


def sum_(terms) -> float:
    """Left-to-right float64 sum from +0.0."""
    v = 0.0
    for x in terms:
        v = v + x
    return v


def _relpose_pair(F, B, p):
    f32 = np.float32
    h, w = F.shape[:2]
    s = int(p["step"])
    u, v = F[..., 0], F[..., 1]
    X = np.arange(w, dtype=f32)[None, :]
    Y = np.arange(h, dtype=f32)[:, None]
    with np.errstate(invalid="ignore", over="ignore"):
        xs, ys = X + u, Y + v
        lim = f32(MOTION_UNKNOWN_THRESH)
        valid = (np.abs(u) <= lim) & (np.abs(v) <= lim) & (xs >= 0) & (xs <= f32(w - 1)) & (ys >= 0) & \
            (ys <= f32(h - 1))
    if p["fb_check"]:
        valid &= consistency_check(F, B, p["alpha"], p["beta"])[0] == 0
    ncx, ncy = (w - 1) // s + 1, (h - 1) // s + 1
    cell = np.arange(ncx * ncy)
    cxs = np.minimum((cell % ncx) * s + s // 2, w - 1)
    cys = np.minimum((cell // ncx) * s + s // 2, h - 1)
    sel = valid[cys, cxs]
    cxs, cys = cxs[sel], cys[sel]
    corr = np.stack([cxs.astype(f32), cys.astype(f32), xs[cys, cxs], ys[cys, cxs]], -1).astype(f32)
    m = corr.shape[0]
    thr = p["threshold"]
    fx, fy = float(f32(p["fx"])), float(f32(p["fy"]))
    st = np.zeros((), MOTION_STATS_DTYPE)
    st["n_corr"], st["best_hypothesis"] = m, -1
    status = 1 if m < 8 else 0
    nx, ny, nxp, nyp = (a.astype(np.float64) for a in _relpose_norm(corr, p))
    if not status:
        idx = motion_draws(int(p["seed"]), int(p["hypotheses"]), 8, m)
        x, y, xp, yp = nx[idx], ny[idx], nxp[idx], nyp[idx]
        A = np.stack([xp * x, xp * y, xp, yp * x, yp * y, yp, x, y, np.ones_like(x)], -1)
        Es, ok = relpose_null(A)
        g = relpose_fmat(Es, p["fx"], p["fy"], p["cx"], p["cy"])
        counts = np.zeros(idx.shape[0], np.int64)
        for h0 in range(0, idx.shape[0], 256):
            counts[h0:h0 + 256] = relpose_sampson(g[h0:h0 + 256], corr, thr)[0].sum(axis=1)
        if not ok.any():
            status = 2
    pose = np.full(12, _QNAN64)
    if not status:
        keys = np.where(ok, (counts << 32) | (0xFFFFFFFF - np.arange(idx.shape[0])), -1)
        best = int(np.argmax(keys))
        st["best_hypothesis"], st["ransac_inliers"] = best, counts[best]
        inl = relpose_sampson(g[best], corr, thr)[0]
        cands = relpose_decompose(Es[best])
        votes = [int(relpose_front(Rc, tc, nx[inl], ny[inl], nxp[inl], nyp[inl]).sum()) for Rc, tc in cands]
        R, t = cands[int(np.argmax(votes))]
        R, t = [float(v) for v in R], [float(v) for v in t]
        refits = 0
        for r in range(int(p["refine"]) + 1):
            E = [(-(t[2] * R[3 + j])) + (t[1] * R[6 + j]) for j in range(3)] + \
                [(t[2] * R[j]) - (t[0] * R[6 + j]) for j in range(3)] + \
                [(-(t[1] * R[j])) + (t[0] * R[3 + j]) for j in range(3)]
            gm = relpose_fmat(np.array(E), p["fx"], p["fy"], p["cx"], p["cy"])
            a = min(range(3), key=lambda i: (abs(t[i]), i))
            ea = [1.0 if i == a else 0.0 for i in range(3)]
            b1 = _unit3(_vcross(t, ea))
            b2 = _vcross(t, b1)
            inl = relpose_sampson(gm, corr, thr)[0]
            cnt = int(inl.sum())
            T = relpose_refit_terms(R, t, b1, b2, E, nx, ny, nxp, nyp, fx, fy)
            v = _chunk_tree(np.where(inl[:, None], T, 0.0))
            if r == int(p["refine"]) or cnt < 8:
                break
            An = np.zeros((5, 5))
            e = 0
            for a_ in range(5):
                for b_ in range(a_, 5):
                    An[a_, b_] = An[b_, a_] = v[e]
                    e += 1
            xs_, okn = motion_solve(An[None], v[None, 15:20])
            if not okn[0]:
                break
            d = xs_[0]
            Rm = ego_update(np.array([R[0], R[1], R[2], 0.0, R[3], R[4], R[5], 0.0, R[6], R[7], R[8], 0.0]),
                            np.array([d[0], d[1], d[2], 0.0, 0.0, 0.0]))
            R = [float(Rm[4 * i + j]) for i in range(3) for j in range(3)]
            t = _unit3([(t[i] + d[3] * b1[i]) + d[4] * b2[i] for i in range(3)])
            refits += 1
        st["refits"], st["n_inliers"] = refits, cnt
        with np.errstate(all="ignore"):
            parallax = (v[21] if v[21] < v[20] else v[20]) / np.float64(cnt)
        status = 0 if parallax >= float(f32(p["min_parallax"])) else 3
        if not status:
            P = np.array([R[0], R[1], R[2], t[0], R[3], R[4], R[5], t[1], R[6], R[7], R[8], t[2]])
            pose = np.where(np.isnan(P), _QNAN64, P)
    st["status"] = status
    mask = np.full((h, w), 2, np.uint8)
    samp = np.full((h, w), _QNAN, f32)
    depth = np.full((h, w), _QNAN, f32)
    if status:
        return pose, st, mask, samp, depth
    cpx = np.stack([np.broadcast_to(X, (h, w)), np.broadcast_to(Y, (h, w)), xs, ys], -1).reshape(-1, 4).astype(f32)
    inl, e, den = (a.reshape(h, w) for a in relpose_sampson(gm, cpx, thr))
    mask = np.where(valid, np.where(inl, 0, 1), 2).astype(np.uint8)
    with np.errstate(all="ignore"):
        sq = np.sqrt((e * e) / den).astype(f32)
        g32 = pose.astype(f32)
        Rf, tf = g32[[0, 1, 2, 4, 5, 6, 8, 9, 10]], g32[[3, 7, 11]]
        x, y, xp, yp = (a.reshape(h, w) for a in _relpose_norm(cpx, p))
        q = [(Rf[3 * i] * x + Rf[3 * i + 1] * y) + Rf[3 * i + 2] for i in range(3)]
        c1 = [yp * q[2] - q[1], q[0] - xp * q[2], xp * q[1] - yp * q[0]]
        c2 = [yp * tf[2] - tf[1], tf[0] - xp * tf[2], xp * tf[1] - yp * tf[0]]
        lam = -((c1[0] * c2[0] + c1[1] * c2[1]) + c1[2] * c2[2]) / ((c1[0] * c1[0] + c1[1] * c1[1]) + c1[2] * c1[2])
        front = (lam > 0) & (lam * q[2] + tf[2] > 0)
    samp = np.where(valid, np.where(np.isnan(sq), _QNAN, sq), _QNAN).astype(f32)
    depth = np.where(valid & front, lam, _QNAN).astype(f32)
    return pose, st, mask, samp, depth


def relpose_params(params) -> dict:
    return {k: params[k] for k in RELPOSE_PARAM_FIELDS}


def relpose(F: np.ndarray, B: np.ndarray | None, params):
    """ofdis_relpose_fullres bit for bit.  F: the forward flows (n, h, w, 2) exactly as ofdis_get_flow_fullres returns
    them, B the partner flows of fb_check (else None); params a mapping with RELPOSE_PARAM_FIELDS.  Returns (pose
    (n, 3, 4) float64, stats (n,) MOTION_STATS_DTYPE, mask (n, h, w) uint8, sampson and depth (n, h, w) float32)."""
    p = relpose_params(params)
    F = np.asarray(F, np.float32)
    n, h, w = F.shape[:3]
    out = [_relpose_pair(F[k], None if B is None else np.asarray(B[k], np.float32), p) for k in range(n)]
    pose = np.stack([o[0] for o in out]).reshape(n, 3, 4) if n else np.zeros((0, 3, 4))
    stats = np.array([o[1] for o in out], MOTION_STATS_DTYPE).reshape(n)
    return (pose, stats, np.stack([o[2] for o in out]), np.stack([o[3] for o in out]),
            np.stack([o[4] for o in out]))


def relpose_errors(rel, gt_rel):
    """The standard monocular metrics of relative poses rel against ground truth gt_rel (n, 3, 4) (camera t to camera
    t+1): the rotation error acos((trace(R_gt^T R) - 1) / 2) in degrees and the angle between the translation
    directions in degrees.  Returns (r_err (n,), t_dir_err (n,)); NaN where a pose is NaN or a translation is zero."""
    rel = np.asarray(rel, np.float64).reshape(-1, 3, 4)
    gt = np.asarray(gt_rel, np.float64).reshape(-1, 3, 4)
    r_err, t_err = [], []
    for P, G in zip(rel, gt):
        c = 0.5 * (np.trace(G[:, :3].T @ P[:, :3]) - 1.0)
        r_err.append(float(np.degrees(np.arccos(np.clip(c, -1.0, 1.0)))) if np.isfinite(c) else np.nan)
        a, b = P[:, 3], G[:, 3]
        with np.errstate(all="ignore"):
            ct = float(a @ b / (np.linalg.norm(a) * np.linalg.norm(b)))
        t_err.append(float(np.degrees(np.arccos(np.clip(ct, -1.0, 1.0)))) if np.isfinite(ct) else np.nan)
    return np.array(r_err), np.array(t_err)


# ---- poses (float64 host helpers, no bit contract) -------------------------------------------------------------------
def _pose44(P) -> np.ndarray:
    T = np.eye(4)
    T[:3, :4] = np.asarray(P, np.float64).reshape(3, 4)
    return T


def chain_poses(rel, scales=None) -> np.ndarray:
    """Camera-to-world poses (n+1, 3, 4) of a clip in KITTI's odometry convention from its relative poses rel (n, 3, 4)
    (camera t to camera t+1, as ofdis_egomotion_fullres returns them): T_0 = I, T_(k+1) = T_k inv([R | t]_k).
    scales: optional (n,) factors of the translations, e.g. ground-truth step lengths for the unit translations of
    ofdis_relpose_fullres."""
    rel = np.asarray(rel, np.float64).reshape(-1, 3, 4)
    T = np.eye(4)
    out = [T[:3].copy()]
    for k, P in enumerate(rel):
        Q = _pose44(P)
        if scales is not None:
            Q[:3, 3] *= float(scales[k])
        T = T @ np.linalg.inv(Q)
        out.append(T[:3].copy())
    return np.stack(out)


def write_kitti_poses(path: str, poses) -> None:
    """KITTI's odometry poses file: one line of the 12 row-major numbers of [R | t] per frame (%.17g)."""
    with open(path, "w") as f:
        for P in np.asarray(poses, np.float64).reshape(-1, 12):
            f.write(" ".join("%.17g" % v for v in P) + "\n")


def read_kitti_poses(path: str) -> np.ndarray:
    """A KITTI odometry poses file as (n, 3, 4) float64."""
    rows = [list(map(float, line.split())) for line in open(path) if line.strip()]
    if any(len(r) != 12 for r in rows):
        raise ValueError("%s: every line of a KITTI poses file has 12 numbers" % path)
    return np.array(rows, np.float64).reshape(-1, 3, 4)


def pose_errors(rel, gt_abs):
    """Per pair k the relative pose error of rel[k] (camera k to k+1) against ground-truth camera-to-world poses
    gt_abs (n+1, 3, 4), formed as KITTI's devkit forms it: E = inv(inv(G_k) G_(k+1)) inv([R | t]_k), the translation
    error |E_t| in metres and the rotation error acos((trace(E_R) - 1) / 2) in degrees.  Returns (t_err (n,),
    r_err (n,))."""
    rel = np.asarray(rel, np.float64).reshape(-1, 3, 4)
    G = np.asarray(gt_abs, np.float64).reshape(-1, 3, 4)
    t_err, r_err = [], []
    for k, P in enumerate(rel):
        d_gt = np.linalg.inv(_pose44(G[k])) @ _pose44(G[k + 1])
        d_est = np.linalg.inv(_pose44(P))
        E = np.linalg.inv(d_gt) @ d_est
        t_err.append(float(np.linalg.norm(E[:3, 3])))
        c = min(1.0, max(-1.0, 0.5 * (np.trace(E[:3, :3]) - 1.0)))
        r_err.append(float(np.degrees(np.arccos(c))))
    return np.array(t_err), np.array(r_err)


# ---- volumetric fusion (ofdis_fuse_begin / ofdis_fuse_push / ofdis_fuse_extract / ofdis_fuse_render) ----------------
FUSE_PARAM_FIELDS = ("nx", "ny", "nz", "origin", "voxel", "trunc", "max_weight", "color")
# ofdis_fuse_point, field for field (28 bytes)
FUSE_POINT_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4"),
                             ("r", "u1"), ("g", "u1"), ("b", "u1"), ("pad", "u1")])
FUSE_MAX_SAMPLES = 65536
f32 = np.float32


def fuse_new_volume(params) -> dict:
    """The volume of ofdis_fuse_begin: T and W float32 (nz, ny, nx) of +0 and, with colour, C uint8 (nz, ny, nx, 3)."""
    shape = (int(params["nz"]), int(params["ny"]), int(params["nx"]))
    return {"T": np.zeros(shape, f32), "W": np.zeros(shape, f32),
            "C": np.zeros(shape + (3,), np.uint8) if params["color"] else None}


def fuse_world_to_camera(P) -> np.ndarray:
    """g of ofdis_fuse_push: [R^T | -R^T t] of a camera-to-world pose, formed in float64 and rounded to float32 (12,)."""
    p = np.asarray(P, np.float64).reshape(12)
    g = np.empty(12, np.float64)
    for r in range(3):
        g[4 * r:4 * r + 3] = p[r], p[4 + r], p[8 + r]
        g[4 * r + 3] = -(((p[r] * p[3]) + (p[4 + r] * p[7])) + (p[8 + r] * p[11]))
    return g.astype(f32)


def _fuse_axes(params):
    o = [f32(v) for v in params["origin"]]
    vox = f32(params["voxel"])
    return [o[e] + np.arange(int(params[k]), dtype=np.float64).astype(f32) * vox
            for e, k in enumerate(("nx", "ny", "nz"))]


def fuse_integrate(vol: dict, params, disp, poses, camera, max_depth=np.inf, frames=None, weights=None) -> dict:
    """Restates ofdis_fuse_push on vol (fuse_new_volume's dict), in place: disp (n, H, W) float32 positive disparities
    (NaN unknown), poses (n, 3, 4) camera-to-world float64, frames (n, H, W[, 3]) uint8 when the volume keeps colour.
    With weights (n, H, W) float32 it restates ofdis_fuse_push_weighted: an observation counts with its pixel's weight
    c in place of 1, and only where 0 < c <= FLT_MAX."""
    disp = np.asarray(disp, f32).reshape((-1,) + np.shape(disp)[-2:])
    n, H, W = disp.shape
    poses = np.asarray(poses, np.float64).reshape(n, 12)
    cam = {k: f32(camera[k]) for k in STEREO_CAMERA_FIELDS}
    fb = f32(cam["fx"] * cam["baseline"])
    mu, maxw, maxd = f32(params["trunc"]), f32(params["max_weight"]), f32(max_depth)
    xa, ya, za = _fuse_axes(params)
    Z, Y, X = np.meshgrid(za, ya, xa, indexing="ij")
    T, Wt, C = vol["T"], vol["W"], vol["C"]
    one, half = f32(1), f32(0.5)
    for k in range(n):
        q = fuse_world_to_camera(poses[k])
        with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
            Zc = ((q[8] * X + q[9] * Y) + q[10] * Z) + q[11]
            Xc = ((q[0] * X + q[1] * Y) + q[2] * Z) + q[3]
            Yc = ((q[4] * X + q[5] * Y) + q[6] * Z) + q[7]
            ok = Zc > 0
            Zs = np.where(ok, Zc, one)
            uu = ((cam["fx"] * Xc) / Zs + cam["cx"]) + half
            vv = ((cam["fy"] * Yc) / Zs + cam["cy"]) + half
            ok &= (uu >= 0) & (uu < f32(W)) & (vv >= 0) & (vv < f32(H))
            px = np.where(ok, np.floor(np.where(ok, uu, 0)), 0).astype(np.int64)
            py = np.where(ok, np.floor(np.where(ok, vv, 0)), 0).astype(np.int64)
            d = disp[k][py, px]
            s = d + cam["doffs"]
            ok &= (d >= 0) & (d <= f32(1e9)) & (s > 0)
            z = fb / np.where(ok, s, one)
            ok &= ~(z > maxd)
            sdf = z - Zc
            ok &= ~(sdf < -mu)
            f = np.minimum(one, sdf / mu)
            if weights is None:
                c, fc = one, f
            else:
                c = np.asarray(weights[k], f32).reshape(H, W)[py, px]
                ok &= (c > 0) & (c <= np.finfo(f32).max)
                fc = f * c
        with np.errstate(all="ignore"):  # where a weight skips, W1 may be 0 or NaN
            W1 = Wt + c
            Tn = (T * Wt + fc) / W1
        if C is not None:
            fr = np.asarray(frames[k], np.uint8).reshape(H, W, -1)
            obs = fr[py, px] if fr.shape[-1] == 3 else np.repeat(fr[py, px], 3, -1)
            with np.errstate(all="ignore"):
                obs = obs.astype(f32) if weights is None else obs.astype(f32) * c[..., None]
                cn = np.floor((C.astype(f32) * Wt[..., None] + obs) / W1[..., None] + half)
            C[ok] = cn[ok].astype(np.uint8)
        T[ok] = Tn[ok]
        Wt[ok] = np.fmin(W1, maxw)[ok]  # fminf: a NaN W becomes max_weight
    return vol


def _fuse_crossings(T, Wt, min_weight):
    """The crossings of ofdis_fuse_extract in its order, as keys voxel * 3 + axis, and the per-voxel test."""
    good = (Wt >= f32(min_weight)) & (np.abs(T) < f32(1))
    pos = T > 0
    parts = []
    for e, ax in ((0, 2), (1, 1), (2, 0)):
        m = np.zeros(T.shape, bool)
        a = [slice(None)] * 3
        b = [slice(None)] * 3
        a[ax], b[ax] = slice(0, -1), slice(1, None)
        m[tuple(a)] = good[tuple(a)] & good[tuple(b)] & (pos[tuple(a)] != pos[tuple(b)])
        parts.append(np.flatnonzero(m) * 3 + e)
    return np.sort(np.concatenate(parts)), good


def fuse_extract(vol: dict, params, min_weight) -> np.ndarray:
    """Restates ofdis_fuse_extract: every zero crossing of vol as a FUSE_POINT_DTYPE array, in the header's order."""
    T, Wt, C = vol["T"], vol["W"], vol["C"]
    nz, ny, nx = T.shape
    idx, _ = _fuse_crossings(T, Wt, min_weight)
    a, e = idx // 3, idx % 3
    i, j, k = a % nx, (a // nx) % ny, a // (nx * ny)
    step = np.array([1, nx, nx * ny])[e]
    Tf = T.ravel()
    Ta, Tb = Tf[a], Tf[a + step]
    with np.errstate(invalid="ignore", divide="ignore"):
        t = Ta / (Ta - Tb)
        gx = T[k, j, np.minimum(i + 1, nx - 1)] - T[k, j, np.maximum(i - 1, 0)]
        gy = T[k, np.minimum(j + 1, ny - 1), i] - T[k, np.maximum(j - 1, 0), i]
        gz = T[np.minimum(k + 1, nz - 1), j, i] - T[np.maximum(k - 1, 0), j, i]
        L = np.sqrt((gx * gx + gy * gy) + gz * gz)
        nrm = [np.where(L > 0, g / np.where(L > 0, L, f32(1)), _QNAN).astype(f32) for g in (gx, gy, gz)]
    xa, ya, za = _fuse_axes(params)
    P = [xa[i], ya[j], za[k]]
    dt = t * f32(params["voxel"])
    out = np.zeros(len(idx), FUSE_POINT_DTYPE)
    for c, name in enumerate(("x", "y", "z")):
        out[name] = np.where(e == c, P[c] + dt, P[c])
    for c, name in enumerate(("nx", "ny", "nz")):
        out[name] = nrm[c]
    if C is not None:
        src = np.where(t < f32(0.5), a, a + step)
        Cf = C.reshape(-1, 3)
        out["r"], out["g"], out["b"] = Cf[src, 0], Cf[src, 1], Cf[src, 2]
    return out


def fuse_render(vol: dict, params, poses, camera, z_near, z_far, step, min_weight, width: int, height: int):
    """Restates ofdis_fuse_render: depth (n, height, width) float32, qNaN where no ray crosses the surface."""
    poses = np.asarray(poses, np.float64).reshape(-1, 12)
    n = poses.shape[0]
    cam = {k: f32(camera[k]) for k in STEREO_CAMERA_FIELDS}
    T, Wt = vol["T"].ravel(), vol["W"].ravel()
    nz, ny, nx = vol["T"].shape
    o = [f32(v) for v in params["origin"]]
    vox, mw = f32(params["voxel"]), f32(min_weight)
    zn, zf, st = f32(z_near), f32(z_far), f32(step)
    y, x = np.mgrid[0:height, 0:width]
    r0 = (x.astype(f32) - cam["cx"]) / cam["fx"]
    r1 = (y.astype(f32) - cam["cy"]) / cam["fy"]
    p = poses.astype(f32)[:, :, None, None]
    depth = np.full((n, height, width), _QNAN, f32)
    done = np.zeros((n, height, width), bool)
    prev = np.zeros((n, height, width), bool)
    Tp = np.zeros((n, height, width), f32)
    Zp, one = f32(0), f32(1)
    for s in range(FUSE_MAX_SAMPLES + 1):
        Zs = zn + f32(s) * st
        if not Zs <= zf or done.all():
            break
        cx, cy = r0 * Zs, r1 * Zs
        known = np.ones((n, height, width), bool)
        i0, fr = [], []
        with np.errstate(invalid="ignore", over="ignore"):
            for e, dim in enumerate((nx, ny, nz)):
                Pw = ((p[:, 4 * e] * cx + p[:, 4 * e + 1] * cy) + p[:, 4 * e + 2] * Zs) + p[:, 4 * e + 3]
                q = (Pw - o[e]) / vox
                fl = np.floor(q)
                known &= (fl >= 0) & (fl <= f32(dim - 2))
                i0.append(np.where(known, fl, 0).astype(np.int64))
                fr.append((q - fl).astype(f32))
        i0 = [np.where(known, v, 0) for v in i0]
        base = (i0[2] * ny + i0[1]) * nx + i0[0]
        offs = (0, 1, nx, nx + 1, nx * ny, nx * ny + 1, nx * ny + nx, nx * ny + nx + 1)
        corner = [np.minimum(base + off, T.size - 1) for off in offs]  # clipped where the sample is unknown anyway
        for ci in corner:
            known &= Wt[ci] >= mw
        c = [T[ci] for ci in corner]
        gx, gy, gz = one - fr[0], one - fr[1], one - fr[2]
        x00, x10 = c[0] * gx + c[1] * fr[0], c[2] * gx + c[3] * fr[0]
        x01, x11 = c[4] * gx + c[5] * fr[0], c[6] * gx + c[7] * fr[0]
        Ts = (x00 * gy + x10 * fr[1]) * gz + (x01 * gy + x11 * fr[1]) * fr[2]
        hit = ~done & known & prev & (Tp > 0) & (Ts <= 0)
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            depth = np.where(hit, Zp + st * (Tp / (Tp - Ts)), depth).astype(f32)
        done |= hit
        prev = known
        Tp = Ts
        Zp = Zs
    return depth


def write_fused_ply(path: str, pts) -> None:
    """The fused points (FUSE_POINT_DTYPE) as a binary little-endian PLY: x y z nx ny nz float, red green blue uchar --
    the file of the batch command's --fuse."""
    pts = np.asarray(pts, FUSE_POINT_DTYPE)
    rec = np.empty(len(pts), [("p", "<f4", (6,)), ("c", "u1", (3,))])
    rec["p"] = np.stack([pts[k] for k in ("x", "y", "z", "nx", "ny", "nz")], -1) if len(pts) else np.zeros((0, 6))
    rec["c"] = np.stack([pts[k] for k in ("r", "g", "b")], -1) if len(pts) else np.zeros((0, 3))
    with open(path, "wb") as f:
        f.write(("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\n"
                 "property float z\nproperty float nx\nproperty float ny\nproperty float nz\nproperty uchar red\n"
                 "property uchar green\nproperty uchar blue\nend_header\n" % len(pts)).encode())
        f.write(rec.tobytes())


# ---- marching cubes of the fused volume (ofdis_fuse_mesh) -------------------------------------------------------------
def fuse_mc_edge(n: int):
    """Cube edge n = 4*axis + r of the header: (lower corner q, axis); q is r with a 0 bit inserted at bit `axis`."""
    axis, r = n >> 2, n & 3
    return (r & ((1 << axis) - 1)) | ((r >> axis) << (axis + 1)), axis


def _mc_loops(case: int):
    """The oriented loops of one case: lists of edge numbers, each starting at its lowest edge."""
    pos = [(case >> q) & 1 for q in range(8)]
    xyz = [np.array([q & 1, (q >> 1) & 1, q >> 2], float) for q in range(8)]
    edges = [fuse_mc_edge(n) for n in range(12)]
    mid = [(xyz[q] + xyz[q | (1 << ax)]) / 2 for q, ax in edges]
    nxt = {}
    for f in range(3):
        u, v = [a for a in range(3) if a != f]
        for side in (0, 1):
            nf = np.zeros(3)
            nf[f] = 1.0 if side else -1.0
            ring = [(side << f) | (a << u) | (b << v) for a, b in ((0, 0), (1, 0), (1, 1), (0, 1))]
            # the face edge between ring[m] and ring[m + 1]
            fe = []
            for m in range(4):
                a, b = ring[m], ring[(m + 1) % 4]
                fe.append(next(n for n, (q, ax) in enumerate(edges) if {q, q | (1 << ax)} == {a, b}))
            s = [pos[c] for c in ring]
            cross = [m for m in range(4) if s[m] != s[(m + 1) % 4]]
            if not cross:
                continue
            if len(cross) == 4:
                # ambiguous: a segment cuts off each T > 0 corner (its two face edges: m - 1 and m)
                segs = [((m - 1) % 4, m, xyz[ring[m]] - (xyz[ring[0]] + xyz[ring[2]]) / 2) for m in range(4) if s[m]]
            else:
                p = np.mean([xyz[c] for c in ring if pos[c]], 0) - np.mean([xyz[c] for c in ring if not pos[c]], 0)
                segs = [(cross[0], cross[1], p)]
            for ma, mb, p in segs:
                a, b = fe[ma], fe[mb]
                # with the patch's normal towards T > 0, its boundary runs along p x nf on this face
                if np.dot(mid[b] - mid[a], np.cross(p, nf)) < 0:
                    a, b = b, a
                assert a not in nxt
                nxt[a] = b
    loops, seen = [], set()
    for n in sorted(nxt):
        if n in seen:
            continue
        loop = [n]
        while nxt[loop[-1]] != n:
            loop.append(nxt[loop[-1]])
        seen.update(loop)
        loops.append(loop)
    return loops


def _mc_triangulations(lo: int, hi: int):
    """Triangulations of the polygon lo..hi (loop positions) in the header's enumeration: the triangle on side
    (lo, hi) with apex k ascending, then the polygon lo..k, then k..hi."""
    if hi - lo < 2:
        yield []
        return
    for k in range(lo + 1, hi):
        for left in _mc_triangulations(lo, k):
            for right in _mc_triangulations(k, hi):
                yield [(lo, k, hi)] + left + right


def _mc_faces(n: int):
    q, ax = fuse_mc_edge(n)
    return {(f, (q >> f) & 1) for f in range(3) if f != ax}


@functools.lru_cache(maxsize=None)
def _mc_table_cached() -> bytes:
    tab = np.full((256, 16), 255, np.uint8)
    for case in range(256):
        tris = []
        for loop in _mc_loops(case):
            L = len(loop)
            for tri in _mc_triangulations(0, L - 1):
                sides = {tuple(sorted((t[a], t[b]))) for t in tri for a, b in ((0, 1), (1, 2), (0, 2))}
                diag = [(a, b) for a, b in sides if b - a not in (1, L - 1)]
                if all(not (_mc_faces(loop[a]) & _mc_faces(loop[b])) for a, b in diag):
                    tris += [[loop[a] for a in t] for t in tri]
                    break
            else:
                raise AssertionError("case %d: a loop without a valid triangulation" % case)
        tab[case, 0] = len(tris)
        tab[case, 1:1 + 3 * len(tris)] = np.asarray(tris, np.uint8).ravel()
    return tab.tobytes()


def fuse_mc_table() -> np.ndarray:
    """The marching-cubes table of ofdis_fuse_mesh, generated from the header's rules: (256, 16) uint8, row = case,
    [0] the triangles, [1 + 3t + s] the edge of triangle t's vertex s, 255 past the last."""
    return np.frombuffer(_mc_table_cached(), np.uint8).reshape(256, 16).copy()


def fuse_mesh(vol: dict, params, min_weight):
    """Restates ofdis_fuse_mesh: (points, faces) with points = fuse_extract(vol, params, min_weight) and faces (F, 3)
    uint32 vertex indices, meshed cubes in ascending voxel index of corner 0 and each cube's triangles in table order."""
    pts = fuse_extract(vol, params, min_weight)
    T = vol["T"]
    nz, ny, nx = T.shape
    idx, good = _fuse_crossings(T, vol["W"], min_weight)
    pos = T > 0
    # the vertex of crossing (voxel a, axis e) is its position in fuse_extract's order
    key = np.full(T.size * 3, -1, np.int64)
    key[idx] = np.arange(len(idx))
    if nx < 2 or ny < 2 or nz < 2:
        return pts, np.zeros((0, 3), np.uint32)
    sl = [(slice(dk, nz - 1 + dk), slice(dj, ny - 1 + dj), slice(di, nx - 1 + di))
          for q in range(8) for di, dj, dk in [(q & 1, (q >> 1) & 1, q >> 2)]]
    meshed = np.ones((nz - 1, ny - 1, nx - 1), bool)
    case = np.zeros((nz - 1, ny - 1, nx - 1), np.int64)
    for q in range(8):
        meshed &= good[sl[q]]
        case |= pos[sl[q]].astype(np.int64) << q
    kk, jj, ii = np.nonzero(meshed)  # C order: ascending voxel index
    case = case[kk, jj, ii]
    tab = fuse_mc_table().astype(np.int64)
    ntri = tab[case, 0]
    cube = np.repeat(np.arange(len(case)), ntri)
    t = np.arange(len(cube)) - np.repeat(np.cumsum(ntri) - ntri, ntri)
    a0 = ((kk * ny + jj) * nx + ii)[cube]
    faces = np.empty((len(cube), 3), np.int64)
    for s in range(3):
        edge = tab[case[cube], 1 + 3 * t + s]
        q, e = (edge & 3), edge >> 2
        q = (q & ((1 << e) - 1)) | ((q >> e) << (e + 1))
        aq = a0 + (q & 1) + ((q >> 1) & 1) * nx + (q >> 2) * (nx * ny)
        faces[:, s] = key[aq * 3 + e]
    assert (faces >= 0).all()
    return pts, faces.astype(np.uint32)


def write_fused_mesh_ply(path: str, pts, faces) -> None:
    """The mesh as a binary little-endian PLY: the vertices of write_fused_ply, then `element face F` with
    `property list uchar uint vertex_indices` -- the file of the batch command's --mesh."""
    pts = np.asarray(pts, FUSE_POINT_DTYPE)
    faces = np.asarray(faces, np.uint32).reshape(-1, 3)
    rec = np.empty(len(pts), [("p", "<f4", (6,)), ("c", "u1", (3,))])
    rec["p"] = np.stack([pts[k] for k in ("x", "y", "z", "nx", "ny", "nz")], -1) if len(pts) else np.zeros((0, 6))
    rec["c"] = np.stack([pts[k] for k in ("r", "g", "b")], -1) if len(pts) else np.zeros((0, 3))
    frec = np.empty(len(faces), [("n", "u1"), ("v", "<u4", (3,))])
    frec["n"], frec["v"] = 3, faces
    with open(path, "wb") as f:
        f.write(("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\n"
                 "property float z\nproperty float nx\nproperty float ny\nproperty float nz\nproperty uchar red\n"
                 "property uchar green\nproperty uchar blue\nelement face %d\nproperty list uchar uint vertex_indices\n"
                 "end_header\n" % (len(pts), len(faces))).encode())
        f.write(rec.tobytes())
        f.write(frec.tobytes())


# ---- camera tracking against the volume (ofdis_fuse_track) ------------------------------------------------------------
FUSE_TRACK_PARAM_FIELDS = ("step", "rounds", "min_weight", "max_depth", "huber", "damping", "min_corr", "max_shift",
                           "min_cos", "eps", "integrate")
# ofdis_fuse_track_stats, field for field (32 bytes, 4 of padding after rounds)
FUSE_TRACK_STATS_DTYPE = np.dtype({"names": ["status", "n_corr", "rounds", "cost0", "cost"],
                                   "formats": ["<i4", "<i4", "<i4", "<f8", "<f8"], "offsets": [0, 4, 8, 16, 24],
                                   "itemsize": 32})


def fuse_track_predict(prev, motion) -> np.ndarray:
    """Step 1 of ofdis_fuse_track: T(k-1) inv(M) in the header's float64 order (12,), or T(k-1) when motion is None."""
    P = np.asarray(prev, np.float64).reshape(12)
    if motion is None:
        return P.copy()
    m = np.asarray(motion, np.float64).reshape(12)
    Ri = [[m[4 * c + r] for c in range(3)] for r in range(3)]
    ti = [-(((m[r] * m[3]) + (m[4 + r] * m[7])) + (m[8 + r] * m[11])) for r in range(3)]
    M = np.empty(12)
    for r in range(3):
        for c in range(3):
            M[4 * r + c] = ((P[4 * r] * Ri[0][c]) + (P[4 * r + 1] * Ri[1][c])) + (P[4 * r + 2] * Ri[2][c])
        M[4 * r + 3] = (((P[4 * r] * ti[0]) + (P[4 * r + 1] * ti[1])) + (P[4 * r + 2] * ti[2])) + P[4 * r + 3]
    return M


def fuse_track_cells(vol: dict, params, D: np.ndarray, cam: dict, step: int, min_weight, max_depth, M):
    """Step 2 of ofdis_fuse_track at every cell of the map D (H, W) float32 for the float64 pose M (12,): returns
    (valid (cells,) bool, r (cells,), G (cells, 3) and Pw (cells, 3) float32, meaningful where valid)."""
    g = np.asarray(M, np.float64).reshape(12).astype(f32)
    H, W = D.shape
    s = int(step)
    ncx, ncy = (W - 1) // s + 1, (H - 1) // s + 1
    cell = np.arange(ncx * ncy)
    px = np.minimum((cell % ncx) * s + s // 2, W - 1)
    py = np.minimum((cell // ncx) * s + s // 2, H - 1)
    T, Wt = vol["T"].ravel(), vol["W"].ravel()
    nz, ny, nx = vol["T"].shape
    o = [f32(v) for v in params["origin"]]
    vox = f32(params["voxel"])
    d = D[py, px]
    with np.errstate(all="ignore"):
        sd = d + cam["doffs"]
        ok = (d >= 0) & (d <= f32(1e9)) & (sd > 0)
        Z = cam["fb"] / sd
        ok &= Z <= f32(max_depth)
        X = ((px.astype(f32) - cam["cx"]) * Z) / cam["fx"]
        Y = ((py.astype(f32) - cam["cy"]) * Z) / cam["fy"]
        Pw, i0, fr = [], [], []
        for e, n in enumerate((nx, ny, nz)):
            Pw.append(((g[4 * e] * X + g[4 * e + 1] * Y) + g[4 * e + 2] * Z) + g[4 * e + 3])
            q = (Pw[e] - o[e]) / vox
            fl = np.floor(q)
            ok &= (fl >= 0) & (fl <= f32(n - 2))
            i0.append(fl)
            fr.append((q - fl).astype(f32))
    i0 = [np.where(ok, v, 0).astype(np.int64) for v in i0]
    base = (i0[2] * ny + i0[1]) * nx + i0[0]
    c = []
    for off in (0, 1, nx, nx + 1, nx * ny, nx * ny + 1, nx * ny + nx, nx * ny + nx + 1):
        ci = np.minimum(base + off, T.size - 1)  # clipped where the cell is invalid anyway
        with np.errstate(invalid="ignore"):
            ok &= (Wt[ci] >= f32(min_weight)) & (np.abs(T[ci]) < f32(1))
        c.append(T[ci])
    one = f32(1)
    with np.errstate(all="ignore"):
        gx, gy, gz = one - fr[0], one - fr[1], one - fr[2]
        x00, x10 = c[0] * gx + c[1] * fr[0], c[2] * gx + c[3] * fr[0]
        x01, x11 = c[4] * gx + c[5] * fr[0], c[6] * gx + c[7] * fr[0]
        y0, y1 = x00 * gy + x10 * fr[1], x01 * gy + x11 * fr[1]
        r = y0 * gz + y1 * fr[2]
        G0 = (((c[1] - c[0]) * gy + (c[3] - c[2]) * fr[1]) * gz + ((c[5] - c[4]) * gy + (c[7] - c[6]) * fr[1]) * fr[2]) / vox
        G1 = ((x10 - x00) * gz + (x11 - x01) * fr[2]) / vox
        G2 = (y1 - y0) / vox
    return ok, r.astype(f32), np.stack([G0, G1, G2], -1).astype(f32), np.stack(Pw, -1).astype(f32)


def fuse_track_terms(r, G, Pw, huber, c=None) -> np.ndarray:
    """The 28 float64 terms of cells (m, 28): N (21, upper triangle row-major), b (6) and the cost, step 2's order.
    c (m,) float32: the cells' weights of ofdis_fuse_track_weighted, which multiply the Huber weight in float32."""
    a = [G[:, e].astype(np.float64) for e in range(3)]
    w0, w1, w2 = (2.0 * Pw[:, e].astype(np.float64) for e in range(3))
    J = [(a[1] * -w2) + (a[2] * w1), (a[0] * w2) + (a[2] * -w0), (a[0] * -w1) + (a[1] * w0), a[0], a[1], a[2]]
    ar = np.abs(r)
    with np.errstate(all="ignore"):
        wt = np.where(ar <= f32(huber), f32(1), f32(huber) / ar).astype(f32)
        wt = (wt if c is None else wt * np.asarray(c, f32)).astype(np.float64)
    rd = r.astype(np.float64)
    terms = [(wt * J[i]) * J[j] for i in range(6) for j in range(i, 6)]
    terms += [-((wt * J[i]) * rd) for i in range(6)]
    terms.append((wt * rd) * rd)
    return np.stack(terms, -1)


def fuse_track_eval(vol: dict, params, D, cam: dict, p: dict, M, weight=None):
    """One evaluation of ofdis_fuse_track: (N (6, 6) mirrored, b (6,), cost, n_corr) at the pose M; with weight (H, W)
    float32, of ofdis_fuse_track_weighted."""
    ok, r, G, Pw = fuse_track_cells(vol, params, D, cam, p["step"], p["min_weight"], p["max_depth"], M)
    c = None
    if weight is not None:
        H, W = D.shape
        s = int(p["step"])
        ncx, ncy = (W - 1) // s + 1, (H - 1) // s + 1
        cell = np.arange(ncx * ncy)
        c = np.asarray(weight, f32).reshape(H, W)[np.minimum((cell // ncx) * s + s // 2, H - 1),
                                                  np.minimum((cell % ncx) * s + s // 2, W - 1)]
        ok = ok & (c > 0) & (c <= np.finfo(f32).max)
    with np.errstate(all="ignore"):
        T = np.where(ok[:, None], fuse_track_terms(r, G, Pw, p["huber"], c), 0.0)
    v = _chunk_tree(T)
    A = np.zeros((6, 6))
    e = 0
    for a in range(6):
        for b in range(a, 6):
            A[a, b] = A[b, a] = v[e]
            e += 1
    return A, v[21:27], v[27], int(ok.sum())


def fuse_track_guard(M, pred, max_shift, min_cos) -> bool:
    """Step 4's test of ofdis_fuse_track: the last evaluated pose M against the prediction."""
    dt = [M[3] - pred[3], M[7] - pred[7], M[11] - pred[11]]
    shift = np.sqrt((dt[0] * dt[0] + dt[1] * dt[1]) + dt[2] * dt[2])
    s = [((M[4 * i] * pred[4 * i]) + (M[4 * i + 1] * pred[4 * i + 1])) + (M[4 * i + 2] * pred[4 * i + 2])
         for i in range(3)]
    return bool(shift <= max_shift) and bool((((s[0] + s[1]) + s[2]) - 1.0) / 2.0 >= min_cos)


def fuse_track_params(params) -> dict:
    return {k: params[k] for k in FUSE_TRACK_PARAM_FIELDS}


def fuse_track(vol: dict, fuse_params, track_params, disp, motions, prev, camera, frames=None, weights=None):
    """Restates ofdis_fuse_track: disp (n, H, W) float32, motions (n, 3, 4) float64 or None (the identity), prev (3, 4)
    camera-to-world, frames (n, H, W[, 3]) uint8 when integrating into a volume with colour.  With integrate, vol is
    updated in place by fuse_integrate.  With weights (n, H, W) float32 it restates ofdis_fuse_track_weighted.
    Returns (poses (n, 3, 4) float64, stats (n,) FUSE_TRACK_STATS_DTYPE)."""
    p = fuse_track_params(track_params)
    cam = _ego_cam(camera)
    disp = np.asarray(disp, f32).reshape((-1,) + np.shape(disp)[-2:])
    n = disp.shape[0]
    mot = None if motions is None else np.asarray(motions, np.float64).reshape(n, 12)
    P = np.asarray(prev, np.float64).reshape(12)
    poses = np.zeros((n, 12))
    stats = np.zeros(n, FUSE_TRACK_STATS_DTYPE)
    for k in range(n):
        pred = fuse_track_predict(P, None if mot is None else mot[k])
        M, applied, status = pred, 0, 0
        for r in range(int(p["rounds"]) + 1):
            A, b, cost, cnt = fuse_track_eval(vol, fuse_params, disp[k], cam, p, M,
                                              None if weights is None else weights[k])
            if r == 0:
                cost0 = cost
            if cnt < int(p["min_corr"]):
                status = 1 if r == 0 else 0
                break
            if r == int(p["rounds"]):
                break
            for i in range(6):
                A[i, i] = A[i, i] + float(p["damping"])
            x, ok = motion_solve(A[None], b[None])
            if not ok[0] or np.max(np.abs(x[0])) <= float(p["eps"]):
                break
            M, applied = ego_update(M, x[0]), r + 1
        if status == 0 and not fuse_track_guard(M, pred, float(p["max_shift"]), float(p["min_cos"])):
            status = 2
        F = pred if status else M
        poses[k] = F
        stats[k] = (status, cnt, applied, cost0, cost)
        if p["integrate"]:
            fuse_integrate(vol, fuse_params, disp[k:k + 1], F.reshape(1, 3, 4), camera, p["max_depth"],
                           None if vol["C"] is None else np.asarray(frames)[k:k + 1],
                           None if weights is None else np.asarray(weights)[k:k + 1])
        P = F
    return poses.reshape(n, 3, 4), stats


def trajectory_errors(abs_poses, gt_abs):
    """Per frame the absolute error of camera-to-world poses abs_poses against gt_abs (both (n, 3, 4), expressed in
    the same world, e.g. sharing frame 0): the translation error |t - t_gt| in metres and the rotation error
    acos((trace(R_gt^T R) - 1) / 2) in degrees.  Returns (t_err (n,), r_err (n,))."""
    A = np.asarray(abs_poses, np.float64).reshape(-1, 3, 4)
    G = np.asarray(gt_abs, np.float64).reshape(-1, 3, 4)
    t_err = np.linalg.norm(A[:, :, 3] - G[:, :, 3], axis=1)
    c = np.clip(0.5 * (np.einsum("kij,kij->k", A[:, :, :3], G[:, :, :3]) - 1.0), -1.0, 1.0)
    return t_err, np.degrees(np.arccos(c))


# ---- video stabilisation (ofdis_stab_begin / ofdis_stab_push / ofdis_stab_finish) ---------------------------------
STAB_PARAM_FIELDS = ("radius", "crop", "limit")
# ofdis_stab_frame, field for field (96 bytes)
STAB_FRAME_DTYPE = np.dtype({"names": ["frame", "status", "lambda", "correction"],
                             "formats": ["<i8", "<i4", "<f8", ("<f8", (9,))], "offsets": [0, 8, 16, 24],
                             "itemsize": 96})
_EYE = (1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0)


def gaussian_weights(r: int, sigma: float | None = None) -> list:
    """w_d = exp(-d*d / (2 sigma^2)) for d = 0 .. r; sigma^2 = r by default (OpenCV videostab's stdev sqrt(r))."""
    s2 = float(r) if sigma is None else float(sigma) * float(sigma)
    return [math.exp(-d * d / (2 * s2)) for d in range(int(r) + 1)]


def _mat_mul(A, B):
    return tuple((A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j]) + A[3 * i + 2] * B[6 + j]
                 for i in range(3) for j in range(3))


def _mat_norm(A):
    d = A[8]
    if not (math.isfinite(d) and d != 0.0):
        return None
    R = tuple(v / d for v in A)
    return R if all(math.isfinite(v) for v in R) else None


def _mat_inv(a):
    C = (a[4] * a[8] - a[5] * a[7], a[2] * a[7] - a[1] * a[8], a[1] * a[5] - a[2] * a[4],
         a[5] * a[6] - a[3] * a[8], a[0] * a[8] - a[2] * a[6], a[2] * a[3] - a[0] * a[5],
         a[3] * a[7] - a[4] * a[6], a[1] * a[6] - a[0] * a[7], a[0] * a[4] - a[1] * a[3])
    return _mat_norm(C)


def stab_model(m) -> tuple:
    """A model as received: its 9 entries divided by m22, or the identity (m22 not finite and non-zero, a non-finite
    entry, or m00*m11 - m01*m10 of the divided model not finite and non-zero)."""
    m = [float(v) for v in np.asarray(m, np.float64).reshape(-1)]
    d = m[8]
    if not (math.isfinite(d) and d != 0.0):
        return _EYE
    q = tuple(v / d for v in m)
    if not all(math.isfinite(v) for v in q):
        return _EYE
    a = q[0] * q[4] - q[1] * q[3]
    return q if math.isfinite(a) and a != 0.0 else _EYE


def stab_path(models, t: int, a: int, b: int, weights):
    """S of frame t over the window [a, b] (9 floats), or None where the path is undefined.  models[k] is M_k as
    received (stab_model) for k in [a, b-1]; any mapping of those indices will do."""
    w0 = float(weights[0])
    acc = [w0 if i % 4 == 0 else 0.0 for i in range(9)]
    wsum = w0
    for sign in (1, -1):
        P = _EYE
        for d in range(1, (b - t if sign > 0 else t - a) + 1):
            if sign > 0:
                P = _mat_norm(_mat_mul(models[t + d - 1], P))
            else:
                Q = _mat_inv(models[t - d])
                P = None if Q is None else _mat_norm(_mat_mul(Q, P))
            if P is None:
                return None
            wd = float(weights[d])
            acc = [acc[i] + wd * P[i] for i in range(9)]
            wsum = wsum + wd
    S = tuple(v / wsum for v in acc)
    return S if all(math.isfinite(v) for v in S) else None


def _stab_map(S, lam, crop, w, h):
    """(S(lam), A(lam) rounded to float32 or None)."""
    SL = tuple((1.0 - lam) + lam * S[i] if i % 4 == 0 else lam * S[i] for i in range(9))
    s = 1.0 - 2.0 * float(np.float32(crop))
    cx, cy = 0.5 * float(w - 1), 0.5 * float(h - 1)
    Si = _mat_inv(SL)
    A = None if Si is None else _mat_norm(_mat_mul(Si, (s, 0.0, cx * (1.0 - s), 0.0, s, cy * (1.0 - s), 0.0, 0.0, 1.0)))
    return SL, None if A is None else np.array(A).astype(np.float32)


def _stab_project(a, X, Y):
    """(wq, mx/wq, my/wq) of the per-pixel rule, float32."""
    with np.errstate(all="ignore"):
        mx = (a[0] * X + a[1] * Y) + a[2]
        my = (a[3] * X + a[4] * Y) + a[5]
        wq = (a[6] * X + a[7] * Y) + a[8]
        return wq, mx / wq, my / wq


def stab_correction(S, params, w: int, h: int):
    """The crop and limit of frame t's S (None: an undefined path): (status, lambda, S(lambda) (9 floats), a0..a8
    (9,) float32)."""
    f32 = np.float32
    crop, limit = params["crop"], int(params["limit"])
    X = np.array([0, w - 1, 0, w - 1], f32)
    Y = np.array([0, 0, h - 1, h - 1], f32)

    def passes(lam):
        SL, a = _stab_map(S, lam, crop, w, h)
        if a is None:
            return False
        wq, xw, yw = _stab_project(a, X, Y)
        with np.errstate(invalid="ignore"):
            return bool(((wq > 0) & (xw >= 0) & (xw <= f32(w - 1)) & (yw >= 0) & (yw <= f32(h - 1))).all())

    if S is not None:
        lam = 1.0
        if limit and not passes(1.0):
            lo, hi = 0.0, 1.0
            for _ in range(20):
                mid = 0.5 * (lo + hi)
                if passes(mid):
                    lo = mid
                else:
                    hi = mid
            lam = lo
        SL, a = _stab_map(S, lam, crop, w, h)
        if a is not None:
            return 0, lam, SL, a
    SL, a = _stab_map(_EYE, 0.0, crop, w, h)
    return 1, 0.0, SL, a


def stab_warp(frame: np.ndarray, a: np.ndarray) -> np.ndarray:
    """The stabilised bytes of one frame (h, w[, noc]) under a0..a8."""
    h, w = frame.shape[:2]
    X = np.arange(w, dtype=np.float32)[None, :]
    Y = np.arange(h, dtype=np.float32)[:, None]
    wq, xw, yw = _stab_project(a, X, Y)
    return _sample_u8(frame, wq, xw, yw)


def stab_params(params) -> dict:
    return {k: params[k] for k in STAB_PARAM_FIELDS}


def stabilize(frames: np.ndarray, models: np.ndarray, params, weights):
    """ofdis_stab_begin on frames[0], pushes of the others and ofdis_stab_finish, bit for bit, however the clip is cut
    into pushes: float64 path, float32 warp, without contraction.  frames (N, h, w[, noc]) uint8, models (N-1, 3, 3)
    (model k maps frame k to frame k+1, as ofdis_global_motion_fullres returns it), params a mapping with
    STAB_PARAM_FIELDS, weights r+1 floats.  Returns (stabilised frames (N, h, w[, noc]) uint8, records (N,) of
    STAB_FRAME_DTYPE)."""
    p = stab_params(params)
    frames = np.asarray(frames, np.uint8)
    n = frames.shape[0]
    h, w = frames.shape[1:3]
    r = int(p["radius"])
    M = [stab_model(m) for m in np.asarray(models, np.float64).reshape(-1, 9)]
    assert len(M) == n - 1
    out = np.empty_like(frames)
    info = np.zeros(n, STAB_FRAME_DTYPE)
    for t in range(n):
        S = stab_path(M, t, max(0, t - r), min(n - 1, t + r), weights)
        status, lam, SL, a = stab_correction(S, p, w, h)
        out[t] = stab_warp(frames[t], a)
        info[t] = (t, status, lam, SL)
    return out, info


def global_motion(F: np.ndarray, B: np.ndarray | None, frames1: np.ndarray | None, params):
    """ofdis_global_motion_fullres, bit for bit: float32 as the header marks it, float64 in the solver, without
    contraction.  F: the full-resolution flows of the pairs, (n, h, w, 2) or one pair (h, w, 2) float32, exactly what
    ofdis_get_flow_fullres returns; B: their partners' (read with fb_check only); frames1: the 8-bit I1 of every pair,
    (n, h, w[, noc]) (None: no registered frames); params: a mapping with MOTION_PARAM_FIELDS (the model as a number or
    a name of MOTION_MODELS).  Returns (models (n, 3, 3) float64, stats (n,) MOTION_STATS_DTYPE, mask (n, h, w) uint8,
    residual (n, h, w, 2) float32, registered (n, h, w[, noc]) uint8 or None), without the leading axis for one pair."""
    p = motion_params(params)
    Fa = np.asarray(F, np.float32)
    one = Fa.ndim == 3
    Fa = Fa[None] if one else Fa
    Ba = None if B is None else np.asarray(B, np.float32).reshape(Fa.shape)
    I1 = None if frames1 is None else np.asarray(frames1, np.uint8)
    if I1 is not None and one:
        I1 = I1[None]
    res = [_motion_pair(Fa[i], None if Ba is None else Ba[i], None if I1 is None else I1[i], p)
           for i in range(Fa.shape[0])]
    models = np.stack([r[0] for r in res]).reshape(-1, 3, 3)
    stats = np.stack([r[1] for r in res])
    mask = np.stack([r[2] for r in res])
    residual = np.stack([r[3] for r in res])
    reg = None if I1 is None else np.stack([r[4] for r in res])
    if one:
        return models[0], stats[0], mask[0], residual[0], None if reg is None else reg[0]
    return models, stats, mask, residual, reg


# ---- trajectory descriptors (ofdis_traj_begin / ofdis_traj_advance) -------------------------------------------------
# ofdis_traj_params, ofdis_traj_record and ofdis_traj_stats, field for field
TRAJ_PARAM_FIELDS = ("L", "nt", "N", "ns", "min_flow", "eps", "min_disp", "min_var", "max_var", "max_dis")
TRAJ_RECORD_DTYPE = np.dtype([("id", "<i4"), ("start", "<i4"), ("mean_x", "<f4"), ("mean_y", "<f4"),
                              ("sd_x", "<f4"), ("sd_y", "<f4"), ("length", "<f4")])
TRAJ_STATS_FIELDS = ("emitted", "rejected_static", "rejected_erratic", "rejected_jump", "rejected_camera")
# Wang and Schmid's improved dense trajectories (ICCV 2013)
TRAJ_DEFAULTS = {"L": 15, "nt": 3, "N": 32, "ns": 2, "min_flow": 0.4, "eps": 0.05, "min_disp": 1.0,
                 "min_var": math.sqrt(3.0), "max_var": 50.0, "max_dis": 20.0}
TRAJ_BINS = 33                   # HOG 8, HOF 9, MBHx 8, MBHy 8 per spatial cell
_TRAJ_LO = (0, 8, 17, 25)        # first entry of each in a cell's 33
_TRAJ_NB = (8, 9, 8, 8)
_TWO_PI_F = np.float32(6.2831855)
_BIN_SCALE = np.float32(1.2732395)  # 8 / (2 pi)
_NO_BIN = 255
_FLT_MAX = np.float32(np.finfo(np.float32).max)


def traj_dim(p) -> int:
    """Floats per descriptor: 2L + ns^2 nt 33 (426 with TRAJ_DEFAULTS)."""
    return 2 * int(p["L"]) + int(p["ns"]) ** 2 * int(p["nt"]) * TRAJ_BINS


def traj_bound(capacity: int, n: int, L: int) -> int:
    """The most segments a call of n pairs emits: capacity * ceil((n + L - 1) / L)."""
    return int(capacity) * ((int(n) + 2 * int(L) - 2) // int(L)) if n > 0 else 0


def orientation_bins(a, b):
    """The orientation bins of the vectors (a, b) (ofdis_traj_params' header): (bin0, mag0, mag1), bin0 uint8 with
    255 where mag = sqrtf(a*a + b*b) is not finite (mag0 = mag1 = 0 there); bin1 = (bin0 + 1) % 8."""
    f32 = np.float32
    a, b = np.asarray(a, f32), np.asarray(b, f32)
    with np.errstate(invalid="ignore", over="ignore"):
        mag = np.sqrt(a * a + b * b)
        ok = mag <= _FLT_MAX
        ang = atan2_f32(b, a)
        ang = np.where(ang < 0, ang + _TWO_PI_F, ang).astype(f32)
        fbin = (ang * _BIN_SCALE).astype(f32)
        fb0 = np.floor(fbin)
        m1 = ((fbin - fb0) * mag).astype(f32)
        m0 = (mag - m1).astype(f32)
    b0 = np.where(ok, fb0, 0).astype(np.int64)
    b0 = np.where(b0 >= 8, 0, b0)
    return (np.where(ok, b0, _NO_BIN).astype(np.uint8), np.where(ok, m0, f32(0)).astype(f32),
            np.where(ok, m1, f32(0)).astype(f32))


def traj_model(m) -> np.ndarray:
    """A received model (9 float64, or None) as the descriptors apply it: stab_model, then float32."""
    return np.array(_EYE if m is None else stab_model(m), np.float32)


def traj_residual(F: np.ndarray, m32: np.ndarray):
    """(R, known): the residual flow F - the model's flow, (h, w, 2) float32, and where it is known."""
    f32 = np.float32
    F = np.asarray(F, f32)
    h, w = F.shape[:2]
    m = [f32(v) for v in np.asarray(m32, f32).reshape(9)]
    X = np.broadcast_to(np.arange(w, dtype=f32)[None, :], (h, w))
    Y = np.broadcast_to(np.arange(h, dtype=f32)[:, None], (h, w))
    u, v = F[..., 0], F[..., 1]
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        mx = (m[0] * X + m[1] * Y) + m[2]
        my = (m[3] * X + m[4] * Y) + m[5]
        wq = (m[6] * X + m[7] * Y) + m[8]
        ru = u - (mx / wq - X)
        rv = v - (my / wq - Y)
        known = (np.abs(u) <= f32(1e9)) & (np.abs(v) <= f32(1e9)) & (wq > 0) & (np.abs(ru) <= _FLT_MAX) & \
            (np.abs(rv) <= _FLT_MAX)
    return np.stack([ru, rv], -1).astype(f32), known


def _brightness(frame: np.ndarray) -> np.ndarray:
    f32 = np.float32
    I = np.asarray(frame, np.uint8)
    if I.ndim == 3 and I.shape[2] == 3:
        return (I[..., 0].astype(f32) + I[..., 1].astype(f32) + I[..., 2].astype(f32)) / f32(3)
    return I.reshape(I.shape[:2]).astype(f32)


def _cdiff(f: np.ndarray):
    """The tracker's clamped central differences of an (h, w) plane: (dx, dy)."""
    h, w = f.shape
    xs, ys = np.arange(w), np.arange(h)
    with np.errstate(invalid="ignore", over="ignore"):
        dx = (f[:, np.minimum(xs + 1, w - 1)] - f[:, np.maximum(xs - 1, 0)]) * np.float32(0.5)
        dy = (f[np.minimum(ys + 1, h - 1), :] - f[np.maximum(ys - 1, 0), :]) * np.float32(0.5)
    return dx, dy


def traj_fields(frame: np.ndarray, F: np.ndarray, m32: np.ndarray, min_flow):
    """The per-pixel fields of one source frame: (contrib, R, known).  contrib (h, w, 33) float32 is what the pixel
    adds to each of a cell's 33 bins (HOG 0-7, HOF 8-16 with the zero bin 16, MBHx 17-24, MBHy 25-32), 0 elsewhere."""
    f32 = np.float32
    R, known = traj_residual(F, m32)
    h, w = known.shape
    gx, gy = _cdiff(_brightness(frame))
    xs, ys = np.arange(w), np.arange(h)
    xl, xr = np.maximum(xs - 1, 0), np.minimum(xs + 1, w - 1)
    yu, yd = np.maximum(ys - 1, 0), np.minimum(ys + 1, h - 1)
    kn = known[:, xl] & known[:, xr] & known[yu, :] & known[yd, :]
    fields = [(gx, gy, np.ones((h, w), bool))]
    fields.append((R[..., 0], R[..., 1], known))
    for c in range(2):
        dx, dy = _cdiff(R[..., c])
        fields.append((dx, dy, kn))
    contrib = np.zeros((h, w, TRAJ_BINS), f32)
    rows, cols = np.indices((h, w))
    for q, (a, b, ok) in enumerate(fields):
        b0, m0, m1 = orientation_bins(np.where(ok, a, f32(0)), np.where(ok, b, f32(0)))
        has = ok & (b0 != _NO_BIN)
        if q == 1:
            with np.errstate(invalid="ignore", over="ignore"):
                zero = has & (np.sqrt(R[..., 0] * R[..., 0] + R[..., 1] * R[..., 1]) <= f32(min_flow))
            b0 = np.where(zero, 8, b0)
            m0 = np.where(zero, f32(1), m0)
            m1 = np.where(zero, f32(0), m1)
        lo = _TRAJ_LO[q]
        b1 = np.where(b0 == 8, 1, (b0.astype(np.int64) + 1) % 8)
        contrib[rows[has], cols[has], lo + b0[has].astype(np.int64)] = m0[has]
        contrib[rows[has], cols[has], lo + b1[has]] += m1[has]
    return contrib, R, known


def traj_frame_hist(contrib: np.ndarray, xs: np.ndarray, ys: np.ndarray, p) -> np.ndarray:
    """The RootSIFT-normalised frame histograms of tracks at (xs, ys): (T, ns*ns, 33) float32, cells (cx, cy) as
    cx * ns + cy; each cell's sums in the lane order of the header."""
    f32 = np.float32
    h, w = contrib.shape[:2]
    N, ns = int(p["N"]), int(p["ns"])
    c = N // ns
    T = xs.size
    chunk = max(1, (1 << 24) // (((c * c + 31) // 32) * 32 * TRAJ_BINS))  # tracks per 64 MB of lane sums
    if T > chunk:
        return np.concatenate([traj_frame_hist(contrib, xs[i:i + chunk], ys[i:i + chunk], p)
                               for i in range(0, T, chunk)])
    xr = np.floor(xs.astype(f32) + f32(0.5)).astype(np.int64)
    yr = np.floor(ys.astype(f32) + f32(0.5)).astype(np.int64)
    ox = np.minimum(np.maximum(xr - N // 2, 0), w - N)
    oy = np.minimum(np.maximum(yr - N // 2, 0), h - N)
    cc = c * c
    rounds = (cc + 31) // 32
    q = np.arange(cc)
    v = np.empty((T, ns * ns, TRAJ_BINS), f32)
    for cx in range(ns):
        for cy in range(ns):
            px = ox[:, None] + cx * c + q[None, :] % c
            py = oy[:, None] + cy * c + q[None, :] // c
            a = np.zeros((T, rounds * 32, TRAJ_BINS), f32)
            a[:, :cc] = contrib[py, px]
            a = a.reshape(T, rounds, 32, TRAJ_BINS)
            lane = a[:, 0]
            for r in range(1, rounds):
                lane = lane + a[:, r]
            s = lane[:, 0]
            for l in range(1, 32):
                s = s + lane[:, l]
            v[:, cx * ns + cy] = s + f32(p["eps"])
    out = np.empty_like(v)
    for d in range(4):
        lo, nb = _TRAJ_LO[d], _TRAJ_NB[d]
        s = np.zeros(T, f32)
        for cell in range(ns * ns):
            for k in range(nb):
                s = s + v[:, cell, lo + k]
        out[:, :, lo:lo + nb] = np.sqrt(v[:, :, lo:lo + nb] / s[:, None, None])
    return out


def traj_segment_tests(pos: np.ndarray, disp: np.ndarray, p):
    """The tests of S completed segments: pos (S, L+1, 2), disp (S, L, 2) float32.  Returns (why, stats, dsum): why
    (S,) 0 emitted, 1 static, 2 erratic, 3 jump, 4 camera; stats (mean_x, mean_y, sd_x, sd_y, length) and dsum (S,)
    float32, each sum over j in order."""
    f32 = np.float32
    S, L = disp.shape[:2]
    fn = f32(L + 1)
    z = lambda: np.zeros(S, f32)  # noqa: E731
    with np.errstate(invalid="ignore", over="ignore"):
        sx, sy = z(), z()
        for j in range(L + 1):
            sx = sx + pos[:, j, 0]
            sy = sy + pos[:, j, 1]
        mx, my = sx / fn, sy / fn
        vx, vy = z(), z()
        for j in range(L + 1):
            dx, dy = pos[:, j, 0] - mx, pos[:, j, 1] - my
            vx = vx + dx * dx
            vy = vy + dy * dy
        sdx, sdy = np.sqrt(vx / fn), np.sqrt(vy / fn)
        length, smax = z(), z()
        for j in range(L):
            dx, dy = pos[:, j + 1, 0] - pos[:, j, 0], pos[:, j + 1, 1] - pos[:, j, 1]
            s = np.sqrt(dx * dx + dy * dy)
            length = length + s
            smax = np.where(s > smax, s, smax)
        dsum, dmax = z(), z()
        known = np.ones(S, bool)
        for j in range(L):
            du, dv = disp[:, j, 0], disp[:, j, 1]
            a = np.sqrt(du * du + dv * dv)
            known &= a <= _FLT_MAX
            dsum = dsum + a
            dmax = np.where(a > dmax, a, dmax)
        why = np.where(~known | (dmax <= f32(p["min_disp"])), 4, 0)
        why = np.where((smax > f32(p["max_dis"])) & (smax > f32(0.7) * length), 3, why)
        why = np.where((sdx > f32(p["max_var"])) | (sdy > f32(p["max_var"])), 2, why)
        why = np.where((sdx < f32(p["min_var"])) & (sdy < f32(p["min_var"])), 1, why)
    return why, (mx, my, sdx, sdy, length), dsum


def traj_segment_test(pos: np.ndarray, disp: np.ndarray, p):
    """traj_segment_tests of one segment: pos (L+1, 2), disp (L, 2) float32; why an int, the rest float32 scalars."""
    why, stats, dsum = traj_segment_tests(np.asarray(pos, np.float32)[None], np.asarray(disp, np.float32)[None], p)
    return int(why[0]), tuple(v[0] for v in stats), dsum[0]


class TrajStream:
    """ofdis_traj_begin / ofdis_traj_advance restated bit for bit, one call at a time, on the tracker of
    track_points: begin(frame), then advance(frames, fw, bw, models) for every call with the call's target frames
    (n, h, w[, noc]), full-resolution flows (n, h, w, 2) and models (n, 9) float64 or None."""

    def __init__(self, track_params, traj_params):
        self.tp = {k: track_params[k] for k in TRACK_PARAM_FIELDS}
        self.p = {k: traj_params[k] for k in TRAJ_PARAM_FIELDS}
        L, nt, ns = int(self.p["L"]), int(self.p["nt"]), int(self.p["ns"])
        assert L % nt == 0 and int(self.p["N"]) % ns == 0
        self.L, self.nt, self.ns, self.tl = L, nt, ns, L // nt

    def _fresh(self, n):
        return (np.zeros(n, np.int64), np.zeros(n, np.int64), np.zeros((n, self.L + 1, 2), np.float32),
                np.zeros((n, self.L, 2), np.float32), np.zeros((n, self.nt, self.ns * self.ns, TRAJ_BINS), np.float32))

    def begin(self, frame):
        self.stats = dict.fromkeys(TRACK_STATS_FIELDS, 0)
        self.tstats = dict.fromkeys(TRAJ_STATS_FIELDS, 0)
        self.tracks, self.next_id = _track_seed(np.asarray(frame, np.uint8), np.empty(0, TRACK_POINT_DTYPE), 0,
                                                self.stats, self.tp)
        self.step, self.start, self.pos, self.disp, self.acc = self._fresh(self.tracks.size)
        self.frame = np.asarray(frame, np.uint8)
        self.fr = 0
        return self.tracks

    def _emit(self, disp, a, dsum):
        """The descriptors (S, dim) of S segments: disp (S, L, 2), a (S, nt, ns^2, 33), dsum (S,)."""
        f32 = np.float32
        S = dsum.size
        parts = [(disp / dsum[:, None, None]).astype(f32).reshape(S, -1)]
        for d in range(4):
            lo, nb = _TRAJ_LO[d], _TRAJ_NB[d]
            parts.append((a[..., lo:lo + nb] / f32(self.tl)).astype(f32).reshape(S, -1))
        return np.concatenate(parts, 1)

    def advance(self, frames, fw, bw, models=None):
        """Returns (lists, records, desc, n_desc), as Context.traj_advance on the host."""
        f32 = np.float32
        clip = np.asarray(frames, np.uint8)
        F = np.asarray(fw, f32)
        B = np.asarray(bw, f32)
        n = F.shape[0]
        lists, recs, descs, n_desc = [], [], [], []
        p, L, tkeys = self.p, self.L, ("mean_x", "mean_y", "sd_x", "sd_y", "length")
        for k in range(n):
            m32 = traj_model(None if models is None else models[k])
            contrib, R, known = traj_fields(self.frame, F[k], m32, p["min_flow"])
            tr = self.tracks
            T = tr.size
            if T:
                xs, ys = tr["x"], tr["y"]
                xr = np.floor(xs + f32(0.5)).astype(np.int64)
                yr = np.floor(ys + f32(0.5)).astype(np.int64)
                hist = traj_frame_hist(contrib, xs, ys, p)
                idx = np.arange(T)
                t = self.step
                self.pos[idx, t, 0], self.pos[idx, t, 1] = xs, ys
                d = np.where(known[yr, xr][:, None], R[yr, xr], f32(np.nan))
                self.disp[idx, t] = d
                tc = t // self.tl
                first = (t % self.tl) == 0
                cur = self.acc[idx, tc]
                self.acc[idx, tc] = np.where(first[:, None, None], hist, cur + hist)
            adv = _track_advance(tr, F[k], B[k], self.stats, self.tp)
            keep = np.isin(tr["id"], adv["id"])
            step, start, pos, disp, acc = (a[keep] for a in (self.step, self.start, self.pos, self.disp, self.acc))
            step = step + 1
            done = np.flatnonzero(step == L)  # in list order, the order of the records
            pos[done, L, 0], pos[done, L, 1] = adv["x"][done], adv["y"][done]
            why, st, dsum = traj_segment_tests(pos[done], disp[done], p)
            for r in range(1, len(TRAJ_STATS_FIELDS)):
                self.tstats[TRAJ_STATS_FIELDS[r]] += int((why == r).sum())
            em = why == 0
            ne = int(em.sum())
            if ne:
                e = done[em]
                rec = np.zeros(ne, TRAJ_RECORD_DTYPE)
                rec["id"], rec["start"] = adv["id"][e], start[e]
                for key, val in zip(tkeys, st):
                    rec[key] = val[em]
                recs.append(rec)
                descs.append(self._emit(disp[e], acc[e], dsum[em]))
            step[done] = 0
            start[done] += L
            self.tstats["emitted"] += ne
            n_desc.append(ne)
            tracks, self.next_id = _track_seed(clip[k], adv, self.next_id, self.stats, self.tp)
            ns_ = tracks.size - adv.size
            fresh = self._fresh(ns_)
            fresh[1][:] = self.fr + 1
            self.step, self.start, self.pos, self.disp, self.acc = (np.concatenate([a, b]) for a, b in
                                                                    zip((step, start, pos, disp, acc), fresh))
            self.tracks = tracks
            lists.append(tracks)
            self.frame = clip[k]
            self.fr += 1
        dim = traj_dim(p)
        records = np.concatenate(recs) if recs else np.zeros(0, TRAJ_RECORD_DTYPE)
        desc = np.concatenate(descs).astype(f32) if descs else np.zeros((0, dim), f32)
        return lists, records, desc, np.array(n_desc, np.int32)

    def track_stats(self):
        st = dict(self.stats)
        st["alive"], st["next_id"] = int(self.tracks.size), int(self.next_id)
        return st


def traj_descriptors(frames: np.ndarray, fw: np.ndarray, bw: np.ndarray, models, track_params, traj_params):
    """ofdis_traj_begin on frames[0] followed by one ofdis_traj_advance through the n pairs, bit for bit.  frames: the
    clip (n + 1, h, w[, noc]) uint8; fw, bw: the full-resolution forward flows and their backward partners (n, h, w, 2)
    float32; models: (n, 9) float64 or None.  Returns (lists, records, desc, n_desc, track_stats, traj_stats)."""
    clip = np.asarray(frames, np.uint8)
    s = TrajStream(track_params, traj_params)
    first = s.begin(clip[0])
    lists, records, desc, n_desc = s.advance(clip[1:], fw, bw, models)
    return [first] + lists, records, desc, n_desc, s.track_stats(), dict(s.tstats)


# ---- Fisher vectors of descriptors (ofdis_fisher_begin / ofdis_fisher_push / ofdis_fisher_take) ----------------------
# The library's float32 exp (exp_f32, ofdis_internal.cuh): Cody-Waite reduction by ln 2 (ln2_hi has 15 significant bits,
# so n * ln2_hi is exact for |n| <= 256), the degree-7 Taylor polynomial of e^r in Horner form, then the exact scale by
# 2^n.  +0 below EXP_CUTOFF (where e^x would leave the normal range), exactly 1 at +-0; within 2 ulp of float64 exp on
# [EXP_CUTOFF, 0] (1.21 ulp at most over every third float32 there).
EXP_CUTOFF = np.float32(-87.0)
_EXP_LOG2E = np.float32(1.44269504)
_EXP_LN2_HI = np.float32(0.693145751953125)
_EXP_LN2_LO = np.float32(1.42860677e-06)
_EXP_C = np.array([1.0, 1.0, 0.5, 0.166666672, 0.0416666679, 0.00833333377, 0.00138888892, 0.000198412701],
                  np.float32)  # 1/k!
FISHER_MAX_K = 256
FISHER_MAX_BLOCKS = 8
FISHER_MAX_DIM = 512
FISHER_MAGIC = b"OFDISFV1"
# ofdis_fisher_stats, field for field (136 bytes)
FISHER_STATS_DTYPE = np.dtype([("pushed", "<i8"), ("n", "<i8", (FISHER_MAX_BLOCKS,)),
                               ("skipped", "<i8", (FISHER_MAX_BLOCKS,))])
FISHER_PARTS = ("mean", "proj", "mu", "isig", "c", "w")  # the packed order of a block's float32 arrays


def exp_f32(x) -> np.ndarray:
    """exp_f32 of float32 x <= 0 (or -inf), elementwise, bit for bit."""
    f32 = np.float32
    x = np.asarray(x, f32)
    with np.errstate(all="ignore"):
        n = np.rint(x * _EXP_LOG2E)
        r = (x - n * _EXP_LN2_HI) - n * _EXP_LN2_LO
        p = np.full(x.shape, _EXP_C[7], f32)
        for k in range(6, -1, -1):
            p = p * r + _EXP_C[k]
        ni = np.fmin(np.fmax(n, np.float32(-126)), np.float32(128)).astype(np.int32)
        scale = ((ni + 127) << 23).astype(np.int32).view(f32)
        return np.where(x < EXP_CUTOFF, f32(0), p * scale).astype(f32)


def fisher_blocks(traj_params):
    """The descriptor blocks of ofdis_traj_advance's descriptors, [(offset, dim_in)]: shape 2L, HOG nt ns^2 8, HOF
    nt ns^2 9, MBHx and MBHy nt ns^2 8 each (30/96/108/96/96 with TRAJ_DEFAULTS)."""
    L, c = int(traj_params["L"]), int(traj_params["nt"]) * int(traj_params["ns"]) ** 2
    out, off = [], 0
    for d in (2 * L, 8 * c, 9 * c, 8 * c, 8 * c):
        out.append((off, d))
        off += d
    return out


def fisher_sizes(K: int, blocks) -> dict:
    """Floats of the packed body, of the vector (2K sum dim) and doubles of the statistics (sum K(1 + 2 dim))."""
    body = sum(di + d * di + 2 * K * d + 2 * K for _, di, d in blocks)
    return {"body": body, "fv": 2 * K * sum(d for _, _, d in blocks),
            "stats": sum(K * (1 + 2 * d) for _, _, d in blocks)}


def fisher_pack(cb) -> np.ndarray:
    """The codebook's float32 body: per block mean[dim_in], proj[dim][dim_in], mu[K][dim], isig[K][dim], c[K], w[K]."""
    return np.concatenate([np.asarray(cb[k][b], np.float32).ravel() for b in range(len(cb["blocks"]))
                           for k in FISHER_PARTS]).astype(np.float32)


def fisher_unpack(K: int, desc_dim: int, blocks, body) -> dict:
    """A codebook dict from its header fields and packed body (fisher_pack's inverse)."""
    body = np.asarray(body, np.float32).ravel()
    blocks = [tuple(int(v) for v in b) for b in blocks]
    if body.size != fisher_sizes(K, blocks)["body"]:
        raise ValueError("fisher codebook: body of %d floats, %d expected" % (body.size, fisher_sizes(K, blocks)["body"]))
    cb = {"K": int(K), "desc_dim": int(desc_dim), "blocks": blocks}
    for k in FISHER_PARTS:
        cb[k] = []
    p = 0
    for _, di, d in blocks:
        for k, shape in zip(FISHER_PARTS, ((di,), (d, di), (K, d), (K, d), (K,), (K,))):
            n = int(np.prod(shape))
            cb[k].append(body[p:p + n].reshape(shape).copy())
            p += n
    return cb


def fisher_check(cb) -> None:
    """Raises ValueError where ofdis_fisher_begin answers OFDIS_ERR_ARG."""
    K, D, blocks = cb["K"], cb["desc_dim"], cb["blocks"]
    if not (1 <= K <= FISHER_MAX_K and 1 <= len(blocks) <= FISHER_MAX_BLOCKS and D >= 1):
        raise ValueError("fisher codebook: K %d, %d blocks, desc_dim %d out of range" % (K, len(blocks), D))
    for b, (o, di, d) in enumerate(blocks):
        if not (1 <= d <= di <= FISHER_MAX_DIM and o >= 0 and o + di <= D):
            raise ValueError("fisher codebook: block %d (%d, %d, %d) out of range" % (b, o, di, d))
        arrs = [np.asarray(cb[k][b], np.float32) for k in FISHER_PARTS]
        if not all(np.isfinite(a).all() for a in arrs) or not (arrs[3] > 0).all() or not (arrs[5] > 0).all():
            raise ValueError("fisher codebook: block %d has non-finite entries or isig, w not > 0" % b)


def write_fisher_codebook(path: str, cb) -> None:
    """The codebook file: OFDISFV1, int32 K, nblocks, desc_dim, (offset, dim_in, dim) per block, the float32 body,
    all little-endian."""
    hdr = [cb["K"], len(cb["blocks"]), cb["desc_dim"]] + [v for b in cb["blocks"] for v in b]
    with open(path, "wb") as f:
        f.write(FISHER_MAGIC + np.asarray(hdr, "<i4").tobytes() + fisher_pack(cb).astype("<f4").tobytes())


def read_fisher_codebook(path: str) -> dict:
    """write_fisher_codebook's file back; ValueError on a malformed file."""
    with open(path, "rb") as f:
        raw = f.read()
    if raw[:8] != FISHER_MAGIC or len(raw) < 20:
        raise ValueError("%s: not a fisher codebook" % path)
    K, nb, D = (int(v) for v in np.frombuffer(raw, "<i4", 3, 8))
    if not 1 <= nb <= FISHER_MAX_BLOCKS or len(raw) < 20 + 12 * nb:
        raise ValueError("%s: bad block count %d" % (path, nb))
    blocks = [tuple(int(v) for v in r) for r in np.frombuffer(raw, "<i4", 3 * nb, 20).reshape(nb, 3)]
    if K < 1 or any(di < 1 or d < 1 for _, di, d in blocks):
        raise ValueError("%s: bad header" % path)
    body = np.frombuffer(raw, "<f4", offset=20 + 12 * nb) if (len(raw) - 20 - 12 * nb) % 4 == 0 else None
    if body is None or body.size != fisher_sizes(K, blocks)["body"]:
        raise ValueError("%s: body size does not match the header" % path)
    cb = fisher_unpack(K, D, blocks, body.astype(np.float32))
    fisher_check(cb)
    return cb


def fisher_project(x: np.ndarray, mean: np.ndarray, proj: np.ndarray) -> np.ndarray:
    """y_d = sum_i proj[d][i] * (x_i - mean_i), float32, from +0.0f in increasing i; x (n, dim_in) -> (n, dim)."""
    f32 = np.float32
    with np.errstate(all="ignore"):
        t = (np.asarray(x, f32) - np.asarray(mean, f32)[None]).astype(f32)
        y = np.zeros((t.shape[0], proj.shape[0]), f32)
        for i in range(t.shape[1]):
            y = y + proj[:, i][None, :] * t[:, i:i + 1]
    return y


def fisher_posteriors(y: np.ndarray, mu: np.ndarray, isig: np.ndarray, c: np.ndarray):
    """(gamma (n, K) float32, skipped (n,) bool) of projected descriptors y (n, dim): q_k = sum_d z_kd^2 in increasing
    d, z_kd = (y_d - mu_kd) * isig_kd, ll_k = c_k - 0.5f q_k, m = max ll, e_k = exp_f32(ll_k - m), s = sum_k e_k in
    increasing k, gamma_k = e_k / s; skipped where a y_d, a q_k or m is not finite."""
    f32 = np.float32
    n, K = y.shape[0], mu.shape[0]
    with np.errstate(all="ignore"):
        q = np.zeros((n, K), f32)
        for d in range(y.shape[1]):
            z = (y[:, d:d + 1] - mu[:, d][None, :]) * isig[:, d][None, :]
            q = q + z * z
        ll = (c[None, :] - f32(0.5) * q).astype(f32)
        m = ll.max(axis=1) if K else np.zeros(n, f32)
        skipped = ~np.isfinite(y).all(axis=1) | ~np.isfinite(q).all(axis=1) | ~np.isfinite(m)
        e = exp_f32(np.where(skipped[:, None], f32(0), ll - m[:, None]))
        s = np.cumsum(e, axis=1, dtype=f32)[:, -1]
        g = (e / s[:, None]).astype(f32)
    return g, skipped


class FisherStream:
    """ofdis_fisher_begin / push / take restated bit for bit: begin(codebook), push(desc) any number of times, then
    take() -> (fv, stats, counters) as Context.fisher_take, which resets the clip."""

    def __init__(self, cb):
        self.begin(cb)

    def begin(self, cb):
        fisher_check(cb)
        self.cb = cb
        self._reset()

    def _reset(self):
        K = self.cb["K"]
        self.S0 = [np.zeros(K) for _ in self.cb["blocks"]]
        self.S1 = [np.zeros((K, d)) for _, _, d in self.cb["blocks"]]
        self.S2 = [np.zeros((K, d)) for _, _, d in self.cb["blocks"]]
        self.pushed = 0
        self.n = np.zeros(len(self.cb["blocks"]), np.int64)
        self.skipped = np.zeros(len(self.cb["blocks"]), np.int64)

    def push(self, desc):
        cb = self.cb
        x = np.asarray(desc, np.float32).reshape(-1, cb["desc_dim"])
        self.pushed += x.shape[0]
        for b, (o, di, d) in enumerate(cb["blocks"]):
            mu, isig = cb["mu"][b], cb["isig"][b]
            y = fisher_project(x[:, o:o + di], cb["mean"][b], cb["proj"][b])
            g, skip = fisher_posteriors(y, mu, isig, cb["c"][b])
            keep = ~skip
            self.n[b] += int(keep.sum())
            self.skipped[b] += int(skip.sum())
            y, g = y[keep], g[keep].astype(np.float64)
            step = max(1, (1 << 21) // (cb["K"] * d))
            for a in range(0, y.shape[0], step):
                z = ((y[a:a + step, None, :] - mu[None]) * isig[None]).astype(np.float64)
                ga = g[a:a + step]
                # sequential sums over the descriptors: cumsum from the running value
                self.S0[b] = np.cumsum(np.concatenate([self.S0[b][None], ga]), axis=0)[-1]
                self.S1[b] = np.cumsum(np.concatenate([self.S1[b][None], ga[:, :, None] * z]), axis=0)[-1]
                self.S2[b] = np.cumsum(np.concatenate([self.S2[b][None], ga[:, :, None] * (z * z)]), axis=0)[-1]

    def take(self):
        cb, K = self.cb, self.cb["K"]
        fv, stats = [], []
        for b, (_, _, d) in enumerate(cb["blocks"]):
            fv.append(fisher_normalize(self.S0[b], self.S1[b], self.S2[b], cb["w"][b], int(self.n[b])))
            stats += [self.S0[b], self.S1[b].ravel(), self.S2[b].ravel()]
        counters = {"pushed": int(self.pushed), "n": self.n.copy(), "skipped": self.skipped.copy()}
        out = np.concatenate(fv).astype(np.float32), np.concatenate(stats), counters
        self._reset()
        return out


def fisher_normalize(S0, S1, S2, w, N: int) -> np.ndarray:
    """One block's vector, float32 [u (K x dim), v (K x dim)]: u = S1 / (N sqrt(w)), v = (S2 - S0) / (N sqrt(2w)) in
    float64, t < 0 ? -sqrt(|t|) : sqrt(|t|), then divided by sqrt of the sum of squares (256 partials over the indices = j mod 256
    in increasing index, then the partials in increasing j) when that is > 0; zeros when N = 0."""
    K, d = S1.shape
    if N == 0:
        return np.zeros(2 * K * d, np.float32)
    wd = np.asarray(w, np.float32).astype(np.float64)
    u = S1 / (float(N) * np.sqrt(wd))[:, None]
    v = (S2 - S0[:, None]) / (float(N) * np.sqrt(2.0 * wd))[:, None]
    f = np.concatenate([u.ravel(), v.ravel()])
    r = np.sqrt(np.abs(f))
    f = np.where(f < 0, -r, r)
    sq = np.zeros(-(-f.size // 256) * 256)
    sq[:f.size] = f * f
    part = np.cumsum(sq.reshape(-1, 256), axis=0)[-1]
    norm = np.sqrt(np.cumsum(part)[-1])
    return (f / norm if norm > 0 else f).astype(np.float32)


def fisher_encode(desc, cb):
    """One clip's Fisher vector, bit for bit what one push of desc (n, desc_dim) and a take give: (fv, stats,
    counters)."""
    s = FisherStream(cb)
    s.push(desc)
    return s.take()


def fisher_pca(samples, blocks, dims):
    """Per block (offset, dim_in) with output size dims[b]: (mean float32, proj float32 (dim, dim_in), eigenvalues
    float64 (dim,)) -- float64 mean and covariance, eigh, the top dim components by eigenvalue (descending), each
    with the sign that makes its largest-magnitude entry positive (the first such entry on a tie)."""
    x = np.asarray(samples, np.float32).astype(np.float64)
    out = []
    for (o, di), d in zip(blocks, dims):
        xb = x[:, o:o + di]
        mean = xb.mean(axis=0)
        xc = xb - mean
        cov = xc.T @ xc / max(xb.shape[0] - 1, 1)
        ev, V = np.linalg.eigh(cov)
        order = np.argsort(-ev, kind="stable")[:d]
        P = V[:, order].T
        big = np.argmax(np.abs(P), axis=1)
        P = P * np.where(P[np.arange(d), big] < 0, -1.0, 1.0)[:, None]
        out.append((mean.astype(np.float32), P.astype(np.float32), ev[order]))
    return out


def _fisher_cb_params(K, mu, var, w):
    """isig, c, w of a block as float32 from float64 variances and weights: isig = 1/sqrt(var), c = log w - sum_d
    log sqrt(var)."""
    sig = np.sqrt(var)
    return ((1.0 / sig).astype(np.float32), (np.log(w) - np.log(sig).sum(axis=1)).astype(np.float32),
            np.asarray(w).astype(np.float32))


FISHER_EIG_FLOOR = 1e-12  # eigenvalues below this (degenerate data) are raised to it before they become variances


def fisher_init(samples, blocks, dims, K: int, seed: int):
    """The fit's initial codebook: PCA as fisher_pca; as means, the projections of K distinct samples drawn with
    splitmix64 from the seed (draw t = ((splitmix64(seed + (t+1) 0x9E3779B97F4A7C15) >> 32) * n) >> 32, repeats
    skipped); the eigenvalues as every Gaussian's variances; w = 1/K.  Returns (codebook, eigenvalues per block)."""
    x = np.asarray(samples, np.float32)
    n = x.shape[0]
    if n < K:
        raise ValueError("fisher_init: %d samples for K = %d" % (n, K))
    idx, seen, t = [], set(), 0
    while len(idx) < K:
        batch = np.arange(t + 1, t + 1 + 4 * K, dtype=np.uint64)
        with np.errstate(over="ignore"):
            z = splitmix64(np.uint64(seed % 2 ** 64) + batch * np.uint64(_SPLITMIX_GAMMA))
        for j in ((z >> np.uint64(32)) * np.uint64(n)) >> np.uint64(32):
            j = int(j)
            if j not in seen and len(idx) < K:
                seen.add(j)
                idx.append(j)
        t += 4 * K
    pca = fisher_pca(x, blocks, dims)
    cb = {"K": int(K), "desc_dim": int(x.shape[1]), "blocks": [(o, di, d) for (o, di), d in zip(blocks, dims)]}
    for k in FISHER_PARTS:
        cb[k] = []
    eigs = []
    for (o, di), (mean, P, ev) in zip(blocks, pca):
        ev = np.maximum(ev, FISHER_EIG_FLOOR)
        mu = fisher_project(x[idx, o:o + di], mean, P)
        isig, c, w = _fisher_cb_params(K, mu, np.tile(ev, (K, 1)), np.full(K, 1.0 / K))
        for k, v in zip(FISHER_PARTS, (mean, P, mu, isig, c, w)):
            cb[k].append(v)
        eigs.append(ev)
    return cb, eigs


def fisher_mstep(cb, stats, eigvals, var_floor: float):
    """The M-step from take's statistics, float64, with y = mu + z / isig: mu += (S1/S0) / isig, var = (S2/S0 -
    (S1/S0)^2) / isig^2 floored at var_floor * eigenvalue, w = S0 / sum S0; isig and c recomputed.  A Gaussian with
    S0 = 0 keeps its parameters."""
    K = cb["K"]
    out = {k: cb[k] for k in ("K", "desc_dim", "blocks", "mean", "proj")}
    for k in ("mu", "isig", "c", "w"):
        out[k] = []
    stats = np.asarray(stats, np.float64)
    p = 0
    for b, (_, _, d) in enumerate(cb["blocks"]):
        S0 = stats[p:p + K]
        S1 = stats[p + K:p + K + K * d].reshape(K, d)
        S2 = stats[p + K + K * d:p + K + 2 * K * d].reshape(K, d)
        p += K * (1 + 2 * d)
        mu0 = cb["mu"][b].astype(np.float64)
        is0 = cb["isig"][b].astype(np.float64)
        live = S0 > 0
        s0 = np.where(live, S0, 1.0)[:, None]
        r1, r2 = S1 / s0, S2 / s0
        mu = mu0 + r1 / is0
        var = np.maximum((r2 - r1 * r1) / (is0 * is0), var_floor * np.asarray(eigvals[b])[None, :])
        tot = S0.sum()
        w = S0 / tot if tot > 0 else np.full(K, 1.0 / K)
        isig, c, w32 = _fisher_cb_params(K, mu, var, np.where(live, w, 1.0))
        out["mu"].append(np.where(live[:, None], mu.astype(np.float32), cb["mu"][b]))
        out["isig"].append(np.where(live[:, None], isig, cb["isig"][b]))
        out["c"].append(np.where(live, c, cb["c"][b]))
        out["w"].append(np.where(live, w32, cb["w"][b]))
    return out


def fisher_fit(samples, blocks, dims, K: int = 256, iters: int = 10, seed: int = 0, var_floor: float = 1e-3,
               estep=None):
    """EM for a diagonal GMM per block on the PCA-projected samples: fisher_init, then `iters` rounds of an E-step
    (estep(codebook, samples) -> take's statistics; fisher_encode's by default) and fisher_mstep.  Context.fisher_fit
    runs the same loop with the E-step on the device, so both return the same codebook bytes."""
    x = np.asarray(samples, np.float32)
    cb, eigs = fisher_init(x, blocks, dims, K, seed)
    for _ in range(iters):
        stats = estep(cb, x) if estep is not None else fisher_encode(x, cb)[1]
        cb = fisher_mstep(cb, stats, eigs, var_floor)
    return cb
