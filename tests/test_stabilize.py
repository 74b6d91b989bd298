"""preprocess.stabilize, the restatement of ofdis_stab_begin / ofdis_stab_push / ofdis_stab_finish: exact weighted
means on translation clips, the same output however a clip is cut into pushes, the rules for invalid models and
undefined paths, the limit, the jitter it removes from synth.shaky_clip, and the batch command's refusals."""
from fractions import Fraction

import numpy as np
import pytest

from of_dis_b200 import preprocess, synth


def sp(radius, crop=0.0, limit=0):
    return dict(radius=radius, crop=crop, limit=limit)


def translations(shifts):
    out = np.zeros((len(shifts), 3, 3))
    for k, (dx, dy) in enumerate(shifts):
        out[k] = [[1, 0, dx], [0, 1, dy], [0, 0, 1]]
    return out


def mapped(A, x, y):
    q = A[2, 0] * x + A[2, 1] * y + A[2, 2]
    return np.stack([(A[0, 0] * x + A[0, 1] * y + A[0, 2]) / q, (A[1, 0] * x + A[1, 1] * y + A[1, 2]) / q], -1)


def jitter(models, corrections, h, w, step=16):
    """Mean over a pixel grid and over t of |D_t(x) - D_{t-1}(x)|, D_t the displacement of the stabilised inter-frame
    motion S_{t+1} M_t S_t^-1 (the raw motion with identity corrections)."""
    y, x = np.mgrid[0:h:step, 0:w:step].astype(np.float64)
    D = []
    for t in range(len(models)):
        A = corrections[t + 1] @ models[t] @ np.linalg.inv(corrections[t])
        D.append(mapped(A, x, y) - np.stack([x, y], -1))
    return float(np.mean([np.linalg.norm(D[t] - D[t - 1], axis=-1).mean() for t in range(1, len(D))]))


def corrections(info):
    return info["correction"].reshape(-1, 3, 3)


class Streaming:
    """The stabiliser as ofdis_stab_push / ofdis_stab_finish run it: only the frames not emitted yet and the models
    their windows still need are kept (a KeyError would show a window reaching past them)."""

    def __init__(self, params, weights, frame0):
        self.p, self.wts, self.r = params, weights, params["radius"]
        self.frames, self.models = {0: frame0}, {}
        self.last, self.next = 0, 0

    def _emit(self, upto, cut):
        h, w = self.frames[self.next].shape[:2]
        out, info = [], []
        while self.next <= upto:
            t = self.next
            b = min(self.last, t + self.r) if cut else t + self.r
            S = preprocess.stab_path(self.models, t, max(0, t - self.r), b, self.wts)
            status, lam, SL, a = preprocess.stab_correction(S, self.p, w, h)
            out.append(preprocess.stab_warp(self.frames.pop(t), a))
            info.append((t, status, lam, SL))
            self.next += 1
        for k in [k for k in self.models if k < self.next - self.r]:
            del self.models[k]
        return out, info

    def push(self, models, frames):
        for k, (m, f) in enumerate(zip(models, frames)):
            self.models[self.last + k] = preprocess.stab_model(m)
            self.frames[self.last + 1 + k] = f
        self.last += len(frames)
        return self._emit(self.last - self.r, False)

    def finish(self):
        return self._emit(self.last, True)


def streamed(frames, models, params, weights, cuts):
    s = Streaming(params, weights, frames[0])
    out, info = [], []
    k = 1
    for c in cuts:
        o, i = s.push(models[k - 1:k - 1 + c], frames[k:k + c])
        out += o
        info += i
        k += c
    o, i = s.finish()
    rec = np.array([tuple(x) for x in info + i], preprocess.STAB_FRAME_DTYPE)
    return np.stack(out + o), rec


def same_bits(a, b):
    """Bitwise equal arrays; records field by field (their padding is not compared)."""
    if a.dtype.names:
        return a.dtype == b.dtype and all(same_bits(a[k], b[k]) for k in a.dtype.names)
    return a.shape == b.shape and np.ascontiguousarray(a).tobytes() == np.ascontiguousarray(b).tobytes()


@pytest.mark.parametrize("r", [1, 2, 4])
def test_translation_paths_are_exact_weighted_means(r):
    """Dyadic shifts and weights: every sum is exact, so S_t is the correctly rounded weighted mean of the shifts from
    frame t into its window, at both truncated ends too."""
    rng = np.random.default_rng(r)
    n = 13
    shifts = rng.integers(-64, 64, (n - 1, 2)) / 16.0
    weights = [1.0 / (1 << d) for d in range(r + 1)]
    frames = np.zeros((n, 6, 8), np.uint8)
    _, info = preprocess.stabilize(frames, translations(shifts), sp(r), weights)
    for t in range(n):
        num, den = [Fraction(0), Fraction(0)], Fraction(0)
        for u in range(max(0, t - r), min(n - 1, t + r) + 1):
            wd = Fraction(weights[abs(u - t)])
            lo, hi = min(t, u), max(t, u)
            for c in range(2):
                off = sum((Fraction(float(s)) for s in shifts[lo:hi, c]), Fraction(0))
                num[c] += wd * (off if u >= t else -off)
            den += wd
        S = info["correction"][t]
        assert S[2] == float(num[0] / den) and S[5] == float(num[1] / den), (t, S)
        assert list(S[[0, 1, 3, 4, 6, 7, 8]]) == [1, 0, 0, 1, 0, 0, 1]
        assert info["status"][t] == 0 and info["lambda"][t] == 1.0 and info["frame"][t] == t


@pytest.mark.parametrize("ch", [1, 3])
@pytest.mark.parametrize("cuts", [[1] * 11, [3, 5, 3], [11], [2, 1, 4, 4]], ids=["ones", "3-5-3", "whole", "mixed"])
def test_any_split_into_pushes_gives_the_same_output(cuts, ch):
    frames, models, _ = synth.shaky_clip(12, 24, 32, ch, seed=5, pan=(0.5, 0.25), jitter=1.5)
    for p in (sp(4, 0.1, 1), sp(1, 0.0, 0), sp(3, 0.2, 0)):
        wts = preprocess.gaussian_weights(p["radius"])
        out, info = preprocess.stabilize(frames, models, p, wts)
        got, ginfo = streamed(frames, models, p, wts, cuts)
        assert same_bits(got, out) and same_bits(ginfo, info), (p, cuts)


def test_clip_shorter_than_the_radius():
    frames, models, _ = synth.shaky_clip(3, 16, 20, 1, seed=2)
    p = sp(8, 0.05, 1)
    wts = preprocess.gaussian_weights(8)
    out, info = preprocess.stabilize(frames, models, p, wts)
    got, ginfo = streamed(frames, models, p, wts, [2])
    assert same_bits(got, out) and same_bits(ginfo, info)
    assert list(info["frame"]) == [0, 1, 2]


def test_invalid_models_are_the_identity():
    frames, models, _ = synth.shaky_clip(8, 16, 20, 1, seed=3)
    bad = models.copy()
    bad[1] = np.nan                                        # a status != 0 pair
    bad[2, 2, 2] = 0.0                                     # m22 = 0
    bad[3] = [[1, 2, 0], [2, 4, 0], [0, 0, 1]]             # singular: m00*m11 - m01*m10 = 0
    bad[4] = [[1e300, 0, 0], [0, 1e300, 0], [0, 0, 1e-300]]  # an entry of the divided model overflows
    eye = models.copy()
    eye[1:5] = np.eye(3)
    for p in (sp(2), sp(3, 0.1, 1)):
        wts = preprocess.gaussian_weights(p["radius"])
        a = preprocess.stabilize(frames, bad, p, wts)
        b = preprocess.stabilize(frames, eye, p, wts)
        assert same_bits(a[0], b[0]) and same_bits(a[1], b[1])
    # a model is divided by its m22 first
    scaled = models.copy()
    scaled[0] *= 4.0
    assert same_bits(preprocess.stabilize(frames, scaled, sp(2), [1.0, 0.5, 0.25])[1],
                     preprocess.stabilize(frames, models, sp(2), [1.0, 0.5, 0.25])[1])


def test_a_chain_through_p22_zero_is_undefined():
    """M_0 shifts x by 1 and M_1 has the row (-1, 0, 1): (M_1 M_0)_22 = 0, so the forward path of frame 0 is undefined
    at d = 2; frames whose windows do not hold both models keep a defined path."""
    models = np.stack([np.eye(3)] * 5)
    models[0] = [[1, 0, 1], [0, 1, 0], [0, 0, 1]]
    models[1] = [[1, 0, 0], [0, 1, 0], [-1, 0, 1]]
    frames = np.full((6, 10, 12), 200, np.uint8)
    for p in (sp(2), sp(2, 0.1, 1)):
        out, info = preprocess.stabilize(frames, models, p, [1.0, 1.0, 1.0])
        assert info["status"][0] == 1 and info["lambda"][0] == 0.0
        assert (info["correction"][0] == np.eye(3).reshape(-1)).all()
        assert list(info["status"][3:]) == [0, 0, 0]
        if p["crop"] == 0:
            assert (out[0] == frames[0]).all(), "the identity correction without crop keeps the frame"


def test_the_limit_keeps_the_corners_inside():
    h, w = 48, 64
    frames, models, _ = synth.shaky_clip(16, h, w, 1, seed=4, pan=(0.0, 0.0), jitter=6.0)
    corners = np.array([[0, 0], [w - 1, 0], [0, h - 1], [w - 1, h - 1]], np.float64)
    for crop in (0.0, 0.05, 0.2):
        _, info = preprocess.stabilize(frames, models, sp(4, crop, 1), preprocess.gaussian_weights(4))
        s = 1 - 2 * float(np.float32(crop))
        c = (0.5 * (w - 1), 0.5 * (h - 1))
        Z = np.array([[s, 0, c[0] * (1 - s)], [0, s, c[1] * (1 - s)], [0, 0, 1]])
        for t in range(len(frames)):
            A = np.linalg.inv(corrections(info)[t]) @ Z
            q = mapped(A, corners[:, 0], corners[:, 1])
            assert (q >= -1e-3).all() and (q[:, 0] <= w - 1 + 1e-3).all() and (q[:, 1] <= h - 1 + 1e-3).all(), (crop, t)
        if crop == 0.0:
            assert (info["lambda"] < 1).all()
        if crop == 0.2:
            assert (info["lambda"] < 1).sum() < len(frames)
    # small corrections inside a generous crop are kept whole
    frames, models, _ = synth.shaky_clip(16, h, w, 1, seed=4, jitter=0.5)
    _, info = preprocess.stabilize(frames, models, sp(4, 0.1, 1), preprocess.gaussian_weights(4))
    assert (info["lambda"] == 1.0).all() and (info["status"] == 0).all()


# Measured on the true models of shaky_clip(24, 218, 512, seed 0, pan (1, 0.5), jitter 2) at r = 8, crop 0.1 with the
# limit (which keeps every correction whole there, lambda = 1): the raw jitter is 4.23 px, the stabilised one 0.086 px,
# a factor of 49.  The test asks for 40.
JITTER_FACTOR = 40.0


def test_stabilisation_removes_the_shake():
    h, w = 218, 512
    frames, models, smooth = synth.shaky_clip(24, h, w, 1, seed=0, pan=(1.0, 0.5), jitter=2.0)
    eye = np.stack([np.eye(3)] * len(frames))
    raw = jitter(models, eye, h, w)
    ideal = jitter(models, smooth, h, w)
    assert ideal < 1e-9 * raw + 1e-6, "the true corrections leave the pan alone"
    _, info = preprocess.stabilize(frames, models, sp(8, 0.1, 1), preprocess.gaussian_weights(8))
    stab = jitter(models, corrections(info), h, w)
    assert raw / stab >= JITTER_FACTOR, (raw, stab)


def test_gaussian_weights():
    assert preprocess.gaussian_weights(1) == [1.0, np.exp(-0.5)]
    w = preprocess.gaussian_weights(15)
    assert len(w) == 16 and w[0] == 1.0 and all(a > b > 0 for a, b in zip(w, w[1:]))
    assert preprocess.gaussian_weights(4, sigma=2.0) == preprocess.gaussian_weights(4)


@pytest.mark.parametrize("exe,args", [
    ("run_DE_INT", ["--global-motion", "homography", "gm.txt", "--stabilize", "4", "0.1", "out"]),
    ("run_DE_RGB", ["--stabilize", "4", "0.1", "out"]),
    ("run_OF_INT", ["--warm-start", "--global-motion", "homography", "gm.txt", "--stabilize", "4", "0.1", "out"]),
    ("run_OF_INT", ["--stabilize", "4", "0.1", "out"]),
    ("run_OF_RGB", ["--global-motion", "affine", "gm.txt", "--stabilize", "0", "0.1", "out"]),
    ("run_OF_RGB", ["--global-motion", "affine", "gm.txt", "--stabilize", "65", "0.1", "out"]),
    ("run_OF_INT", ["--global-motion", "affine", "gm.txt", "--stabilize", "4", "0.5", "out"]),
    ("run_OF_INT", ["--global-motion", "affine", "gm.txt", "--stabilize", "4", "-0.1", "out"]),
    ("run_OF_INT", ["--global-motion", "affine", "gm.txt", "--stabilize", "4", "nan", "out"]),
    ("run_OF_INT", ["--global-motion", "affine", "gm.txt", "--stabilize", "4x", "0.1", "out"]),
    ("run_OF_INT", ["--global-motion", "affine", "gm.txt", "--stabilize", "4", "0.1", "missing/dir"]),
    ("run_OF_INT", ["--global-motion", "affine", "gm.txt", "--stabilize", "4", "0.1"]),
])
def test_batch_command_refuses_stabilize(tmp_path, exe, args):
    """The stereo binaries, --warm-start, --stabilize without --global-motion, a radius outside 1..64, a crop outside
    [0, 0.5) and an unwritable directory are refused before any work."""
    import subprocess

    from of_dis_b200 import build

    bindir = build.build_host()
    (tmp_path / "out").mkdir()
    lst = tmp_path / "list.txt"
    lst.write_text("")
    r = subprocess.run([str(bindir) + "/" + exe + "_batch", str(lst)] + args, capture_output=True, text=True,
                       cwd=str(tmp_path))
    assert r.returncode == 2 or (r.returncode == 1 and "missing/dir" in args), (args, r.stdout, r.stderr)
    assert not (tmp_path / "gm.txt").exists() and not list((tmp_path / "out").iterdir())


def test_batch_command_accepts_stabilize(tmp_path):
    import subprocess

    from of_dis_b200 import build

    bindir = build.build_host()
    lst = tmp_path / "list.txt"
    lst.write_text("")
    r = subprocess.run([str(bindir) + "/run_OF_RGB_batch", str(lst), "--global-motion", "homography", "gm.txt",
                        "--stabilize", "15", "0.1", "."], capture_output=True, text=True, cwd=str(tmp_path))
    assert r.returncode == 0, (r.stdout, r.stderr)
    assert (tmp_path / "stab.txt").read_text() == ""
