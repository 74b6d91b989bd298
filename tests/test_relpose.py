"""preprocess.relpose, the restatement of ofdis_relpose_fullres: its eight-point solver and decomposition against a
plain float64 numpy reference built on the SVD, the full-pivot elimination's failures, the parallax guard, and the
fit on the exact flow of synth.rigid_stereo_clip."""
import math

import numpy as np
import pytest

from of_dis_b200 import preprocess, synth


def motion(w=(0.0, 0.0, 0.0), t=(0.0, 0.0, 0.0)):
    return np.concatenate([synth.axis_angle(w), np.asarray(t, np.float64).reshape(3, 1)], 1)


def rays(P, rng, m):
    """m noise-free normalized correspondences of random points in front of both cameras of the pose P."""
    X = np.stack([rng.uniform(-4, 4, m), rng.uniform(-2, 2, m), rng.uniform(4, 30, m)], -1)
    Y = X @ P[:, :3].T + P[:, 3]
    return X[:, :2] / X[:, 2:], Y[:, :2] / Y[:, 2:]


def reference_pose(x0, x1):
    """Textbook eight-point in float64: the SVD null vector, projection to rank 2, the four decompositions and the
    cheirality vote by linear triangulation."""
    A = np.stack([x1[:, 0] * x0[:, 0], x1[:, 0] * x0[:, 1], x1[:, 0], x1[:, 1] * x0[:, 0], x1[:, 1] * x0[:, 1],
                  x1[:, 1], x0[:, 0], x0[:, 1], np.ones(len(x0))], -1)
    E = np.linalg.svd(A)[2][-1].reshape(3, 3)
    U, _, Vt = np.linalg.svd(E)
    U *= np.sign(np.linalg.det(U))
    Vt *= np.sign(np.linalg.det(Vt))
    W = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    best, bestn = None, -1
    for R in (U @ W @ Vt, U @ W.T @ Vt):
        for t in (U[:, 2], -U[:, 2]):
            n = 0
            for a, b in zip(x0, x1):
                r0, r1 = np.append(a, 1.0), np.append(b, 1.0)
                M = np.stack([R @ r0, -r1], 1)
                lam = np.linalg.lstsq(M, -t, rcond=None)[0]
                n += int(lam[0] > 0 and lam[1] > 0)
            if n > bestn:
                best, bestn = (R, t), n
    return best


@pytest.mark.parametrize("P", [motion((0.0, 0.01, 0.0), (0.0, 0.0, -1.0)),
                               motion((0.0, 0.0, 0.02), (1.0, 0.0, 0.0)),
                               motion((0.02, -0.03, 0.01), (0.3, -0.2, -0.9))], ids=["forward", "sideways", "oblique"])
def test_solver_against_the_svd_reference(P):
    rng = np.random.default_rng(1)
    x0, x1 = rays(P, rng, 8)
    A = np.stack([x1[:, 0] * x0[:, 0], x1[:, 0] * x0[:, 1], x1[:, 0], x1[:, 1] * x0[:, 0], x1[:, 1] * x0[:, 1],
                  x1[:, 1], x0[:, 0], x0[:, 1], np.ones(8)], -1)
    e, ok = preprocess.relpose_null(A[None])
    assert ok[0]
    Rr, tr = reference_pose(x0, x1)
    cands = preprocess.relpose_decompose(e[0])
    votes = [int(preprocess.relpose_front(R, t, x0[:, 0], x0[:, 1], x1[:, 0], x1[:, 1]).sum()) for R, t in cands]
    R, t = cands[int(np.argmax(votes))]
    assert max(votes) == 8
    tt = P[:, 3] / np.linalg.norm(P[:, 3])
    assert np.abs(R.reshape(3, 3) - Rr).max() < 1e-9 and np.abs(t - tr).max() < 1e-9
    assert np.abs(R.reshape(3, 3) - P[:, :3]).max() < 1e-9 and np.abs(t - tt).max() < 1e-9


def test_elimination_fails_on_degenerate_draws():
    rng = np.random.default_rng(2)
    x0, x1 = rays(motion((0.0, 0.01, 0.0), (0.0, 0.0, -1.0)), rng, 8)
    A = np.stack([x1[:, 0] * x0[:, 0], x1[:, 0] * x0[:, 1], x1[:, 0], x1[:, 1] * x0[:, 0], x1[:, 1] * x0[:, 1],
                  x1[:, 1], x0[:, 0], x0[:, 1], np.ones(8)], -1)
    rep = A.copy()
    rep[5] = rep[2]                       # a repeated draw: its row eliminates to exactly zero
    zero = np.zeros_like(A)               # no pivot > 0 at all
    nan = A.copy()
    nan[0, 0] = np.nan                    # NaN is never a pivot; the solution is not finite
    e, ok = preprocess.relpose_null(np.stack([A, rep, zero, nan]))
    assert ok.tolist() == [True, False, False, False]
    assert abs(np.linalg.norm(e[0]) - 1.0) < 1e-15
    # a rank-1 E: u1 x E v2 is zero, and the decomposition gives NaN candidates (as the device) instead of raising
    cands = preprocess.relpose_decompose(np.array([1.0, 0, 0, 0, 0, 0, 0, 0, 0]))
    assert all(np.isnan(t).all() for _, t in cands)


def test_refit_on_the_exact_flow_of_a_synthetic_clip():
    """KITTI's size and camera, the clip's exact flow: the pose within 1e-4 degrees and the depth equal to
    fb / (disp + doffs) / |t| on the static background."""
    h, w, n = 375, 1242, 2
    cam = dict(fx=721.5, fy=721.5, cx=609.6, cy=172.9, baseline=0.54, doffs=0.0)
    rels = [motion((0.0, math.radians(0.5), 0.0), (0.0, 0.0, -0.9)),
            motion((math.radians(0.3), math.radians(-0.8), 0.0), (0.1, 0.0, -0.6))]
    clip = synth.rigid_stereo_clip(n, h, w, 1, 2, cam, rels)
    p = dict(fx=721.5, fy=721.5, cx=609.6, cy=172.9, step=8, fb_check=0, alpha=0.01, beta=0.5, hypotheses=256,
             threshold=0.05, refine=5, min_parallax=0.5, seed=0)
    pose, st, mask, samp, depth = preprocess.relpose(clip["flow"].astype(np.float32), None, p)
    assert (st["status"] == 0).all(), st
    r_err, t_err = preprocess.relpose_errors(pose, clip["poses"])
    assert (r_err < 1e-4).all() and (t_err < 1e-4).all(), (r_err, t_err)
    assert np.abs(np.linalg.norm(pose[:, :, 3], axis=1) - 1.0).max() < 1e-12
    fb = float(np.float32(np.float32(cam["fx"]) * np.float32(cam["baseline"])))
    for k in range(n):
        true = fb / (clip["disp"][k].astype(np.float64) + cam["doffs"]) / np.linalg.norm(clip["poses"][k][:, 3])
        sel = (mask[k] == 0) & ~clip["box"][k] & np.isfinite(depth[k])
        assert sel.mean() > 0.5
        rel = np.abs(depth[k][sel] - true[sel]) / true[sel]
        assert np.median(rel) < 1e-3, np.median(rel)
        assert (mask[k][clip["box"][k]] != 0).mean() > 0.9
        assert np.isnan(samp[k][mask[k] == 2]).all() and (samp[k][mask[k] == 0] <= np.float32(0.05)).all()


def test_zero_translation_gives_status_3():
    """A zero flow and a pure rotation of a static scene: the derotated flow of the pose's twisted pair is ~0, so the
    guard reports status 3 even though the cheirality vote may pick the twisted candidate."""
    h, w = 120, 200
    cam = dict(fx=180.0, fy=180.0, cx=99.5, cy=59.5, baseline=0.54, doffs=0.0)
    p = dict(fx=180.0, fy=180.0, cx=99.5, cy=59.5, step=2, fb_check=0, alpha=0.01, beta=0.5, hypotheses=128,
             threshold=1.0, refine=5, min_parallax=0.5, seed=0)
    static = dict(velocity=(0.0, 0.0, 0.0))  # a moving object is real parallax
    rot = synth.rigid_stereo_clip(1, h, w, 1, 2, cam, [motion((0.0, 0.02, 0.0))], block=static)
    flows = np.stack([np.zeros((h, w, 2), np.float32), rot["flow"][0].astype(np.float32)])
    st = preprocess.relpose(flows, None, p)[1]
    assert st["status"].tolist() == [3, 3], st


def test_chain_poses_with_scales():
    rels = np.stack([motion((0.0, 0.01, 0.0), (0.0, 0.0, -1.0)), motion((0.01, 0.0, 0.0), (0.6, 0.0, -0.8))])
    unit = rels.copy()
    unit[:, :, 3] /= np.linalg.norm(unit[:, :, 3], axis=1, keepdims=True)
    got = preprocess.chain_poses(unit, np.linalg.norm(rels[:, :, 3], axis=1))
    assert np.abs(got - preprocess.chain_poses(rels)).max() < 1e-12
    assert np.array_equal(preprocess.chain_poses(rels), preprocess.chain_poses(rels, None))


def test_relpose_errors():
    P = motion((0.0, 0.01, 0.0), (0.0, 0.0, -1.0))
    Q = motion((0.0, 0.01 + math.radians(0.5), 0.0), (math.tan(math.radians(2.0)), 0.0, -1.0))
    r, t = preprocess.relpose_errors(np.stack([P, Q]), np.stack([P, P]))
    assert abs(r[0]) < 1e-6 and abs(t[0]) < 1e-6
    assert abs(r[1] - 0.5) < 1e-6 and abs(t[1] - 2.0) < 1e-6
