"""The lazily allocated workspaces of the C-ABI's stages outside ofdis_run.

Grow-only workspaces: one context calls a stage at a small geometry, then at a larger one that reallocates the
workspace, then at the small one again; each result must be bitwise what the same call gives on a fresh context.  The
parameter that grows each one: the tracker's and the descriptor stage's capacity and spacing, the stabiliser's radius,
the Fisher encoder's K, the fusion volume's nx * ny * nz (and with it the mesh's), the fused tracking's step, and the
hypotheses and step of global motion and ego-motion.

Host scratch: host-memory outputs go through one scratch that is at least what ofdis_get_flow_fullres asks for.  Each
path's host output must equal its device output at n < max_frames and at n = max_frames, interleaved with host
get_flow_fullres calls whose flows must not change.  Paths compared elsewhere: confidence
(test_confidence_gpu.py), disparity (test_disparity_gpu.py), interpolation (test_interpolate_gpu.py), the
stabiliser (test_stabilize_gpu.py), fusion push, extract and render (test_fusion_gpu.py), the mesh
(test_fusion_mesh_gpu.py) and fused tracking (test_fusion_track_gpu.py)."""
import numpy as np
import pytest

from of_dis_b200 import params, preprocess, synth

pytestmark = pytest.mark.gpu

f32 = np.float32
LEVEL0 = "3 0 8 8 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0"  # sc_l 0: the level-0 flows are the full-resolution ones
H, W, N = 48, 64, 3  # frame size, pairs; slots 0 .. N-1 hold the forward flows, N .. 2N-1 the backward ones
CAM = dict(fx=60.0, fy=58.5, cx=31.25, cy=23.5, baseline=0.5, doffs=0.25)


@pytest.fixture(scope="module")
def api():
    from of_dis_b200 import api as _api

    _api.lib()
    return _api


def flows(n, nop):
    """(F, B): n smooth forward flows (n, H, W, nop) and B = -F."""
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    F = np.empty((n, H, W, nop), f32)
    for k in range(n):
        u = 0.6 + 0.4 * k + 1.5 * np.sin(x / 9.0 + k) * np.cos(y / 7.0)
        v = -0.3 + 1.2 * np.cos(x / 11.0) * np.sin(y / 6.0 + 0.5 * k)
        F[k] = np.stack([u, v], -1)[..., :nop]
    return F, -F


def clip(n=N):
    return synth.synthetic_sequence(n + 1, H, W, 1, seed=41, amp=3.0)


def disparities(n=N + 1):
    """n positive disparity maps of a wavy surface at about 1.3 m, with some unknown."""
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    rng = np.random.default_rng(5)
    d = np.empty((n, H, W), f32)
    for k in range(n):
        Z = 1.3 + 0.03 * np.sin(x / 6.0 + k) + 0.002 * y
        d[k] = (f32(CAM["fx"] * CAM["baseline"]) / Z - CAM["doffs"]).astype(f32)
    d[rng.random(d.shape) < 0.03] = np.nan
    return d


def context(api, nop=2, max_frames=2 * N):
    prm = params.from_cli_numbers(LEVEL0.split(), noc=1, nop=nop)
    ctx = api.Context(prm, W, H, prm.p_samp_s, max_frames)
    F, B = flows(max_frames // 2, nop)
    for k in range(max_frames // 2):
        ctx.set_flow(k, 0, F[k])
        ctx.set_flow(max_frames // 2 + k, 0, B[k])
    return ctx


def bits(x):
    """A result as a flat list that compares bitwise; records field by field, so that padding bytes (which the
    kernels leave unwritten, as in ofdis_stab_frame) do not count."""
    if isinstance(x, np.ndarray) and x.dtype.names:
        return [b for f in x.dtype.names for b in [f] + bits(x[f])]
    if isinstance(x, np.ndarray):
        return [(x.dtype.str, x.shape, np.ascontiguousarray(x).tobytes())]
    if isinstance(x, dict):
        return [b for k in sorted(x) for b in [k] + bits(x[k])]
    if isinstance(x, (list, tuple)):
        return [b for v in x for b in bits(v)]
    return [repr(x)]


def pose(t=(0.0, 0.0, 0.0)):
    return np.concatenate([np.eye(3), np.asarray(t, np.float64).reshape(3, 1)], 1)


# ---- grow-only workspaces ----------------------------------------------------------------------------------------
def track_params(capacity, spacing):
    return dict(capacity=capacity, spacing=spacing, alpha=0.01, beta=0.5, mb_alpha=0.01, mb_beta=0.002, min_eig=1.0)


def run_track(ctx, g):
    c = clip()
    lists = [ctx.track_begin(track_params(*g), c[0], W, H)] + ctx.track_advance(0, N, N, c[1:], W, H)
    return lists, ctx.track_stats()


def run_traj(ctx, g):
    c = clip()
    tp = dict(L=2, nt=1, N=8, ns=2, min_flow=0.1, eps=0.05, min_disp=0.0, min_var=0.0, max_var=1e9, max_dis=1e9)
    first = ctx.traj_begin(track_params(*g), tp, c[0], W, H)
    return first, ctx.traj_advance(0, N, N, c[1:], W, H), ctx.traj_stats(), ctx.track_stats()


def run_stab(ctx, radius):
    c = clip()
    models = np.stack([np.array([[1.0, 0.002 * k, 0.4 - 0.2 * k], [-0.002 * k, 1.0, 0.3], [0.0, 0.0, 1.0]])
                       for k in range(N)])
    ctx.stab_begin(dict(radius=radius, crop=0.1, limit=1), c[0], W, H)
    return ctx.stab_push(models, c[1:]), ctx.stab_finish()


def run_fisher(ctx, K):
    rng = np.random.default_rng(K)
    blocks = [(0, 8, 4), (8, 12, 6)]
    cb = {"K": K, "desc_dim": 20, "blocks": blocks}
    for k in preprocess.FISHER_PARTS:
        cb[k] = []
    for _, di, d in blocks:
        w = rng.uniform(0.2, 1.0, K)
        w /= w.sum()
        sig = rng.uniform(0.3, 1.5, (K, d))
        cb["mean"].append(rng.normal(0, 0.1, di).astype(f32))
        cb["proj"].append(rng.normal(0, 1.0 / np.sqrt(di), (d, di)).astype(f32))
        cb["mu"].append(rng.normal(0, 0.3, (K, d)).astype(f32))
        cb["isig"].append((1.0 / sig).astype(f32))
        cb["c"].append((np.log(w) - np.log(sig).sum(1)).astype(f32))
        cb["w"].append(w.astype(f32))
    ctx.fisher_begin(cb)
    ctx.fisher_push(np.random.default_rng(9).normal(0, 1, (300, 20)).astype(f32))
    return ctx.fisher_take()


def volume(n):
    """n^3-ish voxels of 0.1 m from (-0.8, -0.6, 0.9): the surface lies inside at every size."""
    return dict(nx=n, ny=3 * n // 4, nz=n, origin=(-0.8, -0.6, 0.9), voxel=0.1 * 16 / n, trunc=0.2, max_weight=6.0,
                color=0)


def run_fuse(ctx, n):
    d = disparities()
    poses = np.stack([pose((0.01 * k, 0.0, 0.0)) for k in range(N)])
    ctx.fuse_begin(volume(n))
    ctx.fuse_push(d[:N], poses, CAM, width_org=W, height_org=H)
    render = ctx.fuse_render(poses[:1], CAM, z_near=0.5, z_far=2.5, step=0.02, width_org=W, height_org=H)
    return ctx.fuse_extract(), render, ctx.fuse_mesh(), ctx.fuse_volume()


def run_fuse_track(ctx, step):
    d = disparities()
    tp = dict(step=step, rounds=4, min_weight=1.0, max_depth=float("inf"), huber=0.3, damping=0.0, min_corr=6,
              max_shift=0.5, min_cos=0.99, eps=0.0, integrate=1)
    ctx.fuse_begin(volume(16))
    ctx.fuse_push(d[:1], pose()[None], CAM, width_org=W, height_org=H)
    return ctx.fuse_track(d[1:], None, pose(), CAM, tp, width_org=W, height_org=H), ctx.fuse_volume()


def motion_params(g):
    step, hyps = g
    return dict(model="affine", step=step, fb_check=1, alpha=0.01, beta=0.5, hypotheses=hyps, threshold=1.0, refine=3,
                seed=11)


def run_motion(ctx, g):
    c = clip()
    outs = dict(mask=np.empty((N, H, W), np.uint8), residual=np.empty((N, H, W, 2), f32),
                registered=np.empty((N, H, W), np.uint8))
    models, stats = ctx.global_motion_fullres(0, N, motion_params(g), width_org=W, height_org=H, b0=N, i1=c[1:], **outs)
    return models, stats, outs


def run_ego(ctx, g):
    step, hyps = g
    d = disparities()
    p = dict(step=step, fb_check=1, alpha=0.01, beta=0.5, edge_diff=1.0, hypotheses=hyps, threshold=1.0, refine=5,
             seed=3)
    return ctx.egomotion_fullres(0, N, d[:N], d[1:], p, camera=CAM, width_org=W, height_org=H, b0=N,
                                 outputs=("mask", "residual", "object_motion"))


GROW = {  # name: (call, small, large)
    "track": (run_track, (256, 4), (4096, 1)),
    "traj": (run_traj, (256, 4), (4096, 1)),
    "stab": (run_stab, 1, 9),
    "fisher": (run_fisher, 2, 48),
    "fuse+mesh": (run_fuse, 16, 40),
    "fuse_track": (run_fuse_track, 4, 1),
    "global_motion": (run_motion, (8, 16), (2, 512)),
    "egomotion": (run_ego, (8, 16), (2, 512)),
}


@pytest.mark.parametrize("name", list(GROW))
def test_grown_workspace_equals_a_fresh_one(name, api):
    call, small, large = GROW[name]
    ctx = context(api)
    got = [call(ctx, g) for g in (small, large, small)]
    ctx.close()
    for g, r in zip((small, large, small), got):
        fresh = context(api)
        exp = call(fresh, g)
        fresh.close()
        assert bits(r) == bits(exp), "%s at %s differs from a fresh context" % (name, g)


# ---- host scratch ------------------------------------------------------------------------------------------------
def device(shape, dtype):
    import torch

    return torch.empty(int(np.prod(shape)) * np.dtype(dtype).itemsize, dtype=torch.uint8, device="cuda"), shape, dtype


def host_of(buf):
    t, shape, dtype = buf
    return t.cpu().numpy().view(dtype).reshape(shape)


def consistency(ctx, n, mem):
    mf = 2 * N
    if mem == "host":
        return ctx.consistency_fullres(0, n, mf - n, W, H, with_err=True)
    m, e = device((n, H, W), np.uint8), device((n, H, W), f32)
    ctx.consistency_fullres(0, n, mf - n, W, H, with_err=True, memkind=1, mask=m[0].data_ptr(), err=e[0].data_ptr())
    ctx.sync()
    return host_of(m), host_of(e)


def color(ctx, n, mem):
    if mem == "host":
        return ctx.flow_color_fullres(0, n, W, H, with_scale=True)
    o, s = device((n, H, W, 3), np.uint8), device((n,), f32)
    ctx.flow_color_fullres(0, n, W, H, out=o[0].data_ptr(), scale=s[0].data_ptr(), memkind=1)
    ctx.sync()
    return host_of(o), host_of(s)


def encoded(ctx, n, mem):
    if mem == "host":
        return ctx.get_flow_fullres_encoded(0, n, "kitti", W, H)
    o = device((n, H, W, 3), np.uint16)
    ctx.get_flow_fullres_encoded(0, n, "kitti", W, H, out=o[0].data_ptr(), memkind=1)
    ctx.sync()
    return host_of(o)


def flow_error(ctx, n, mem):
    import torch

    gt = flows(2 * N, 2)[0][:n] * f32(1.1)
    cls = (np.arange(n * H * W) % 3).astype(np.uint8).reshape(n, H, W)
    if mem == "host":
        return ctx.flow_error_fullres(0, n, gt, W, H, classes=cls, nclasses=3, with_err=True)
    dgt, dcls = torch.from_numpy(gt).cuda(), torch.from_numpy(cls).cuda()
    e = device((n, H, W), f32)
    torch.cuda.synchronize()
    stats, _ = ctx.flow_error_fullres(0, n, dgt.data_ptr(), W, H, classes=dcls.data_ptr(), nclasses=3, memkind=1,
                                      err=e[0].data_ptr())
    return stats, host_of(e)


def global_motion(ctx, n, mem):
    import torch

    c = clip(2 * N)
    p = motion_params((4, 64))
    if mem == "host":
        return run_motion_n(ctx, n, p, c)
    di1 = torch.from_numpy(np.ascontiguousarray(c[1:n + 1])).cuda()
    m, r, g = device((n, H, W), np.uint8), device((n, H, W, 2), f32), device((n, H, W), np.uint8)
    torch.cuda.synchronize()
    models, stats = ctx.global_motion_fullres(0, n, dict(p, fb_check=0), width_org=W, height_org=H,
                                              i1=di1.data_ptr(), mask=m[0].data_ptr(), residual=r[0].data_ptr(),
                                              registered=g[0].data_ptr(), memkind=1)
    return models, stats, host_of(m), host_of(r), host_of(g)


def run_motion_n(ctx, n, p, c):
    m, r, g = np.empty((n, H, W), np.uint8), np.empty((n, H, W, 2), f32), np.empty((n, H, W), np.uint8)
    models, stats = ctx.global_motion_fullres(0, n, dict(p, fb_check=0), width_org=W, height_org=H, i1=c[1:n + 1],
                                              mask=m, residual=r, registered=g)
    return models, stats, m, r, g


def egomotion(ctx, n, mem):
    import torch

    d = disparities(2 * N + 1)
    p = dict(step=4, fb_check=0, alpha=0.01, beta=0.5, edge_diff=1.0, hypotheses=64, threshold=1.0, refine=5, seed=3)
    outs = ("mask", "residual", "object_motion")
    if mem == "host":
        return ctx.egomotion_fullres(0, n, d[:n], d[1:n + 1], p, camera=CAM, width_org=W, height_org=H, outputs=outs)
    dd = torch.from_numpy(d).cuda()
    bufs = dict(mask=device((n, H, W), np.uint8), residual=device((n, H, W, 2), f32),
                object_motion=device((n, H, W, 3), f32))
    torch.cuda.synchronize()
    pose_, stats, _ = ctx.egomotion_fullres(0, n, dd[:n].data_ptr(), dd[1:].data_ptr(), p, camera=CAM, width_org=W,
                                            height_org=H, outputs=outs, out={k: b[0].data_ptr() for k, b in
                                                                             bufs.items()}, memkind=1)
    ctx.sync()
    return pose_, stats, {k: host_of(b) for k, b in bufs.items()}


def scene_flow(ctx, n, mem):
    import torch

    d = disparities(2 * N + 1)
    outs = ("disp1", "status", "motion")
    if mem == "host":
        return ctx.scene_flow_fullres(0, n, d[:n], d[1:n + 1], width_org=W, height_org=H, camera=CAM, outputs=outs)[0]
    dd = torch.from_numpy(d).cuda()
    bufs = {"disp1": device((n, H, W), f32), "status": device((n, H, W), np.uint8),
            "motion": device((n, H, W, 3), f32)}
    torch.cuda.synchronize()
    ctx.scene_flow_fullres(0, n, dd[:n].data_ptr(), dd[1:].data_ptr(), width_org=W, height_org=H, camera=CAM,
                           outputs=outs, out={k: b[0].data_ptr() for k, b in bufs.items()}, memkind=1)
    ctx.sync()
    return {k: host_of(b) for k, b in bufs.items()}


SCRATCH = {"consistency": consistency, "flow_color": color, "kitti": encoded, "flow_error": flow_error,
           "global_motion": global_motion, "egomotion": egomotion, "scene_flow": scene_flow}


@pytest.mark.parametrize("name", list(SCRATCH))
def test_host_scratch_equals_device_output(name, api):
    call = SCRATCH[name]
    mf = 2 * N
    ctx = context(api)
    full = np.empty((mf, H, W, 2), f32)
    ctx.get_flow_fullres(0, mf, full, W, H)
    ctx.sync()
    for n in (N - 1, mf):
        dev = call(ctx, n, "device")
        host = call(ctx, n, "host")
        again = np.empty_like(full)
        ctx.get_flow_fullres(0, mf, again, W, H)
        ctx.sync()
        assert bits(again) == bits(full), "%s: get_flow_fullres changed after n %d" % (name, n)
        assert bits(host) == bits(dev), "%s: host output differs from device output at n %d" % (name, n)
    ctx.close()
