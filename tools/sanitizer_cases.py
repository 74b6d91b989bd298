"""Small runs of every kernel family for compute-sanitizer (memcheck / racecheck / synccheck):
  compute-sanitizer --tool racecheck python tools/sanitizer_cases.py
the smoke configuration (P=8 gray flow) with both exact SOR kernels (sor_lane_kernel: flag-synchronised warps;
sor_wave_kernel: single CTA), a forward-backward case, a P=12 RGB and a P=12 stereo case (window-staged patch
kernel, stereo SOR), a 70-row level as three bands of the lane kernel and forced into a cluster of bands of the
wave kernel with 1 and 2 rows per thread (st.async halo exchange), and the 8-bit frame path (pyramid and
upsampling kernels), and a frame interpolation, a point tracking (advance, seed, block scan, scatter) and a filtered
disparity (union-find speckles, fill, depth and xyz) and a global motion (correspondences, compaction, hypotheses,
the bulk-copied score tiles with and without refills, refits, per-pixel outputs), a stereo ego-motion (the same
stages on 32-byte correspondences, non-finite disparities, score tile refills), a Fisher encoding (projection,
posteriors, float64 statistics, the take) and a TSDF fusion (integration, crossing count, scan and write, ray casting)
and its marching cubes (set_volume, the write with vertex bases, cube count, scan, faces) and a camera tracking
against it (the evaluation kernel's chunk sums, arrival counter and tree, with and without the push), the same
tracking and push weighted by per-pixel weights with special values, a per-pixel confidence (the halo-staged tile
and its window sums, planted level flows) and a monocular relative pose (full-pivot hypotheses, Sampson score tiles,
the refit CTA, per-pixel outputs, planted level flows) checked against their restatements.  Results are checked against the
oracle so that a clean log means a correct run."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from of_dis_b200 import api, params, preprocess, synth
from oracle import port_driver

CASES = [
    ("smoke_p8_gray", (128, 256), 1, 2, "3 1 12 12 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0", {"sor_lane": 1}),
    ("smoke_p8_gray_wave", (128, 256), 1, 2, "3 1 12 12 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0", {"sor_lane": 0}),
    ("lane_rows70_3bands", (140, 176), 1, 2, "2 1 6 6 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 2 1.6 0", {"sor_lane": 1}),
    ("fbcon_p8_gray", (64, 96), 1, 2, "3 1 8 8 0.05 0.95 0 8 0.4 1 1 0 1 10 10 5 1 3 1.6 0", {}),
    ("p12_rgb_l1", (96, 128), 3, 2, "3 1 8 8 0.05 0.95 0 12 0.75 0 1 1 1 10 10 5 1 3 1.6 0", {}),
    ("p12_stereo", (96, 128), 1, 1, "3 1 8 8 0.05 0.95 0 12 0.75 0 1 0 1 10 10 5 1 3 1.6 0", {}),
    ("cluster_rows70_rt1", (140, 176), 1, 2, "2 1 6 6 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 2 1.6 0",
     {"sor_lane": 0, "sor_single_max": 32, "sor_rows_per_thread": 1}),
    ("cluster_rows140_rt2", (140, 96), 1, 1, "1 0 6 6 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0",
     {"sor_lane": 0, "sor_single_max": 32, "sor_rows_per_thread": 2}),
]
if os.environ.get("SANITIZER_LANE") is not None:  # racecheck: force one SOR kernel everywhere (DESIGN.md section 5.4)
    CASES = [(n, sz, ch, nop, num, dict(o, sor_lane=int(os.environ["SANITIZER_LANE"]))) for n, sz, ch, nop, num, o in CASES]
for name, (h, w), ch, nop, numbers, opts in CASES:
    prm = params.from_cli_numbers(numbers.split(), noc=ch, nop=nop)
    i0, i1, _ = synth.synthetic_pair(h, w, ch, seed=5, stereo=(nop == 1), amp=3.0)
    pyr = preprocess.PairPyramids(i0, i1, prm.sc_f, prm.p_samp_s)
    ctx = api.Context(prm, pyr.width, pyr.height, pyr.imgpadding, 2)
    for k, v in opts.items():
        ctx.set_option(k, v)
    frames = np.ascontiguousarray(np.stack([np.stack([i0, i1])] * 2))
    if ch == 1:
        frames = frames[..., None]
    ctx.upload_frames_u8(0, 2, frames, w, h)
    ctx.run(2)
    got = ctx.get_flow(1, prm.sc_l)
    full = np.empty((2, h, w, nop), np.float32)
    ctx.get_flow_fullres(0, 2, full, w, h)
    ctx.sync()
    ctx.close()
    exp = port_driver.port_run(pyr, prm)
    ok = np.array_equal(got.view(np.uint32), exp.view(np.uint32))
    print("%-22s %s" % (name, "bitwise equal to the oracle" if ok else "MISMATCH"), flush=True)
    if not ok:
        sys.exit(1)
# frame interpolation (consistency masks, splat, resolve, fill rounds, blend) on a two-way clip, RGB flow
h, w, n = 61, 90, 2
prm = params.from_cli_numbers("3 1 8 8 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0".split(), noc=3, nop=2)
clip = synth.synthetic_sequence(n + 1, h, w, 3, seed=5, amp=3.0)
ctx = api.Context(prm, 96, 64, prm.p_samp_s, 2 * n)
ctx.upload_sequence_bidir_u8(0, n, clip, w, h)
ctx.run(2 * n)
full = np.empty((2 * n, h, w, 2), np.float32)
ctx.get_flow_fullres(0, 2 * n, full, w, h)
out, ut = ctx.interpolate_fullres(0, n, n, clip[:-1], clip[1:], 0.5, w, h, with_flow=True)
ctx.close()
exp, exp_ut = preprocess.interpolate_frames(clip[:-1], clip[1:], full[:n], full[n:], 0.5, 0.01, 0.5)
ok = np.array_equal(out, exp) and np.array_equal(ut.view(np.uint32), exp_ut.view(np.uint32))
print("%-22s %s" % ("interpolate_rgb", "bitwise equal to the restatement" if ok else "MISMATCH"), flush=True)
if not ok:
    sys.exit(1)
# point tracking through the same two-way clip, with a capacity that drops seeds (every tracker kernel, the
# single-CTA scan over several blocks of flags)
tp = dict(capacity=1000, spacing=2, alpha=0.01, beta=0.5, mb_alpha=0.01, mb_beta=0.002, min_eig=4.0)
ctx = api.Context(prm, 96, 64, prm.p_samp_s, 2 * n)
ctx.upload_sequence_bidir_u8(0, n, clip, w, h)
ctx.run(2 * n)
lists = [ctx.track_begin(tp, clip[0], w, h)] + ctx.track_advance(0, n, n, clip[1:], w, h)
st = ctx.track_stats()
ctx.close()
exp, est = preprocess.track_points(clip, full[:n], full[n:], tp)
ok = st == est and all(np.array_equal(g.view(np.uint8), e.view(np.uint8)) for g, e in zip(lists, exp))
print("%-22s %s" % ("track_rgb", "bitwise equal to the restatement" if ok else "MISMATCH"), flush=True)
if not ok:
    sys.exit(1)
# filtered disparities on a two-way stereo clip with a non-divisible size (classify, tile and border union-find,
# count, row and column fill, outputs), every stage on and every output asked for
prm = params.from_cli_numbers("3 1 8 8 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0".split(), noc=1, nop=1)
clip = synth.synthetic_sequence(n + 1, h, w, 1, seed=5, amp=3.0, stereo=True)
ctx = api.Context(prm, 96, 64, prm.p_samp_s, 2 * n)
ctx.upload_sequence_bidir_u8(0, n, clip, w, h)
ctx.run(2 * n)
full = np.empty((2 * n, h, w, 1), np.float32)
ctx.get_flow_fullres(0, 2 * n, full, w, h)
ctx.sync()
filt = dict(lr_check=1, alpha=0.0, beta=1.0, speckle_size=20, speckle_diff=0.05, fill=1)
cam = dict(fx=100.0, fy=100.0, cx=45.0, cy=30.0, baseline=0.5, doffs=0.0)
got = ctx.disparity_fullres(n, 2 * n, 0, w, h, camera=cam, outputs=("disp", "status", "depth", "xyz"), **filt)
ctx.close()
ok = True
for k in range(n):
    exp = preprocess.disparity_filter(full[n + k], full[k], True, camera=cam, **filt)
    ok &= all(np.array_equal(np.asarray(g[k]).view(np.uint8), np.asarray(e).view(np.uint8))
              for g, e in zip((got["disp"], got["status"], got["depth"], got["xyz"]), exp))
print("%-22s %s" % ("disparity_stereo", "bitwise equal to the restatement" if ok else "MISMATCH"), flush=True)
if not ok:
    sys.exit(1)
# global motion on a two-way RGB flow clip with fb_check and every per-pixel output; a step of 1 gives more
# correspondences than one 4096-entry score tile
prm = params.from_cli_numbers("3 1 8 8 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0".split(), noc=3, nop=2)
clip = synth.synthetic_sequence(n + 1, h, w, 3, seed=5, amp=3.0)
ctx = api.Context(prm, 96, 64, prm.p_samp_s, 2 * n)
ctx.upload_sequence_bidir_u8(0, n, clip, w, h)
ctx.run(2 * n)
full = np.empty((2 * n, h, w, 2), np.float32)
ctx.get_flow_fullres(0, 2 * n, full, w, h)
ctx.sync()
mp = dict(model="homography", step=1, fb_check=1, alpha=0.01, beta=0.5, hypotheses=100, threshold=1.0, refine=3, seed=3)
mask, res, reg = np.empty((n, h, w), np.uint8), np.empty((n, h, w, 2), np.float32), np.empty((n, h, w, 3), np.uint8)
models, stats = ctx.global_motion_fullres(0, n, mp, width_org=w, height_org=h, b0=n, i1=clip[1:], mask=mask,
                                          residual=res, registered=reg)
ctx.close()
exp = preprocess.global_motion(full[:n], full[n:], clip[1:], mp)
ok = all(np.array_equal(np.asarray(g).view(np.uint8), np.asarray(e).view(np.uint8))
         for g, e in zip((models, stats, mask, res, reg), exp))
print("%-22s %s" % ("global_motion_rgb", "bitwise equal to the restatement" if ok else "MISMATCH"), flush=True)
if not ok:
    sys.exit(1)
# and on 128 x 160 gray frames at step 1 without fb_check: more than 8192 correspondences per pair, so the score
# kernel refills both of its bulk-copied tile buffers
h2, w2 = 128, 160
prm = params.from_cli_numbers("3 1 8 8 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0".split(), noc=1, nop=2)
clip = synth.synthetic_sequence(n + 1, h2, w2, 1, seed=6, amp=3.0)
ctx = api.Context(prm, w2, h2, prm.p_samp_s, n)
ctx.upload_sequence_u8(0, n, clip, w2, h2)
ctx.run(n)
full = np.empty((n, h2, w2, 2), np.float32)
ctx.get_flow_fullres(0, n, full, w2, h2)
ctx.sync()
mp = dict(model="affine", step=1, fb_check=0, alpha=0.01, beta=0.5, hypotheses=70, threshold=1.0, refine=2, seed=4)
mask, res, reg = np.empty((n, h2, w2), np.uint8), np.empty((n, h2, w2, 2), np.float32), np.empty((n, h2, w2), np.uint8)
models, stats = ctx.global_motion_fullres(0, n, mp, width_org=w2, height_org=h2, i1=clip[1:], mask=mask, residual=res,
                                          registered=reg)
ctx.close()
exp = preprocess.global_motion(full, None, clip[1:], mp)
ok = (stats["n_corr"] > 8192).all() and all(np.array_equal(np.asarray(g).view(np.uint8), np.asarray(e).view(np.uint8))
                                            for g, e in zip((models, stats, mask, res, reg), exp))
print("%-22s %s" % ("global_motion_tiles", "bitwise equal to the restatement" if ok else "MISMATCH"), flush=True)
if not ok:
    sys.exit(1)
# stereo ego-motion on the same two gray pairs at step 1 (more than two 2048-entry score tiles per pair), disparities
# with NaN, +inf, -0 and negative entries, fb_check against the backward slots, every per-pixel output
rng = np.random.default_rng(8)
cam = dict(fx=200.0, fy=198.5, cx=79.75, cy=64.5, baseline=0.54, doffs=0.25)
maps = rng.uniform(5.0, 20.0, (n + 1, h2, w2)).astype(np.float32)
maps[rng.random(maps.shape) < 0.05] = np.nan
maps[rng.random(maps.shape) < 0.02] = np.inf
maps[rng.random(maps.shape) < 0.02] = -0.0
maps[rng.random(maps.shape) < 0.02] = -3.0
ctx = api.Context(prm, w2, h2, prm.p_samp_s, 2 * n)
ctx.upload_sequence_bidir_u8(0, n, clip, w2, h2)
ctx.run(2 * n)
full = np.empty((2 * n, h2, w2, 2), np.float32)
ctx.get_flow_fullres(0, 2 * n, full, w2, h2)
ctx.sync()
ep = dict(step=1, fb_check=1, alpha=0.01, beta=0.5, edge_diff=1.0, hypotheses=90, threshold=1.0, refine=3, seed=5)
pose, stats, outs = ctx.egomotion_fullres(0, n, maps[:-1], maps[1:], ep, camera=cam, width_org=w2, height_org=h2,
                                          b0=n, outputs=("mask", "residual", "object_motion"))
ctx.close()
exp = preprocess.egomotion(full[:n], full[n:], maps[:-1], maps[1:], cam, ep)
ok = (stats["n_corr"] > 2 * 2048).all() and all(
    np.array_equal(np.asarray(g).view(np.uint8), np.asarray(e).view(np.uint8))
    for g, e in zip((pose, stats, outs["mask"], outs["residual"], outs["object_motion"]), exp))
print("%-22s %s" % ("egomotion_tiles", "bitwise equal to the restatement" if ok else "MISMATCH"), flush=True)
if not ok:
    sys.exit(1)
# Fisher encoder (projection GEMM, posteriors, float64 statistics, the take): two chunks of descriptors with IDT's
# blocks, non-finite entries among them, K = 24 (a partial Gaussian tile) against preprocess.fisher_encode
rng = np.random.default_rng(7)
blocks = [(o, di, di // 2) for o, di in preprocess.fisher_blocks(preprocess.TRAJ_DEFAULTS)]
K, D = 24, preprocess.traj_dim(preprocess.TRAJ_DEFAULTS)
cb = {"K": K, "desc_dim": D, "blocks": blocks}
for part in preprocess.FISHER_PARTS:
    cb[part] = []
for _, di, d in blocks:
    cb["mean"].append(rng.uniform(0, 0.1, di).astype(np.float32))
    cb["proj"].append(rng.normal(0, di ** -0.5, (d, di)).astype(np.float32))
    cb["mu"].append(rng.normal(0, 0.2, (K, d)).astype(np.float32))
    cb["isig"].append(rng.uniform(1.0, 3.0, (K, d)).astype(np.float32))
    cb["c"].append(rng.normal(0, 1.0, K).astype(np.float32))
    cb["w"].append(np.full(K, 1.0 / K, np.float32))
x = np.abs(rng.normal(0, 0.3, (4096 + 77, D))).astype(np.float32)
x[5, 3], x[9, 100] = np.nan, np.inf
prm = params.from_cli_numbers("3 1 8 8 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0".split(), noc=1, nop=2)
ctx = api.Context(prm, 64, 64, prm.p_samp_s, 1)
ctx.fisher_begin(cb)
ctx.fisher_push(x)
got = ctx.fisher_take()
ctx.close()
exp = preprocess.fisher_encode(x, cb)
ok = all(np.array_equal(g.view(np.uint8), e.view(np.uint8)) for g, e in zip(got[:2], exp[:2])) and \
    np.array_equal(got[2]["n"], exp[2]["n"]) and np.array_equal(got[2]["skipped"], exp[2]["skipped"])
print("%-22s %s" % ("fisher_idt_k24", "bitwise equal to the restatement" if ok else "MISMATCH"), flush=True)
if not ok:
    sys.exit(1)
# volumetric fusion: a 29 x 17 x 33 volume straddling the frustum (beside and behind the cameras), disparities with
# NaN, -0, +inf and 3e9, RGB colour, then the volume, every point and a render checked bitwise
rng = np.random.default_rng(9)
cam = dict(fx=80.0, fy=77.0, cx=31.25, cy=23.5, baseline=0.5, doffs=0.25)
h3, w3 = 48, 64
maps = (np.float32(40.0) / rng.uniform(1.1, 1.6, (3, h3, w3)) - np.float32(0.25)).astype(np.float32)
for v, share in ((np.nan, 0.05), (-0.0, 0.03), (np.inf, 0.02), (3e9, 0.02)):
    maps[rng.random(maps.shape) < share] = v
poses = np.stack([np.concatenate([synth.axis_angle(rng.uniform(-0.1, 0.1, 3)),
                                  rng.uniform(-0.2, 0.2, (3, 1))], 1) for _ in range(3)])
rgb = rng.integers(0, 256, (3, h3, w3, 3)).astype(np.uint8)
fp = dict(nx=29, ny=17, nz=33, origin=(-1.5, -0.8, 0.2), voxel=0.07, trunc=0.2, max_weight=5.0, color=1)
prm = params.from_cli_numbers("3 1 8 8 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0".split(), noc=3, nop=2)
ctx = api.Context(prm, w3, h3, prm.p_samp_s, 2)
ctx.fuse_begin(fp)
ctx.fuse_push(maps, poses, cam, width_org=w3, height_org=h3, frames=rgb)
gv = ctx.fuse_volume()
gp, _ = ctx.fuse_extract(1.0)
gd = ctx.fuse_render(poses, cam, z_near=0.3, z_far=2.5, step=0.03, width_org=w3, height_org=h3)
ctx.close()
ev = preprocess.fuse_integrate(preprocess.fuse_new_volume(fp), fp, maps, poses, cam, frames=rgb)
ok = all(np.array_equal(gv[k].view(np.uint8), ev[k].view(np.uint8)) for k in ("T", "W", "C")) and \
    np.array_equal(gp.view(np.uint8), preprocess.fuse_extract(ev, fp, 1.0).view(np.uint8)) and \
    np.array_equal(gd.view(np.uint8), preprocess.fuse_render(ev, fp, poses, cam, 0.3, 2.5, 0.03, 1.0, w3, h3).view(np.uint8))
print("%-22s %s" % ("fuse", "bitwise equal to the restatement" if ok else "MISMATCH"), flush=True)
if not ok:
    sys.exit(1)
# marching cubes: a 23 x 29 x 41 volume (cubes straddling scan blocks) loaded with fuse_set_volume, T uniform with
# planted +0, -0, +-1, nextafter(1, 0) and NaN, W at, just below and above min_weight and NaN; host output at full
# capacity and device output at capacities one short of the totals
mp = dict(nx=23, ny=29, nz=41, origin=(-0.5, -0.5, 0.5), voxel=0.05, trunc=0.15, max_weight=8.0, color=1)
shape = (mp["nz"], mp["ny"], mp["nx"])
below1 = np.nextafter(np.float32(1), np.float32(0))
mv = preprocess.fuse_new_volume(mp)
mv["T"][:] = rng.uniform(-1.2, 1.2, shape).astype(np.float32)
mv["W"][:] = rng.choice(np.array([1.0, 2.0, 3.0], np.float32), shape)
for v, share in ((0.0, 0.05), (-0.0, 0.05), (1.0, 0.02), (-1.0, 0.02), (below1, 0.02), (np.nan, 0.01)):
    mv["T"][rng.random(shape) < share] = np.float32(v)
for v, share in ((0.0, 0.02), (below1, 0.02), (np.nan, 0.01)):
    mv["W"][rng.random(shape) < share] = np.float32(v)
mv["C"][:] = rng.integers(0, 256, shape + (3,))
ctx = api.Context(prm, w3, h3, prm.p_samp_s, 2)
ctx.fuse_begin(mp)
ctx.fuse_set_volume(mv["T"], mv["W"], mv["C"])
hp, hf, nv, nf = ctx.fuse_mesh(1.0)
dp = torch.zeros(28 * nv, dtype=torch.uint8, device="cuda")
df = torch.zeros(3 * nf, dtype=torch.int32, device="cuda")
ctx.fuse_mesh(1.0, pt_capacity=nv - 1, face_capacity=nf - 1, memkind=api.MEM_DEVICE, pts_out=dp.data_ptr(),
              faces_out=df.data_ptr())
ctx.close()
ep, ef = preprocess.fuse_mesh(mv, mp, 1.0)
ok = nf > 100 and np.array_equal(hp.view(np.uint8), ep.view(np.uint8)) and np.array_equal(hf, ef) and \
    np.array_equal(dp.cpu().numpy()[:28 * (nv - 1)], ep[:nv - 1].view(np.uint8)) and \
    np.array_equal(df.cpu().numpy()[:3 * (nf - 1)].view(np.uint32), ef[:nf - 1].ravel())
print("%-22s %s" % ("fuse_mesh", "bitwise equal to the restatement" if ok else "MISMATCH"), flush=True)
if not ok:
    sys.exit(1)
# camera tracking: a 29 x 17 x 33 volume loaded with fuse_set_volume (a tilted plane's TSDF with planted NaN, +-0 and
# +-1 T, W at, just below and above min_weight and NaN), disparities with NaN, -0, +inf and 3e9, three frames of 4
# rounds, without and with integration, the poses, stats and volume checked bitwise
tp_ = dict(nx=29, ny=17, nz=33, origin=(-1.0, -0.6, 0.4), voxel=0.05, trunc=0.15, max_weight=5.0, color=1)
tv = preprocess.fuse_new_volume(tp_)
zz = tp_["origin"][2] + np.arange(tp_["nz"])[:, None, None] * tp_["voxel"]
yy = tp_["origin"][1] + np.arange(tp_["ny"])[None, :, None] * tp_["voxel"]
tv["T"][:] = np.clip((1.2 + 0.1 * yy - zz) / tp_["trunc"], -1, 1).astype(np.float32)
tv["W"][:] = rng.choice(np.array([1.0, 2.0, 3.0], np.float32), tv["W"].shape)
for v, share in ((0.0, 0.02), (-0.0, 0.02), (1.0, 0.01), (-1.0, 0.01), (np.nan, 0.01)):
    tv["T"][rng.random(tv["T"].shape) < share] = np.float32(v)
for v, share in ((0.0, 0.02), (below1, 0.02), (np.nan, 0.01)):
    tv["W"][rng.random(tv["W"].shape) < share] = np.float32(v)
tv["C"][:] = rng.integers(0, 256, tv["C"].shape)
tmaps = (np.float32(40.0) / rng.uniform(1.15, 1.25, (3, h3, w3)) - np.float32(0.25)).astype(np.float32)
for v, share in ((np.nan, 0.05), (-0.0, 0.03), (np.inf, 0.02), (3e9, 0.02)):
    tmaps[rng.random(tmaps.shape) < share] = v
tmot = np.stack([np.concatenate([synth.axis_angle(rng.uniform(-0.005, 0.005, 3)),
                                 rng.uniform(-0.02, 0.02, (3, 1))], 1) for _ in range(3)])
tprev = np.concatenate([np.eye(3), [[0.01], [0.0], [0.02]]], 1)
ok = True
for integrate in (0, 1):
    trk = dict(step=1, rounds=4, min_weight=1.0, max_depth=float("inf"), huber=0.2, damping=0.1, min_corr=6,
               max_shift=0.5, min_cos=0.99, eps=0.0, integrate=integrate)
    ctx = api.Context(prm, w3, h3, prm.p_samp_s, 2)
    ctx.fuse_begin(tp_)
    ctx.fuse_set_volume(tv["T"], tv["W"], tv["C"])
    gpo, gst = ctx.fuse_track(tmaps, tmot, tprev, cam, trk, width_org=w3, height_org=h3, frames=rgb)
    gv = ctx.fuse_volume()
    ctx.close()
    ev = {k: v.copy() for k, v in tv.items()}
    epo, est = preprocess.fuse_track(ev, tp_, trk, tmaps, tmot, tprev, cam, rgb)
    ok = ok and np.array_equal(gpo.view(np.uint64), epo.view(np.uint64)) and \
        all(np.array_equal(gst[k], est[k]) for k in est.dtype.names) and (est["rounds"] > 0).any() and \
        all(np.array_equal(*(np.where(np.isnan(a), np.float32(np.nan), a).view(np.uint8) if a.dtype == np.float32
                             else a for a in (gv[k], ev[k]))) for k in ("T", "W", "C"))
print("%-22s %s" % ("fuse_track", "bitwise equal to the restatement" if ok else "MISMATCH"), flush=True)
if not ok:
    sys.exit(1)
# confidence-weighted push and tracking on the same volume: weights with 0, -0, NaN, +-inf, negative values, 3e9 and
# 1e-30, the tracking with integration; poses, stats and volume checked bitwise
wts = rng.uniform(0.05, 2.0, tmaps.shape).astype(np.float32)
for v, share in ((0.0, 0.03), (-0.0, 0.03), (np.nan, 0.03), (np.inf, 0.02), (-np.inf, 0.02), (-1.0, 0.03),
                 (3e9, 0.02), (1e-30, 0.02)):
    wts[rng.random(wts.shape) < share] = v
trk = dict(step=1, rounds=4, min_weight=1.0, max_depth=float("inf"), huber=0.2, damping=0.1, min_corr=6,
           max_shift=0.5, min_cos=0.99, eps=0.0, integrate=1)
ctx = api.Context(prm, w3, h3, prm.p_samp_s, 2)
ctx.fuse_begin(tp_)
ctx.fuse_set_volume(tv["T"], tv["W"], tv["C"])
gpo, gst = ctx.fuse_track(tmaps, tmot, tprev, cam, trk, width_org=w3, height_org=h3, frames=rgb, weights=wts)
ctx.fuse_push(tmaps, gpo, cam, width_org=w3, height_org=h3, frames=rgb, weights=wts)
gv = ctx.fuse_volume()
ctx.close()
ev = {k: v.copy() for k, v in tv.items()}
epo, est = preprocess.fuse_track(ev, tp_, trk, tmaps, tmot, tprev, cam, rgb, weights=wts)
preprocess.fuse_integrate(ev, tp_, tmaps, epo, cam, frames=rgb, weights=wts)
ok = np.array_equal(gpo.view(np.uint64), epo.view(np.uint64)) and \
    all(np.array_equal(gst[k], est[k]) for k in est.dtype.names) and (est["rounds"] > 0).any() and \
    all(np.array_equal(*(np.where(np.isnan(a), np.float32(np.nan), a).view(np.uint8) if a.dtype == np.float32
                         else a for a in (gv[k], ev[k]))) for k in ("T", "W", "C"))
print("%-22s %s" % ("fuse_weighted", "bitwise equal to the restatement" if ok else "MISMATCH"), flush=True)
if not ok:
    sys.exit(1)
# per-pixel confidence: a two-way RGB flow clip of partial tiles, one forward and one backward level flow planted
# with NaN, +-inf, -0 and 3e9, r = 1 and 7, with and without partners, host and device outputs
cprm = params.from_cli_numbers("3 1 8 8 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0".split(), noc=3, nop=2)
ch_, cw_, cn = 45, 77, 2
cframes = synth.synthetic_sequence(cn + 1, ch_, cw_, 3, seed=9, amp=3.0)
scf = 1 << cprm.sc_f
ctx = api.Context(cprm, (cw_ + scf - 1) // scf * scf, (ch_ + scf - 1) // scf * scf, cprm.p_samp_s, 2 * cn)
ctx.upload_sequence_bidir_u8(0, cn, cframes, cw_, ch_)
ctx.run(2 * cn)
for slot in (0, cn + 1):
    lv = ctx.get_flow(slot, cprm.sc_l)
    for v, share in ((np.nan, 0.05), (np.inf, 0.03), (-np.inf, 0.03), (-0.0, 0.05), (3e9, 0.03)):
        lv[rng.random(lv.shape) < share] = np.float32(v)
    ctx.set_flow(slot, cprm.sc_l, lv)
F = np.empty((2 * cn, ch_, cw_, 2), np.float32)
ctx.get_flow_fullres(0, 2 * cn, F, cw_, ch_)
ctx.sync()
d_frames = torch.from_numpy(cframes).cuda()
d_conf = torch.zeros((cn, ch_, cw_), device="cuda")
d_terms = torch.zeros((cn, ch_, cw_, 3), device="cuda")
torch.cuda.synchronize()
canon = lambda a: np.where(np.isnan(a), np.float32(np.nan), a).view(np.uint32)  # NaN of arithmetic: any payload
ok = True
for r in (1, 7):
    cp = dict(radius=r, s_fb=1.0, s_tex=100.0, min_count=(2 * r + 1) ** 2 // 2)
    for b0 in (cn, -1):
        hc, ht = ctx.confidence_fullres(0, cn, b0, cframes[:-1], cframes[1:], cp, cw_, ch_, with_terms=True)
        ctx.confidence_fullres(0, cn, b0, d_frames.data_ptr(), d_frames.data_ptr() + ch_ * cw_ * 3, cp, cw_, ch_,
                               with_terms=True, memkind=api.MEM_DEVICE, conf=d_conf.data_ptr(),
                               terms=d_terms.data_ptr(), frame_stride=ch_ * cw_ * 3)
        ctx.sync()
        for k in range(cn):
            ec, et = preprocess.confidence(cframes[k], cframes[k + 1], F[k], None if b0 < 0 else F[cn + k], cp)
            ok = ok and np.array_equal(hc[k].view(np.uint32), ec.view(np.uint32)) and \
                np.array_equal(canon(ht[k]), canon(et)) and \
                np.array_equal(d_conf[k].cpu().numpy().view(np.uint32), ec.view(np.uint32)) and \
                np.array_equal(canon(d_terms[k].cpu().numpy()), canon(et))
ctx.close()
print("%-22s %s" % ("confidence", "bitwise equal to the restatement" if ok else "MISMATCH"), flush=True)
if not ok:
    sys.exit(1)
# monocular relative pose: a rigid clip's exact flow with NaN, +-inf and 3e9 planted as level flows, an all-invalid
# pair, step 1 (more than two 4096-entry score tiles), every per-pixel output in device memory
h3, w3 = 96, 160
rcam = dict(fx=180.0, fy=176.5, cx=79.75, cy=48.5, baseline=0.54, doffs=0.0)
rmo = np.concatenate([synth.axis_angle((0.0, 0.01, 0.0)), np.array([[0.03], [0.0], [-0.5]])], 1)
rclip = synth.rigid_stereo_clip(1, h3, w3, 1, 4, rcam, [rmo])
a = rclip["flow"][0].astype(np.float32).copy()
a[::3, ::5] = np.nan
a[1::7, ::2, 0] = np.inf
a[2::5, 1::3, 1] = -np.inf
a[3::4, 3::4, 0] = 3e9
rflows = np.stack([a, np.full((h3, w3, 2), np.nan, np.float32)])
rprm = params.from_cli_numbers("3 0 8 8 0.05 0.95 0 8 0.4 0 1 0 0 10 10 5 1 3 1.6 0".split(), noc=1, nop=2)
ctx = api.Context(rprm, w3, h3, rprm.p_samp_s, 2)
for k in range(2):
    ctx.set_flow(k, 0, rflows[k])
rp = dict(fx=180.0, fy=176.5, cx=79.75, cy=48.5, step=1, fb_check=0, alpha=0.01, beta=0.5, hypotheses=96,
          threshold=1.0, refine=3, min_parallax=0.25, seed=7)
dev = {"mask": torch.empty((2, h3, w3), dtype=torch.uint8, device="cuda"),
       "sampson": torch.empty((2, h3, w3), device="cuda"), "depth": torch.empty((2, h3, w3), device="cuda")}
torch.cuda.synchronize()
pose, stats, _ = ctx.relpose_fullres(0, 2, rp, width_org=w3, height_org=h3, outputs=tuple(dev),
                                     out={k: v.data_ptr() for k, v in dev.items()}, memkind=api.MEM_DEVICE)
ctx.close()
exp = preprocess.relpose(rflows, None, rp)
ok = stats["n_corr"][0] > 2 * 4096 and stats["status"].tolist()[1] == 1 and all(
    np.array_equal(np.asarray(g).view(np.uint8), np.asarray(e).view(np.uint8))
    for g, e in zip((pose, stats, dev["mask"].cpu().numpy(), dev["sampson"].cpu().numpy(), dev["depth"].cpu().numpy()),
                    exp))
print("%-22s %s" % ("relpose", "bitwise equal to the restatement" if ok else "MISMATCH"), flush=True)
if not ok:
    sys.exit(1)
print("all cases ok")
