"""Monocular relative pose on the device (ofdis_relpose_fullres), measured: one JSON line.

    python tools/relpose_e2e.py [--pairs 64] [--reps 20]

For a gray 1242x375 clip of synth.rigid_stereo_clip (KITTI's camera; the rig moves 0.9 m forward and turns 0.5 deg,
then back, pair by pair; a box moves 2 cm sideways per frame on its own) at operating point 2, 64 pairs with the
two-way upload (128 slots), fb_check against the backward slots, step 8, 1024 hypotheses, 5 refits, device outputs
(mask, Sampson distance, depth):
  * the device-event time of one relpose call over the 64 pairs, median of `reps` calls after two warm-up calls, next
    to ofdis_egomotion_fullres on the same flows (the clip's disparities, the same step, hypotheses and refits) and
    ofdis_run of the 128 slots;
  * the split of the relpose call over correspondences, hypotheses, scoring, refit and apply (torch.profiler, CUDA
    activities, in a pass of its own after the timed calls; the sum over the `reps` calls divided by `reps`);
  * a bitwise check of the first pair against preprocess.relpose.
The card's name and power limit are read in the same run."""
import argparse
import json
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from of_dis_b200 import api, params, preprocess, synth

H, W = 375, 1242
CAM = dict(fx=721.5, fy=721.5, cx=609.6, cy=172.9, baseline=0.54, doffs=0.0)
STAGES = (("corr", "motion_corr_kernel"), ("compact", "motion_compact_kernel"), ("hyp", "relpose_hyp_kernel"),
          ("score", "motion_score_kernel"), ("refit", "relpose_refit_kernel"), ("apply", "relpose_apply_kernel"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def median_ms(stream, fn, reps):
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        fn()
        b.record(stream)
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def measure(n, reps):
    stream = torch.cuda.Stream()
    prm = params.operating_point(2, W, noc=1)
    fwd = np.concatenate([synth.axis_angle((0.0, math.radians(0.5), 0.0)), np.array([[0.0], [0.0], [-0.9]])], 1)
    back = np.concatenate([fwd[:, :3].T, -(fwd[:, :3].T @ fwd[:, 3:])], 1)  # the inverse: the rig stays in the scene
    clip = synth.rigid_stereo_clip(n, H, W, 1, 5, CAM, [fwd if k % 2 == 0 else back for k in range(n)],
                                   block={"velocity": (0.02, 0.0, 0.0)})
    scf = 1 << prm.sc_f
    ctx = api.Context(prm, (W + scf - 1) // scf * scf, (H + scf - 1) // scf * scf, prm.p_samp_s, 2 * n,
                      stream=stream.cuda_stream)
    ctx.upload_sequence_bidir_u8(0, n, clip["left"], W, H)
    ctx.run(2 * n)
    res = {"ofdis_run_ms": median_ms(stream, lambda: ctx.run(2 * n), reps)}
    pix = H * W
    dev = {"mask": torch.empty((n, H, W), dtype=torch.uint8, device="cuda"),
           "sampson": torch.empty((n, H, W), device="cuda"), "depth": torch.empty((n, H, W), device="cuda")}
    ptrs = {k: v.data_ptr() for k, v in dev.items()}
    p = dict(fx=CAM["fx"], fy=CAM["fy"], cx=CAM["cx"], cy=CAM["cy"], step=8, fb_check=1, alpha=0.01, beta=0.5,
             hypotheses=1024, threshold=1.0, refine=5, min_parallax=0.5, seed=0)

    def call(f1=n):
        return ctx.relpose_fullres(0, f1, p, width_org=W, height_org=H, b0=n, outputs=tuple(ptrs), out=ptrs,
                                   memkind=api.MEM_DEVICE)
    d_disp = torch.from_numpy(clip["disp"]).cuda()
    eo = {"mask": torch.empty((n, H, W), dtype=torch.uint8, device="cuda")}
    ep = dict(step=8, fb_check=1, alpha=0.01, beta=0.5, edge_diff=1.0, hypotheses=1024, threshold=1.0, refine=5,
              seed=0)

    def ego():
        return ctx.egomotion_fullres(0, n, d_disp.data_ptr(), d_disp.data_ptr() + 4 * pix, ep, camera=CAM,
                                     width_org=W, height_org=H, b0=n, disp_stride=pix, outputs=("mask",),
                                     out={"mask": eo["mask"].data_ptr()}, memkind=api.MEM_DEVICE)
    torch.cuda.synchronize()
    for _ in range(2):
        pose, stats, _ = call()
        ego()
    res["relpose_ms"] = median_ms(stream, call, reps)
    res["egomotion_ms"] = median_ms(stream, ego, reps)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            call()
        stream.synchronize()
    split = {}
    for ev in prof.key_averages():
        for stage, name in STAGES:
            if name in ev.key:
                t = getattr(ev, "device_time_total", None)
                t = ev.cuda_time_total if t is None else t
                split[stage] = split.get(stage, 0.0) + t / 1000.0 / reps
    res["relpose_kernel_ms"] = split
    r_err, t_err = preprocess.relpose_errors(pose, clip["poses"])
    res["status"] = sorted(set(stats["status"].tolist()))
    res["r_err_deg_max"], res["t_dir_err_deg_max"] = float(np.nanmax(r_err)), float(np.nanmax(t_err))
    full = np.empty((2 * n, H, W, 2), np.float32)
    ctx.get_flow_fullres(0, 2 * n, full, W, H)
    ctx.sync()
    exp = preprocess.relpose(full[:1], full[n:n + 1], p)
    pose, stats, _ = call(1)
    got = (pose, stats) + tuple(dev[k][:1].cpu().numpy() for k in ("mask", "sampson", "depth"))
    res["bitwise_equal_to_restatement"] = bool(all(
        np.asarray(g).tobytes() == np.asarray(e).tobytes() for g, e in zip(got, exp)))
    ctx.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=64)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("relpose_e2e: no CUDA device")
    out = {"card": card(), "pairs": a.pairs, "size": [W, H], "op": 2, "gray": measure(a.pairs, a.reps)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
