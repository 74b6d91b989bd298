"""Camera tracking against the fused volume on the device (ofdis_fuse_track), measured: one JSON line.

    python tools/fuse_track_e2e.py [--frames 64] [--reps 3]

The clip, camera and 400 x 80 x 900 volume (28.8 M voxels, colour on) of tools/fusion_e2e.py, with the analytic
disparities and RGB frames in device memory and the true relative motions as the prediction:
  * per step (4 and 2, 10 rounds, integrating): the device-event time of one call over all frames into a fresh volume
    (median of `reps` calls after a warm-up call), per frame;
  * each kernel's time (torch.profiler, CUDA activities, in a pass of its own after the timed calls): the evaluation
    kernel per launch and the one-frame push per launch;
  * for comparison, one 64-frame push of tools/fusion_e2e.py's kind, per frame;
  * the statuses and rounds of the last call.
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
VOL = dict(nx=400, ny=80, nz=900, origin=(-10.0, -2.2, 2.0), voxel=0.05, trunc=0.15, max_weight=64.0, color=1)
TRACK = dict(step=4, rounds=10, min_weight=1.0, max_depth=45.0, huber=0.2, damping=1.0, min_corr=100,
             max_shift=0.5, min_cos=math.cos(math.radians(5.0)), eps=1e-7, integrate=1)


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("fuse_track_e2e: no CUDA device")
    n = a.frames
    fwd = np.concatenate([synth.axis_angle((0.0, math.radians(0.5), 0.0)), np.array([[0.0], [0.0], [-0.5]])], 1)
    back = np.concatenate([fwd[:, :3].T, -(fwd[:, :3].T @ fwd[:, 3:])], 1)
    rels = np.stack([fwd if k % 2 == 0 else back for k in range(n - 1)])
    clip = synth.rigid_stereo_clip(n - 1, H, W, 3, 5, CAM, list(rels), block={"velocity": (0.0, 0.0, 0.0)})
    stream = torch.cuda.Stream()
    prm = params.operating_point(2, W, noc=3, nop=1)
    scf = 1 << prm.sc_f
    ctx = api.Context(prm, (W + scf - 1) // scf * scf, (H + scf - 1) // scf * scf, prm.p_samp_s, n - 1,
                      stream=stream.cuda_stream)
    d_disp = torch.from_numpy(clip["disp"]).cuda()
    d_frames = torch.from_numpy(np.ascontiguousarray(clip["left"])).cuda()
    torch.cuda.synchronize()
    motions = np.concatenate([np.eye(3, 4)[None], rels])  # frame 0 keeps prev
    out = {}

    def track(step):
        ctx.fuse_begin(VOL)
        return ctx.fuse_track(d_disp.data_ptr(), motions, clip["abs"][0], CAM, dict(TRACK, step=step), width_org=W,
                              height_org=H, n=n, frames=d_frames.data_ptr(), memkind=api.MEM_DEVICE)

    def push():
        ctx.fuse_push(d_disp.data_ptr(), clip["abs"], CAM, width_org=W, height_org=H, frames=d_frames.data_ptr(),
                      memkind=api.MEM_DEVICE)

    from torch.profiler import ProfilerActivity, profile
    for step in (4, 2):
        poses, st = track(step)
        ms = median_ms(stream, lambda: track(step), a.reps)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            track(step)
            stream.synchronize()
        kernels = {}
        for ev in prof.key_averages():
            if "fuse_" in ev.key:
                name = "fuse_" + ev.key.split("fuse_", 1)[1].split("(")[0].split("<")[0]
                t = getattr(ev, "device_time_total", None)
                t = ev.cuda_time_total if t is None else t
                kernels[name] = {"ms_total": t / 1000.0, "launches": ev.count, "us_per_launch": t / max(ev.count, 1)}
        t_err, r_err = preprocess.trajectory_errors(poses, clip["abs"])
        out["step%d" % step] = {
            "call_ms_per_frame": ms / n, "kernels": kernels, "launches_per_call": n * (TRACK["rounds"] + 2),
            "cells": ((W - 1) // step + 1) * ((H - 1) // step + 1), "statuses": np.bincount(st["status"], minlength=3).tolist(),
            "mean_rounds": float(st["rounds"].mean()), "max_t_err_m": float(t_err.max()), "max_r_err_deg": float(r_err.max())}
    ctx.fuse_begin(VOL)
    push()
    push_ms = median_ms(stream, push, a.reps)
    ctx.close()
    print(json.dumps({"card": card(), "frames": n, "size": [W, H], "volume": [VOL["nx"], VOL["ny"], VOL["nz"]],
                      "push64_ms_per_frame": push_ms / n, **out}))


if __name__ == "__main__":
    main()
