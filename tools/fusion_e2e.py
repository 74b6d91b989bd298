"""Volumetric fusion on the device (ofdis_fuse_push / ofdis_fuse_extract / ofdis_fuse_render), measured: one JSON line.

    python tools/fusion_e2e.py [--frames 64] [--reps 10]

For a gray 1242x375 clip of synth.rigid_stereo_clip (KITTI's camera; the rig moves 0.5 m forward and turns 0.5 deg,
then back, frame by frame, so that it stays in the scene) with its analytic disparities and RGB frames in device
memory, and a 400 x 80 x 900 volume of 0.05 m voxels (28.8 M voxels, colour on) from (-10, -2.2, 2) in frame 0's
camera:
  * the device-event time of one push of all frames, one extract (count and write into a device buffer) and one
    render of every frame's pose (z 2 .. 45 m, step 0.05 m), median of `reps` calls after a warm-up call;
  * each kernel's time (torch.profiler, CUDA activities, in a pass of its own after the timed calls);
  * the push's volume traffic (2 x 11 bytes per voxel per call) over its kernel time, and its voxel-frame tests
    (voxels x frames, each a projection and, in the frustum, a disparity and colour gather) per second; the render's
    rays per second;
  * the points of the first push, counted twice: the count of a second extract must be the same.
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

from of_dis_b200 import api, params, synth

H, W = 375, 1242
CAM = dict(fx=721.5, fy=721.5, cx=609.6, cy=172.9, baseline=0.54, doffs=0.0)
VOL = dict(nx=400, ny=80, nz=900, origin=(-10.0, -2.2, 2.0), voxel=0.05, trunc=0.15, max_weight=64.0, color=1)


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
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("fusion_e2e: no CUDA device")
    n = a.frames
    fwd = np.concatenate([synth.axis_angle((0.0, math.radians(0.5), 0.0)), np.array([[0.0], [0.0], [-0.5]])], 1)
    back = np.concatenate([fwd[:, :3].T, -(fwd[:, :3].T @ fwd[:, 3:])], 1)
    clip = synth.rigid_stereo_clip(n - 1, H, W, 3, 5, CAM, [fwd if k % 2 == 0 else back for k in range(n - 1)],
                                   block={"velocity": (0.0, 0.0, 0.0)})
    stream = torch.cuda.Stream()
    prm = params.operating_point(2, W, noc=3, nop=1)
    scf = 1 << prm.sc_f
    ctx = api.Context(prm, (W + scf - 1) // scf * scf, (H + scf - 1) // scf * scf, prm.p_samp_s, n - 1,
                      stream=stream.cuda_stream)
    d_disp = torch.from_numpy(clip["disp"]).cuda()
    d_frames = torch.from_numpy(np.ascontiguousarray(clip["left"])).cuda()
    d_depth = torch.empty((n, H, W), device="cuda")
    ctx.fuse_begin(VOL)
    d_pts = torch.empty(28 * (8 << 20), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()

    def push():
        ctx.fuse_push(d_disp.data_ptr(), clip["abs"], CAM, width_org=W, height_org=H, frames=d_frames.data_ptr(),
                      memkind=api.MEM_DEVICE)

    def extract():
        return ctx.fuse_extract(1.0, capacity=8 << 20, memkind=api.MEM_DEVICE, out=d_pts.data_ptr())[1]

    def render():
        ctx.fuse_render(clip["abs"], CAM, z_near=2.0, z_far=45.0, step=0.05, width_org=W, height_org=H,
                        memkind=api.MEM_DEVICE, out=d_depth.data_ptr())

    push()
    total = extract()
    again = extract()
    render()
    res = {"push_ms": median_ms(stream, push, a.reps), "extract_ms": median_ms(stream, extract, a.reps),
           "render_ms": median_ms(stream, render, a.reps)}
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.reps):
            push()
            extract()
            render()
        stream.synchronize()
    kernels = {}
    for ev in prof.key_averages():
        if "fuse_" in ev.key:
            name = "fuse_" + ev.key.split("fuse_", 1)[1].split("(")[0].split("<")[0]
            t = getattr(ev, "device_time_total", None)
            t = ev.cuda_time_total if t is None else t
            kernels[name] = kernels.get(name, 0.0) + t / 1000.0 / a.reps
    N = VOL["nx"] * VOL["ny"] * VOL["nz"]
    integ = kernels.get("fuse_integrate_kernel", 0.0)
    rk = kernels.get("fuse_render_kernel", 0.0)
    depth = d_depth.cpu().numpy()
    res.update({
        "kernel_ms": kernels, "voxels": N, "points": int(total), "points_again_equal": again == total,
        "push_volume_GBps": 2 * 11 * N / (integ / 1e3) / 1e9 if integ else None,
        "push_voxel_frame_tests_per_s": float(N) * n / (integ / 1e3) if integ else None,
        "render_rays_per_s": float(n) * H * W / (rk / 1e3) if rk else None,
        "render_known_share": float(np.isfinite(depth).mean())})
    ctx.close()
    print(json.dumps({"card": card(), "frames": n, "size": [W, H], "volume": [VOL["nx"], VOL["ny"], VOL["nz"]],
                      "voxel_m": VOL["voxel"], **res}))


if __name__ == "__main__":
    main()
