"""Marching cubes on the device (ofdis_fuse_mesh), measured: one JSON line.

    python tools/mesh_e2e.py [--frames 64] [--reps 10]

The 28.8 M-voxel volume of tools/fusion_e2e.py (400 x 80 x 900 voxels of 0.05 m, colour on, the same clip of
synth.rigid_stereo_clip pushed once), then:
  * the device-event time of one mesh call with device output and with host output (counts first, then everything
    through the full-resolution scratch), and of one extraction into a device buffer for comparison, median of `reps`
    calls after a warm-up call;
  * each kernel's time (torch.profiler, CUDA activities, in a pass of its own after the timed calls);
  * the algorithmic volume traffic of the mesh call -- the volume's T and W read once each by the vertex count, the
    vertex write, the cube count and the face write, 4 x 8 bytes per voxel -- over the sum of its kernel times;
  * the vertices and faces, and whether a second call gives the same counts and bytes.
The card's name and power limit are read in the same run."""
import argparse
import json
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
import torch

from fusion_e2e import CAM, H, VOL, W, card, median_ms
from of_dis_b200 import api, params, synth

MESH_KERNELS = ("fuse_count_kernel", "fuse_scan_kernel", "fuse_write_kernel", "fuse_cube_count_kernel",
                "fuse_face_kernel")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("mesh_e2e: no CUDA device")
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
    ctx.fuse_begin(VOL)
    torch.cuda.synchronize()
    ctx.fuse_push(d_disp.data_ptr(), clip["abs"], CAM, width_org=W, height_org=H, frames=d_frames.data_ptr(),
                  memkind=api.MEM_DEVICE)
    _, _, nv, nf = ctx.fuse_mesh(1.0, pt_capacity=0, face_capacity=0)
    d_pts = torch.empty(28 * nv, dtype=torch.uint8, device="cuda")
    d_faces = torch.empty(3 * nf, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()

    def mesh_device():
        return ctx.fuse_mesh(1.0, pt_capacity=nv, face_capacity=nf, memkind=api.MEM_DEVICE, pts_out=d_pts.data_ptr(),
                             faces_out=d_faces.data_ptr())

    def mesh_host():
        return ctx.fuse_mesh(1.0)

    def extract():
        return ctx.fuse_extract(1.0, capacity=nv, memkind=api.MEM_DEVICE, out=d_pts.data_ptr())

    mesh_device()
    first = (d_pts.cpu().numpy().copy(), d_faces.cpu().numpy().copy())
    hp, hf, nv2, nf2 = mesh_host()
    again = (nv2, nf2) == (nv, nf) and np.array_equal(first[0], hp.view(np.uint8).ravel()) and \
        np.array_equal(first[1].view(np.uint32), hf.ravel())
    extract()
    res = {"mesh_device_ms": median_ms(stream, mesh_device, a.reps),
           "mesh_host_ms": median_ms(stream, mesh_host, a.reps), "extract_ms": median_ms(stream, extract, a.reps)}
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.reps):
            mesh_device()
        stream.synchronize()
    kernels = {}
    for ev in prof.key_averages():
        if "fuse_" in ev.key:
            name = "fuse_" + ev.key.split("fuse_", 1)[1].split("(")[0].split("<")[0]
            t = getattr(ev, "device_time_total", None)
            t = ev.cuda_time_total if t is None else t
            kernels[name] = kernels.get(name, 0.0) + t / 1000.0 / a.reps
    N = VOL["nx"] * VOL["ny"] * VOL["nz"]
    ksum = sum(kernels.get(k, 0.0) for k in MESH_KERNELS)
    res.update({"kernel_ms": kernels, "mesh_kernels_ms": ksum, "voxels": N, "vertices": int(nv), "faces": int(nf),
                "second_call_equal": bool(again),
                "mesh_volume_GBps": 4 * 8 * N / (ksum / 1e3) / 1e9 if ksum else None})
    ctx.close()
    print(json.dumps({"card": card(), "frames": n, "size": [W, H], "volume": [VOL["nx"], VOL["ny"], VOL["nz"]],
                      "voxel_m": VOL["voxel"], **res}))


if __name__ == "__main__":
    main()
