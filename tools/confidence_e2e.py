"""Per-pixel confidence on the device (ofdis_confidence_fullres) and the weighted fusion and tracking, measured: one
JSON line.

    python tools/confidence_e2e.py [--reps 20]

  * confidence: 64 gray pairs of 1024 x 436 at operating point 2, a two-way upload (forward slots against their backward
    partners), device frames and outputs; the device-event median of one call for r = 2 and r = 7, with ofdis_run's
    time for the same 64 pairs (forward slots only) beside it;
  * fusion: on tools/fuse_track_e2e.py's clip and 28.8 M-voxel volume, a 16-frame push and a 16-frame tracking call
    (step 4, 10 rounds, integrating), unweighted and weighted by all-ones maps, alternated; device-event medians.
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


def context(prm, w, h, n, stream):
    scf = 1 << prm.sc_f
    return api.Context(prm, (w + scf - 1) // scf * scf, (h + scf - 1) // scf * scf, prm.p_samp_s, n,
                       stream=stream.cuda_stream)


def confidence(reps, stream):
    n, w, h = 64, 1024, 436
    prm = params.operating_point(2, w, noc=1, nop=2)
    frames = synth.synthetic_sequence(n + 1, h, w, 1, seed=3, amp=4.0)
    ctx = context(prm, w, h, 2 * n, stream)
    ctx.upload_sequence_bidir_u8(0, n, frames, w, h)
    ctx.run(2 * n)
    d_frames = torch.from_numpy(frames).cuda()
    d_conf = torch.empty((n, h, w), device="cuda")
    torch.cuda.synchronize()
    out = {"pairs": n, "size": [w, h]}
    for r in (2, 7):
        p = dict(radius=r, s_fb=1.0, s_tex=100.0, min_count=(2 * r + 1) ** 2 // 2)

        def call():
            ctx.confidence_fullres(0, n, n, d_frames.data_ptr(), d_frames.data_ptr() + w * h, p, w, h,
                                   memkind=api.MEM_DEVICE, conf=d_conf.data_ptr(), frame_stride=w * h)

        call()
        out["r%d_ms" % r] = median_ms(stream, call, reps)
    ctx.close()
    ctx = context(prm, w, h, n, stream)
    ctx.upload_sequence_u8(0, n, frames, w, h)
    ctx.run(n)
    out["run_ms"] = median_ms(stream, lambda: ctx.run(n), reps)
    ctx.close()
    return out


def fusion(reps, stream):
    H, W, n = 375, 1242, 16
    cam = dict(fx=721.5, fy=721.5, cx=609.6, cy=172.9, baseline=0.54, doffs=0.0)
    vol = dict(nx=400, ny=80, nz=900, origin=(-10.0, -2.2, 2.0), voxel=0.05, trunc=0.15, max_weight=64.0, color=1)
    tp = dict(step=4, rounds=10, min_weight=1.0, max_depth=45.0, huber=0.2, damping=1.0, min_corr=100,
              max_shift=0.5, min_cos=math.cos(math.radians(5.0)), eps=1e-7, integrate=1)
    fwd = np.concatenate([synth.axis_angle((0.0, math.radians(0.5), 0.0)), np.array([[0.0], [0.0], [-0.5]])], 1)
    back = np.concatenate([fwd[:, :3].T, -(fwd[:, :3].T @ fwd[:, 3:])], 1)
    rels = np.stack([fwd if k % 2 == 0 else back for k in range(n - 1)])
    clip = synth.rigid_stereo_clip(n - 1, H, W, 3, 5, cam, list(rels), block={"velocity": (0.0, 0.0, 0.0)})
    ctx = context(params.operating_point(2, W, noc=3, nop=1), W, H, n, stream)
    d_disp = torch.from_numpy(clip["disp"]).cuda()
    d_frames = torch.from_numpy(np.ascontiguousarray(clip["left"])).cuda()
    d_ones = torch.ones((n, H, W), device="cuda")
    torch.cuda.synchronize()
    motions = np.concatenate([np.eye(3, 4)[None], rels])
    ctx.fuse_begin(vol)

    def push(wts):
        ctx.fuse_push(d_disp.data_ptr(), clip["abs"], cam, width_org=W, height_org=H, frames=d_frames.data_ptr(),
                      memkind=api.MEM_DEVICE, weights=wts)

    def track(wts):
        ctx.fuse_begin(vol)
        ctx.fuse_track(d_disp.data_ptr(), motions, clip["abs"][0], cam, tp, width_org=W, height_org=H, n=n,
                       frames=d_frames.data_ptr(), memkind=api.MEM_DEVICE, weights=wts)

    times = {"push": [], "push_weighted": [], "track": [], "track_weighted": []}
    push(None), push(d_ones.data_ptr()), track(None), track(d_ones.data_ptr())
    for _ in range(3):  # alternated, so that both see the same state of the card
        times["push"].append(median_ms(stream, lambda: push(None), reps))
        times["push_weighted"].append(median_ms(stream, lambda: push(d_ones.data_ptr()), reps))
        times["track"].append(median_ms(stream, lambda: track(None), max(3, reps // 4)))
        times["track_weighted"].append(median_ms(stream, lambda: track(d_ones.data_ptr()), max(3, reps // 4)))
    ctx.close()
    return {"frames": n, "volume": [vol["nx"], vol["ny"], vol["nz"]],
            **{k + "_ms": float(np.median(v)) for k, v in times.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("confidence_e2e: no CUDA device")
    stream = torch.cuda.Stream()
    print(json.dumps({"card": card(), "confidence": confidence(a.reps, stream), "fusion": fusion(a.reps, stream)}))


if __name__ == "__main__":
    main()
