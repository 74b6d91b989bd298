"""Dense point tracking on the device (ofdis_track_begin / ofdis_track_advance), measured: one JSON line.

    python tools/track_e2e.py [--pairs 64] [--reps 20]

For gray and RGB 1024x436 clips at operating point 2 (64 pairs as a 65-frame clip with the two-way upload, the
backward partners in the same launch), with the batch command's settings (spacing 8, capacity 4 x cells, alpha 0.01,
beta 0.5, mb_alpha 0.01, mb_beta 0.002, min_eig 25):
  * the device-event time of ofdis_track_begin + ofdis_track_advance through all pairs, frames and records in device
    memory, median of `reps` calls after two warm-up calls, next to the same batch's ofdis_run time;
  * the counters (seeded, alive, ended per reason, dropped) and how many of frame 0's cells min_eig rejected;
  * a bitwise check of the first pairs against preprocess.track_points;
  * for the tracks seeded in frame 0, the distance to their analytic position in synth's clip: frame t is the canvas
    at x - t flow(x), so the point p of frame 0 is at the solution of x = p + t flow(x) (fixed-point iteration).  The
    median over every frame, and at the last frame, with the count of frame-0 tracks still alive there.
The card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from of_dis_b200 import api, params, preprocess, synth

H, W = 436, 1024
AMP = 3.0
CHECK_PAIRS = 4


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


def analytic(px, py, t):
    """x with x - t flow(x) = (px, py): synth's flow as a function of continuous positions."""
    x, y = px.astype(np.float64), py.astype(np.float64)
    for _ in range(50):
        u = AMP * np.sin(4.0 * x / W + 0.3) * np.cos(3.0 * y / H)
        v = 0.6 * AMP * np.cos(2.5 * x / W) * np.sin(5.0 * y / H + 0.7)
        x, y = px + t * u, py + t * v
    return x, y


def measure(ch, n, reps):
    stream = torch.cuda.Stream()
    prm = params.operating_point(2, W, noc=ch)
    clip = synth.synthetic_sequence(n + 1, H, W, ch, seed=5, amp=AMP)
    scf = 1 << prm.sc_f
    ctx = api.Context(prm, (W + scf - 1) // scf * scf, (H + scf - 1) // scf * scf, prm.p_samp_s, 2 * n,
                      stream=stream.cuda_stream)
    ctx.upload_sequence_bidir_u8(0, n, clip, W, H)
    ctx.run(2 * n)
    cells = ((W + 7) // 8) * ((H + 7) // 8)
    p = dict(capacity=4 * cells, spacing=8, alpha=0.01, beta=0.5, mb_alpha=0.01, mb_beta=0.002, min_eig=25.0)
    hwc = H * W * ch
    dev = torch.from_numpy(clip.reshape(-1)).cuda()
    pts = torch.empty((n * p["capacity"] * 3,), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()

    def call():
        ctx.track_begin(p, dev.data_ptr(), W, H, memkind=api.MEM_DEVICE, points=pts.data_ptr())
        ctx.track_advance(0, n, n, dev.data_ptr() + hwc, W, H, memkind=api.MEM_DEVICE, points=pts.data_ptr())

    before = ctx.launch_count
    call()
    launches = ctx.launch_count - before
    call()
    t_track = median_ms(stream, call, reps)
    t_run = median_ms(stream, lambda: ctx.run(2 * n), reps)
    # host lists of the whole clip (the run above recomputed the same flows) and the counters
    lists = [ctx.track_begin(p, clip[0], W, H)] + ctx.track_advance(0, n, n, clip[1:], W, H)
    st = ctx.track_stats()
    flows = np.empty((2 * n, H, W, 2), np.float32)
    ctx.get_flow_fullres(0, 2 * n, flows, W, H)
    ctx.sync()
    ctx.close()
    exp, _ = preprocess.track_points(clip[:CHECK_PAIRS + 1], flows[:CHECK_PAIRS], flows[n:n + CHECK_PAIRS], p)
    bitwise = all(np.array_equal(g.view(np.uint8), e.view(np.uint8)) for g, e in zip(lists, exp))
    # accuracy of the tracks from frame 0
    first = lists[0]
    start = {int(i): (x, y) for i, x, y in zip(first["id"], first["x"], first["y"])}
    dist, last = [], None
    for t in range(1, n + 1):
        l = lists[t]
        l = l[l["id"] < len(first)]
        sx = np.array([start[int(i)][0] for i in l["id"]], np.float64)
        sy = np.array([start[int(i)][1] for i in l["id"]], np.float64)
        ax, ay = analytic(sx, sy, t)
        d = np.hypot(l["x"] - ax, l["y"] - ay)
        dist.append(d)
        last = d
    return {"track_ms": round(t_track, 4), "run_ms": round(t_run, 4), "launches_per_call": launches,
            "cells": cells, "frame0_seeded": int(len(first)), "frame0_rejected_min_eig": int(cells - len(first)),
            "stats": st, "bitwise_first_pairs": bool(bitwise),
            "frame0_tracks_alive_at_end": int(len(last)),
            "median_dist_px_all_frames": round(float(np.median(np.concatenate(dist))), 4),
            "median_dist_px_last_frame": round(float(np.median(last)), 4) if len(last) else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=64)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("track_e2e: no CUDA device")
    res = {"card": card(), "size": "%dx%d" % (W, H), "pairs": a.pairs, "oppoint": 2, "memory": "device"}
    for ch, tag in ((1, "gray"), (3, "rgb")):
        res[tag] = measure(ch, a.pairs, a.reps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
