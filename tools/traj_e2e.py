"""Trajectory descriptors on the device (ofdis_traj_begin / ofdis_traj_advance), measured: one JSON line.

    python tools/traj_e2e.py [--pairs 64] [--reps 20]

Workloads at operating point 2, 64 pairs with the two-way upload, frames and outputs in device memory, the batch
command's tracker settings (spacing 8, capacity 4 x cells) and the IDT defaults: a 1024x436 gray
synth.global_motion_clip (a camera similarity and a rectangle that moves on its own) with its true camera models, and
a 1920x1080 RGB synth.synthetic_sequence (amplitude 3) without models (the clip generator's cubic resampling of 65
full-HD frames would take minutes):
  * the device-event times of ofdis_traj_begin + ofdis_traj_advance through all pairs, of ofdis_track_begin +
    ofdis_track_advance on the same slots and of the batch's ofdis_run, medians of `reps` calls after warm-up;
  * the launches per call, and the segments emitted and rejected per reason;
  * the per-kernel device times of one traj call from torch.profiler (in a separate, profiled call), with the
    histogram kernel's field bytes (N^2 pixels x 36 bytes per live track and pair) over its time.
The card's name and power limit are read in the same run."""
import argparse
import json
import os
import re
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from of_dis_b200 import api, params, preprocess, synth


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


def measure(h, w, ch, n, reps, camera):
    stream = torch.cuda.Stream()
    prm = params.operating_point(2, w, noc=ch)
    if camera:
        H = synth.similarity_about_centre(h, w, 0.2, 1.002, (1.5, 0.5))
        clip, models, _ = synth.global_motion_clip(n, h, w, ch, seed=5, H=H)
        M = models.reshape(n, 9)
    else:
        clip, M = synth.synthetic_sequence(n + 1, h, w, ch, seed=5, amp=3.0), None
    scf = 1 << prm.sc_f
    ctx = api.Context(prm, (w + scf - 1) // scf * scf, (h + scf - 1) // scf * scf, prm.p_samp_s, 2 * n,
                      stream=stream.cuda_stream)
    ctx.upload_sequence_bidir_u8(0, n, clip, w, h)
    ctx.run(2 * n)
    cells = ((w + 7) // 8) * ((h + 7) // 8)
    tp = dict(capacity=4 * cells, spacing=8, alpha=0.01, beta=0.5, mb_alpha=0.01, mb_beta=0.002, min_eig=25.0)
    p = preprocess.TRAJ_DEFAULTS
    hwc = h * w * ch
    cap, bound, dim = tp["capacity"], preprocess.traj_bound(tp["capacity"], n, p["L"]), preprocess.traj_dim(p)
    dev = torch.from_numpy(clip.reshape(-1)).cuda()
    pts = torch.empty((n * cap * 3,), dtype=torch.int32, device="cuda")
    rec = torch.empty((bound * 7,), dtype=torch.int32, device="cuda")
    desc = torch.empty((bound * dim,), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    out = {}

    def traj():
        ctx.traj_begin(tp, p, dev.data_ptr(), w, h, memkind=api.MEM_DEVICE, points=pts.data_ptr())
        out["n"] = ctx.traj_advance(0, n, n, dev.data_ptr() + hwc, w, h, models=M, memkind=api.MEM_DEVICE,
                                    points=pts.data_ptr(), records=rec.data_ptr(), desc=desc.data_ptr())

    def track():
        ctx.track_begin(tp, dev.data_ptr(), w, h, memkind=api.MEM_DEVICE, points=pts.data_ptr())
        ctx.track_advance(0, n, n, dev.data_ptr() + hwc, w, h, memkind=api.MEM_DEVICE, points=pts.data_ptr())

    before = ctx.launch_count
    traj()
    launches = ctx.launch_count - before
    stats = ctx.traj_stats()
    alive = [int(c) for c in out["n"][0]]
    track()
    t_traj = t_track = t_run = None
    for _ in range(2):  # alternated, the second round kept
        t_traj = median_ms(stream, traj, reps)
        t_track = median_ms(stream, track, reps)
        t_run = median_ms(stream, lambda: ctx.run(2 * n), reps)
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        traj()
        torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
        if e.device_type.name == "CUDA":
            m = re.search(r"(\w+_kernel)", e.name)
            name = m.group(1) if m else e.name.strip()
            kern[name] = kern.get(name, 0.0) + e.device_time / 1000.0
    ctx.close()
    kern = {k: round(v, 4) for k, v in sorted(kern.items(), key=lambda kv: -kv[1])}
    hist_ms = kern.get("traj_hist_kernel")
    # live tracks before each pair: frame 0's seeds, then the list after pair k - 1
    live = sum(alive[:-1]) + alive[0]
    hist_bytes = live * p["N"] ** 2 * 36
    return {"traj_ms": round(t_traj, 4), "track_ms": round(t_track, 4), "run_ms": round(t_run, 4),
            "launches_per_call": launches, "stats": stats, "kernel_ms_profiled_call": kern,
            "hist_field_bytes": hist_bytes,
            "hist_field_TBps": round(hist_bytes / (hist_ms * 1e-3) / 1e12, 3) if hist_ms else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=64)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("traj_e2e: no CUDA device")
    res = {"card": card(), "pairs": a.pairs, "oppoint": 2, "memory": "device"}
    res["1024x436_gray_camera_models"] = measure(436, 1024, 1, a.pairs, a.reps, True)
    res["1920x1080_rgb_no_models"] = measure(1080, 1920, 3, a.pairs, a.reps, False)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
