"""Video stabilisation on the device (ofdis_stab_push), measured: one JSON line.

    python tools/stabilize_e2e.py [--frames 64] [--reps 20]

For 1024x436 gray and 1920x1080 RGB frames at radius 15, crop 0.1 with the limit, in device memory on one stream:
  * the device-event time of one push of `frames` frames once the clip is longer than the radius (so that every push
    emits `frames` frames), median of `reps` pushes after two warm-up pushes;
  * each kernel's time (torch.profiler, CUDA activities, in a pass of its own after the timed pushes; the sum over the
    `reps` pushes divided by `reps`), and stab_warp_kernel's algorithmic bytes per second -- one read and one write of
    every emitted frame -- against the H100 SXM's data-sheet 3.35 TB/s;
  * the push's other work: the copy of the pushed frames into the frame ring (one read and one write of each).
The frames are random bytes (the warp's cost does not depend on them) under the camera of synth.shaky_clip: a pan of
(1, 0.5) px per frame and a random shake of up to 2 px and 0.5 degrees.  The card's name and power limit are read in
the same run."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from of_dis_b200 import api, params, synth

HBM_BPS = 3.35e12
SIZES = ((1024, 436, 1, "gray_1024x436"), (1920, 1080, 3, "rgb_1920x1080"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def shaky_models(n, h, w, seed=0, pan=(1.0, 0.5), jitter=2.0):
    """The per-pair models of synth.shaky_clip's camera, without rendering the frames."""
    rng = np.random.default_rng(seed + 7)
    poses = []
    for t in range(n + 1):
        J = synth.similarity_about_centre(h, w, rng.uniform(-0.25, 0.25) * jitter, 1.0,
                                          (rng.uniform(-1, 1) * jitter, rng.uniform(-1, 1) * jitter))
        poses.append(J @ np.array([[1.0, 0.0, t * pan[0]], [0.0, 1.0, t * pan[1]], [0.0, 0.0, 1.0]]))
    return np.stack([poses[t + 1] @ np.linalg.inv(poses[t]) for t in range(n)])


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


def measure(w, h, ch, n, reps):
    stream = torch.cuda.Stream()
    prm = params.operating_point(2, w, noc=ch)
    scf = 1 << prm.sc_f
    ctx = api.Context(prm, (w + scf - 1) // scf * scf, (h + scf - 1) // scf * scf, prm.p_samp_s, n,
                      stream=stream.cuda_stream)
    shape = (n, h, w) + ((ch,) if ch > 1 else ())
    gen = torch.Generator(device="cuda").manual_seed(1)
    frames = torch.randint(0, 256, shape, dtype=torch.uint8, device="cuda", generator=gen)
    out = torch.empty(shape, dtype=torch.uint8, device="cuda")
    models = shaky_models(n, h, w)
    hwc = h * w * ch
    torch.cuda.synchronize()
    p = dict(radius=15, crop=0.1, limit=1)
    ctx.stab_begin(p, frames[0].data_ptr(), w, h, memkind=api.MEM_DEVICE)
    emitted = []

    def push():
        (_, k), info = ctx.stab_push(models, frames.data_ptr(), frame_stride=hwc, memkind=api.MEM_DEVICE,
                                     out=out.data_ptr())
        emitted.append(k)
        return info

    for _ in range(2):
        push()
    ms = median_ms(stream, push, reps)
    assert all(k == n for k in emitted[1:]), emitted
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            info = push()
        stream.synchronize()
    kernels, copy_ms = {}, 0.0
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        t = (ev.cuda_time_total if t is None else t) / 1000.0 / reps
        if "stab_" in ev.key:
            name = "stab_" + ev.key.split("stab_", 1)[1].split("(")[0].split("<")[0]
            kernels[name] = kernels.get(name, 0.0) + t
        elif "Memcpy" in ev.key or "memcpy" in ev.key:
            copy_ms += t
    warp = kernels.get("stab_warp_kernel", 0.0)
    warp_bytes = 2.0 * hwc * n
    ctx.stab_finish(memkind=api.MEM_DEVICE, out=out.data_ptr())
    ctx.close()
    return {"push_ms": ms, "kernel_ms": kernels, "copy_ms": copy_ms, "frames_per_push": n,
            "warp_bytes": warp_bytes, "warp_bytes_per_s": warp_bytes / (warp / 1000.0) if warp > 0 else None,
            "warp_share_of_hbm": warp_bytes / (warp / 1000.0) / HBM_BPS if warp > 0 else None,
            "lower_bound_ms": warp_bytes / HBM_BPS * 1000.0, "min_lambda": float(info["lambda"].min()),
            "status": sorted(set(info["status"].tolist()))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("stabilize_e2e: no CUDA device")
    out = {"card": card(), "radius": 15, "crop": 0.1, "limit": 1}
    for w, h, ch, name in SIZES:
        out[name] = measure(w, h, ch, a.frames, a.reps)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
