"""Frame interpolation on the device (ofdis_interpolate_fullres), measured: one JSON line.

    python tools/interp_e2e.py [--pairs 64] [--reps 20]

For gray and RGB 1024x436 clips at operating point 2 (64 pairs, their backward partners in the same launch):
  * the call's device-event time at t = 0.5 into device memory (frames on the device), median of `reps` calls after
    two warm-up calls, next to the same batch's ofdis_run time (median of `reps` runs);
  * the hole-filling rounds: the fill launches of one call (rounds run in batches of 8, 16, ...) and the exact round
    count of the first two pairs from preprocess.interpolate_frames, against which those pairs are checked bitwise;
  * Middlebury's interpolation error (Baker et al., IJCV 2011): the RMS over pixels and channels against the held-out
    frame of a synthetic clip interpolated from frames (2k, 2k + 2), next to the plain blend (1 - t) I0 + t I1 and the
    held frame I0.
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


def context(prm, n, stream):
    scf = 1 << prm.sc_f
    return api.Context(prm, (W + scf - 1) // scf * scf, (H + scf - 1) // scf * scf, prm.p_samp_s, 2 * n,
                       stream=stream.cuda_stream)


def measure(ch, n, reps):
    stream = torch.cuda.Stream()
    prm = params.operating_point(2, W, noc=ch)
    clip = synth.synthetic_sequence(n + 1, H, W, ch, seed=5, amp=3.0)
    ctx = context(prm, n, stream)
    ctx.upload_sequence_bidir_u8(0, n, clip, W, H)
    ctx.run(2 * n)
    hwc = H * W * ch
    dev = torch.from_numpy(clip.reshape(-1)).cuda()
    out = torch.empty((n, H, W, ch), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()

    def call():
        ctx.interpolate_fullres(0, n, n, dev.data_ptr(), dev.data_ptr() + hwc, 0.5, W, H, out=out.data_ptr(),
                                memkind=api.MEM_DEVICE, frame_stride=hwc)

    before = ctx.launch_count
    call()
    fill_launches = ctx.launch_count - before - 5  # two masks, splat, resolve, blend
    call()
    t_interp = median_ms(stream, call, reps)
    t_run = median_ms(stream, lambda: ctx.run(2 * n), reps)
    # bitwise check of the first two pairs (the run above recomputed the same flows)
    flows = np.empty((2 * n, H, W, 2), np.float32)
    ctx.get_flow_fullres(0, 2 * n, flows, W, H)
    call()
    ctx.sync()
    exp, _, rounds = preprocess.interpolate_frames(clip[:2], clip[1:3], flows[:2], flows[n:n + 2], 0.5, 0.01, 0.5,
                                                   with_rounds=True)
    got = out[:2].cpu().numpy().reshape(exp.shape)
    ctx.close()
    return {"interp_ms": round(t_interp, 4), "run_ms": round(t_run, 4), "fill_launches": fill_launches,
            "fill_rounds_first_pairs": rounds, "bitwise_first_pairs": bool(np.array_equal(got, exp))}


def quality(ch, pairs):
    """Interpolation error of (2k, 2k + 2) -> 2k + 1 over `pairs` triples of a synthetic clip."""
    stream = torch.cuda.Stream()
    prm = params.operating_point(2, W, noc=ch)
    clip = synth.synthetic_sequence(2 * pairs + 1, H, W, ch, seed=7, amp=3.0)
    ends = np.ascontiguousarray(clip[::2])
    ctx = context(prm, pairs, stream)
    ctx.upload_sequence_bidir_u8(0, pairs, ends, W, H)
    ctx.run(2 * pairs)
    out, _ = ctx.interpolate_fullres(0, pairs, pairs, ends[:-1], ends[1:], 0.5, W, H)
    ctx.close()
    held = clip[1::2].astype(np.float64)
    rms = lambda a: float(np.sqrt(np.mean((np.asarray(a, np.float64).reshape(held.shape) - held) ** 2)))  # noqa: E731
    naive = 0.5 * clip[0:-1:2].astype(np.float64) + 0.5 * clip[2::2].astype(np.float64)
    return {"ie_interp": round(rms(out), 4), "ie_blend": round(rms(naive), 4), "ie_held_i0": round(rms(clip[0:-1:2]), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=64)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("interp_e2e: no CUDA device")
    res = {"card": card(), "size": "%dx%d" % (W, H), "pairs": a.pairs, "oppoint": 2, "t": 0.5, "memory": "device"}
    for ch, tag in ((1, "gray"), (3, "rgb")):
        res[tag] = measure(ch, a.pairs, a.reps)
        res[tag].update(quality(ch, 8))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
