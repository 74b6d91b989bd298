"""Filtered disparities on the device (ofdis_disparity_fullres), measured: one JSON line.

    python tools/disparity_e2e.py [--pairs 64] [--reps 20]

For gray and RGB 1024x436 stereo clips at operating point 2 (64 pairs with the two-way upload: 128 slots, the right
views as swapped slots), device outputs:
  * the device-event time of one call over the 64 forward slots against their partners with each stage on and off
    (lr_check, speckles 100 px / 1 px, fill) and every output asked for, median of `reps` calls after two warm-up
    calls, next to ofdis_run of the same 128 slots;
  * the time of each kernel of the all-on call (torch.profiler, CUDA activities, in a pass of its own after the timed
    calls; the sum over the `reps` calls divided by `reps`);
  * a bitwise check of the first pairs of the all-on call against preprocess.disparity_filter;
  * KITTI D1 (in numpy: a pixel is an outlier when |d - gt| > 3 and > 0.05 gt, NaN counts as one) on
    synth.layered_stereo at 1024x436 (background 8 px, a foreground block at 24 px), for the raw disparity -F, the
    left-right checked one without fill (invalid pixels count as outliers; its density is reported) and the
    filtered-and-filled one, over all pixels and over the pixels that are not occluded.  A sanity figure for the
    filter on a synthetic scene, not an accuracy claim.
The card's name and power limit are read in the same run."""
import argparse
import itertools
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from of_dis_b200 import api, params, preprocess, synth

H, W = 436, 1024
CHECK_PAIRS = 2
CAM = dict(fx=721.5, fy=721.5, cx=512.0, cy=218.0, baseline=0.54, doffs=0.0)


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


def measure(ch, n, reps):
    stream = torch.cuda.Stream()
    prm = params.operating_point(2, W, noc=ch, nop=1)
    clip = synth.synthetic_sequence(n + 1, H, W, ch, seed=5, amp=3.0, stereo=True)
    scf = 1 << prm.sc_f
    ctx = api.Context(prm, (W + scf - 1) // scf * scf, (H + scf - 1) // scf * scf, prm.p_samp_s, 2 * n,
                      stream=stream.cuda_stream)
    ctx.upload_sequence_bidir_u8(0, n, clip, W, H)
    ctx.run(2 * n)
    run_ms = median_ms(stream, lambda: ctx.run(2 * n), reps)
    dev = {"disp": torch.empty((n, H, W), device="cuda"), "status": torch.empty((n, H, W), dtype=torch.uint8,
                                                                                  device="cuda"),
           "depth": torch.empty((n, H, W), device="cuda"), "xyz": torch.empty((n, H, W, 3), device="cuda")}
    ptrs = {k: v.data_ptr() for k, v in dev.items()}
    torch.cuda.synchronize()
    res = {"ofdis_run_ms": run_ms, "call_ms": {}}
    for lr, sp, fill in itertools.product((0, 1), (0, 1), (0, 1)):
        filt = dict(lr_check=lr, alpha=0.0, beta=1.0, speckle_size=100 if sp else 0, speckle_diff=1.0, fill=fill)

        def call():
            ctx.disparity_fullres(0, n, n, W, H, camera=CAM, outputs=tuple(dev), memkind=api.MEM_DEVICE, out=ptrs,
                                  **filt)
        for _ in range(2):
            call()
        res["call_ms"]["lr%d_speckle%d_fill%d" % (lr, sp, fill)] = median_ms(stream, call, reps)
    stream.synchronize()
    full = np.empty((2 * n, H, W, 1), np.float32)
    ctx.get_flow_fullres(0, 2 * n, full, W, H)
    ctx.sync()
    ok = True
    for k in range(CHECK_PAIRS):
        exp = preprocess.disparity_filter(full[k], full[n + k], False, lr_check=1, alpha=0.0, beta=1.0,
                                          speckle_size=100, speckle_diff=1.0, fill=1, camera=CAM)
        got = [dev[name][k].cpu().numpy() for name in ("disp", "status", "depth", "xyz")]
        ok &= all(np.array_equal(np.asarray(g).view(np.uint8), np.asarray(e).view(np.uint8)) for g, e in zip(got, exp))
        if k == 0:
            res["status_counts_pair0"] = [int((got[1] == s).sum()) for s in range(5)]
    res["bitwise_equal_to_restatement"] = bool(ok)
    filt = dict(lr_check=1, alpha=0.0, beta=1.0, speckle_size=100, speckle_diff=1.0, fill=1)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            ctx.disparity_fullres(0, n, n, W, H, camera=CAM, outputs=tuple(dev), memkind=api.MEM_DEVICE, out=ptrs,
                                  **filt)
        stream.synchronize()
    kernels = {}
    for ev in prof.key_averages():
        if ev.key.startswith("ofdis::") or "disp_" in ev.key:
            name = ev.key.split("disp_", 1)[1].split("(")[0].split("<")[0] if "disp_" in ev.key else ev.key
            t = getattr(ev, "device_time_total", None)
            t = ev.cuda_time_total if t is None else t
            kernels["disp_" + name] = kernels.get("disp_" + name, 0.0) + t / 1000.0 / reps
    res["kernel_ms_all_on"] = kernels
    ctx.close()
    return res


def d1(d, gt, mask):
    """KITTI's D1 share of outliers over `mask`: |d - gt| > 3 and > 0.05 gt; NaN is an outlier."""
    e = np.abs(d - gt)
    good = (e <= 3.0) | (e <= 0.05 * gt)
    return float((~good[mask]).mean())


def layered_d1(ch):
    prm = params.operating_point(2, W, noc=ch, nop=1)
    left, right, gt, occ = synth.layered_stereo(H, W, ch, seed=11)
    scf = 1 << prm.sc_f
    ctx = api.Context(prm, (W + scf - 1) // scf * scf, (H + scf - 1) // scf * scf, prm.p_samp_s, 2)
    ctx.upload_sequence_bidir_u8(0, 1, np.ascontiguousarray(np.stack([left, right])), W, H)
    ctx.run(2)
    full = np.empty((2, H, W, 1), np.float32)
    ctx.get_flow_fullres(0, 2, full, W, H)
    ctx.sync()
    raw = -full[0, ..., 0]
    checked = ctx.disparity_fullres(0, 1, 1, W, H, lr_check=1, speckle_size=100, speckle_diff=1.0, fill=0,
                                    outputs=("disp",))["disp"][0]
    filled = ctx.disparity_fullres(0, 1, 1, W, H, lr_check=1, speckle_size=100, speckle_diff=1.0, fill=1,
                                   outputs=("disp",))["disp"][0]
    ctx.close()
    allpix, noc = np.ones_like(occ), ~occ
    out = {"occluded_share": float(occ.mean())}
    for name, d in (("raw", raw), ("checked", checked), ("filled", filled)):
        out[name] = {"d1_all": d1(d, gt, allpix), "d1_noc": d1(d, gt, noc), "d1_occ": d1(d, gt, occ),
                     "density": float(np.isfinite(d).mean())}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=64)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("disparity_e2e: no CUDA device")
    out = {"card": card(), "pairs": a.pairs, "size": [W, H], "op": 2}
    for ch, name in ((1, "gray"), (3, "rgb")):
        out[name] = measure(ch, a.pairs, a.reps)
        out[name]["layered_d1"] = layered_d1(ch)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
