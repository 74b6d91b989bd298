"""Global camera motion on the device (ofdis_global_motion_fullres), measured: one JSON line.

    python tools/global_motion_e2e.py [--pairs 64] [--reps 20]

For gray and RGB 1024x436 clips of synth.global_motion_clip (rotation 0.5 deg, zoom 1.01 and a 3 px shift per frame, a
rectangle of 15 % of the frame moving on its own) at operating point 2, 64 pairs with the two-way upload (128 slots),
fb_check against the backward slots, step 8, 3 refits, device outputs (mask, residual, registered frames):
  * for each model and 1024 and 4096 hypotheses, the device-event time of one call over the 64 pairs, median of `reps`
    calls after two warm-up calls, next to ofdis_run of the same 128 slots;
  * each kernel's time (torch.profiler, CUDA activities, in a pass of its own after the timed calls; the sum over the
    `reps` calls divided by `reps`), and the score kernel's inlier tests per second: hypotheses x correspondences,
    summed over the pairs, over its time;
  * a bitwise check of the first pair of the homography call against preprocess.global_motion.
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
MODELS = ("similarity", "affine", "homography")


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
    prm = params.operating_point(2, W, noc=ch)
    Hm = synth.similarity_about_centre(H, W, 0.5, 1.01, (3.0, 0.0))
    clip, _, _ = synth.global_motion_clip(n, H, W, ch, seed=5, H=Hm)
    scf = 1 << prm.sc_f
    ctx = api.Context(prm, (W + scf - 1) // scf * scf, (H + scf - 1) // scf * scf, prm.p_samp_s, 2 * n,
                      stream=stream.cuda_stream)
    ctx.upload_sequence_bidir_u8(0, n, clip, W, H)
    ctx.run(2 * n)
    run_ms = median_ms(stream, lambda: ctx.run(2 * n), reps)
    dclip = torch.from_numpy(clip).cuda()
    dev = {"mask": torch.empty((n, H, W), dtype=torch.uint8, device="cuda"),
           "residual": torch.empty((n, H, W, 2), device="cuda"),
           "registered": torch.empty((n, H, W) + ((ch,) if ch > 1 else ()), dtype=torch.uint8, device="cuda")}
    ptrs = {k: v.data_ptr() for k, v in dev.items()}
    torch.cuda.synchronize()
    res = {"ofdis_run_ms": run_ms, "calls": {}}
    stats = None
    for model in MODELS:
        for nh in (1024, 4096):
            p = dict(model=model, step=8, fb_check=1, alpha=0.01, beta=0.5, hypotheses=nh, threshold=1.0, refine=3,
                     seed=0)

            def call():
                return ctx.global_motion_fullres(0, n, p, width_org=W, height_org=H, b0=n, i1=dclip[1:].data_ptr(),
                                                 memkind=api.MEM_DEVICE, **ptrs)
            for _ in range(2):
                _, stats = call()
            ms = median_ms(stream, call, reps)
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(reps):
                    call()
                stream.synchronize()
            kernels = {}
            for ev in prof.key_averages():
                if "motion_" in ev.key:
                    name = "motion_" + ev.key.split("motion_", 1)[1].split("(")[0].split("<")[0]
                    t = getattr(ev, "device_time_total", None)
                    t = ev.cuda_time_total if t is None else t
                    kernels[name] = kernels.get(name, 0.0) + t / 1000.0 / reps
            tests = float(nh) * float(stats["n_corr"].sum())
            score = kernels.get("motion_score_kernel", 0.0)
            res["calls"]["%s_%d" % (model, nh)] = {
                "call_ms": ms, "kernel_ms": kernels, "score_tests": tests,
                "score_tests_per_s": tests / (score / 1000.0) if score > 0 else None,
                "status": sorted(set(stats["status"].tolist())), "n_corr_mean": float(stats["n_corr"].mean()),
                "n_inliers_mean": float(stats["n_inliers"].mean())}
    # the first pair of the last (homography, 4096) call against the restatement
    full = np.empty((2 * n, H, W, 2), np.float32)
    ctx.get_flow_fullres(0, 2 * n, full, W, H)
    ctx.sync()
    exp = preprocess.global_motion(full[0], full[n], clip[1], p)
    models, stats = ctx.global_motion_fullres(0, 1, p, width_org=W, height_org=H, b0=n, i1=dclip[1:].data_ptr(),
                                              memkind=api.MEM_DEVICE, **ptrs)
    got = (models[0], stats[0], dev["mask"][0].cpu().numpy(), dev["residual"][0].cpu().numpy(),
           dev["registered"][0].cpu().numpy())
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
        sys.exit("global_motion_e2e: no CUDA device")
    out = {"card": card(), "pairs": a.pairs, "size": [W, H], "op": 2}
    for ch, name in ((1, "gray"), (3, "rgb")):
        out[name] = measure(ch, a.pairs, a.reps)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
