"""Stereo ego-motion on the device (ofdis_egomotion_fullres), measured: one JSON line.

    python tools/egomotion_e2e.py [--pairs 64] [--reps 20]

For a gray 1242x375 clip of synth.rigid_stereo_clip (KITTI's camera; the rig moves 0.9 m forward and turns 0.5 deg,
then back, pair by pair, so that it stays in the scene; a box moves 2 cm sideways per frame on its own) at operating point 2, 64 pairs with the two-way upload (128 slots), the clip's
disparities in device memory as one chained array, fb_check against the backward slots, step 8, 5 refits, device
outputs (mask, residual, object motion):
  * for 1024 and 4096 hypotheses, the device-event time of one call over the 64 pairs, median of `reps` calls after
    two warm-up calls, next to ofdis_run of the same 128 slots;
  * each kernel's time (torch.profiler, CUDA activities, in a pass of its own after the timed calls; the sum over the
    `reps` calls divided by `reps`), and the score kernel's inlier tests per second: hypotheses x correspondences,
    summed over the pairs, over its time;
  * a bitwise check of the first pair of the last call against preprocess.egomotion.
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


def measure(n, reps):
    stream = torch.cuda.Stream()
    prm = params.operating_point(2, W, noc=1)
    fwd = np.concatenate([synth.axis_angle((0.0, math.radians(0.5), 0.0)), np.array([[0.0], [0.0], [-0.9]])], 1)
    back = np.concatenate([fwd[:, :3].T, -(fwd[:, :3].T @ fwd[:, 3:])], 1)  # the inverse: the rig stays in the scene
    clip = synth.rigid_stereo_clip(n, H, W, 1, 5, CAM, [fwd if k % 2 == 0 else back for k in range(n)],
                                   block={"velocity": (0.02, 0.0, 0.0)})
    scf = 1 << prm.sc_f
    ctx = api.Context(prm, (W + scf - 1) // scf * scf, (H + scf - 1) // scf * scf, prm.p_samp_s, 2 * n,
                      stream=stream.cuda_stream)
    ctx.upload_sequence_bidir_u8(0, n, clip["left"], W, H)
    ctx.run(2 * n)
    run_ms = median_ms(stream, lambda: ctx.run(2 * n), reps)
    d_disp = torch.from_numpy(clip["disp"]).cuda()
    dev = {"mask": torch.empty((n, H, W), dtype=torch.uint8, device="cuda"),
           "residual": torch.empty((n, H, W, 2), device="cuda"),
           "object_motion": torch.empty((n, H, W, 3), device="cuda")}
    ptrs = {k: v.data_ptr() for k, v in dev.items()}
    torch.cuda.synchronize()
    res = {"ofdis_run_ms": run_ms, "calls": {}}
    pix = H * W
    for nh in (1024, 4096):
        p = dict(step=8, fb_check=1, alpha=0.01, beta=0.5, edge_diff=1.0, hypotheses=nh, threshold=1.0, refine=5,
                 seed=0)

        def call(f1=n):
            return ctx.egomotion_fullres(0, f1, d_disp.data_ptr(), d_disp.data_ptr() + 4 * pix, p, camera=CAM,
                                         width_org=W, height_org=H, b0=n, disp_stride=pix, outputs=tuple(ptrs),
                                         out=ptrs, memkind=api.MEM_DEVICE)
        for _ in range(2):
            pose, stats, _ = call()
        ms = median_ms(stream, call, reps)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                call()
            stream.synchronize()
        kernels = {}
        for ev in prof.key_averages():
            if "ego_" in ev.key:
                name = "ego_" + ev.key.split("ego_", 1)[1].split("(")[0].split("<")[0]
                t = getattr(ev, "device_time_total", None)
                t = ev.cuda_time_total if t is None else t
                kernels[name] = kernels.get(name, 0.0) + t / 1000.0 / reps
        tests = float(nh) * float(stats["n_corr"].sum())
        score = kernels.get("ego_score_kernel", 0.0)
        t_err, r_err = preprocess.pose_errors(pose, preprocess.chain_poses(clip["poses"]))
        res["calls"]["hyp_%d" % nh] = {
            "call_ms": ms, "kernel_ms": kernels, "score_tests": tests,
            "score_tests_per_s": tests / (score / 1000.0) if score > 0 else None,
            "status": sorted(set(stats["status"].tolist())), "n_corr_mean": float(stats["n_corr"].mean()),
            "n_inliers_mean": float(stats["n_inliers"].mean()), "t_err_rel_max": float(t_err.max() / 0.9),
            "r_err_deg_max": float(r_err.max())}
    # the first pair of the last (4096) call against the restatement
    full = np.empty((2 * n, H, W, 2), np.float32)
    ctx.get_flow_fullres(0, 2 * n, full, W, H)
    ctx.sync()
    exp = preprocess.egomotion(full[:1], full[n:n + 1], clip["disp"][:1], clip["disp"][1:2], CAM, p)
    pose, stats, _ = call(1)
    got = (pose, stats) + tuple(dev[k][:1].cpu().numpy() for k in ("mask", "residual", "object_motion"))
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
        sys.exit("egomotion_e2e: no CUDA device")
    out = {"card": card(), "pairs": a.pairs, "size": [W, H], "op": 2}
    out["gray"] = measure(a.pairs, a.reps)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
