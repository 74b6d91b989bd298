"""Scene flow on the device (ofdis_scene_flow_fullres), measured: one JSON line.

    python tools/sceneflow_e2e.py [--pairs 64] [--reps 50]

Workload: `pairs` pairs of KITTI's 1242x375 frame size, gray, at operating point 2: the flows of a
synth.synthetic_sequence clip (amplitude 3) run in one batch, a chained clip of pairs + 1 random disparity maps
(5 % unknown) read with disp_stride = one frame, every output (disp1_warped, status, motion) in device memory, and
ground truth and 3 classes in device memory for the evaluated variant.  Reported, each the median of `reps` calls
after warm-up, timed with device events on the context's stream:
  * the call without and with stats (the stats call includes its memset, its 2 KB copy and its synchronise);
  * the algorithmic bytes per pixel (DESIGN.md section 5.21): 16 read (flow 8, d0 4, the d1 gather 4), 17 written
    (disp1_warped 4, status 1, motion 12), plus 17 read for ground truth (4 + 4 + 8) and classes (1), over the time,
    against the H100 SXM data sheet's 3.35 TB/s.
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

CAM = dict(fx=721.5377, fy=721.5377, cx=609.5593, cy=172.854, baseline=0.5372, doffs=0.0)


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
    ap.add_argument("--pairs", type=int, default=64)
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("sceneflow_e2e: no CUDA device")
    h, w, n = 375, 1242, a.pairs
    stream = torch.cuda.Stream()
    prm = params.operating_point(2, w, noc=1)
    scf = 1 << prm.sc_f
    ctx = api.Context(prm, (w + scf - 1) // scf * scf, (h + scf - 1) // scf * scf, prm.p_samp_s, n,
                      stream=stream.cuda_stream)
    ctx.upload_sequence_u8(0, n, synth.synthetic_sequence(n + 1, h, w, 1, seed=5, amp=3.0), w, h)
    ctx.run(n)
    rng = np.random.default_rng(0)
    maps = rng.uniform(5, 60, (n + 1, h, w)).astype(np.float32)
    maps[rng.random(maps.shape) < 0.05] = np.nan
    pix = h * w
    with torch.cuda.stream(stream):
        d_maps = torch.from_numpy(maps).cuda()
        gt = [torch.from_numpy(maps[:-1].copy()).cuda(), torch.from_numpy(maps[1:].copy()).cuda(),
              torch.zeros((n, h, w, 2), device="cuda")]
        cls = torch.from_numpy(rng.integers(0, 3, (n, h, w)).astype(np.uint8)).cuda()
        out = {"disp1": torch.empty((n, h, w), device="cuda"),
               "status": torch.empty((n, h, w), dtype=torch.uint8, device="cuda"),
               "motion": torch.empty((n, h, w, 3), device="cuda")}
    stream.synchronize()
    ptrs = {k: v.data_ptr() for k, v in out.items()}
    out_stats = {}
    res = {"card": card(), "pairs": n, "size": "%dx%d" % (w, h), "oppoint": 2, "memory": "device"}

    def plain():
        ctx.scene_flow_fullres(0, n, d_maps.data_ptr(), d_maps.data_ptr() + 4 * pix, width_org=w, height_org=h,
                               camera=CAM, outputs=("disp1", "status", "motion"), memkind=api.MEM_DEVICE, out=ptrs,
                               disp_stride=pix)

    def evaluated():
        out_stats["v"] = ctx.scene_flow_fullres(0, n, d_maps.data_ptr(), d_maps.data_ptr() + 4 * pix, width_org=w,
                                              height_org=h, camera=CAM, outputs=("disp1", "status", "motion"),
                                              gt=[g.data_ptr() for g in gt], classes=cls.data_ptr(), nclasses=3,
                                              memkind=api.MEM_DEVICE, out=ptrs, disp_stride=pix)[1]

    before = ctx.launch_count
    plain()
    res["launches_per_call"] = ctx.launch_count - before
    evaluated()
    t_plain = t_eval = None
    for _ in range(2):  # warm-up round, then the kept round; the two variants alternate
        t_plain = median_ms(stream, plain, a.reps)
        t_eval = median_ms(stream, evaluated, a.reps)
    px = n * pix
    for name, t, per in (("call_no_stats", t_plain, 16 + 17), ("call_stats", t_eval, 16 + 17 + 17)):
        res[name] = {"ms": round(t, 4), "bytes_per_pixel": per, "TBps": round(px * per / (t * 1e-3) / 1e12, 3),
                     "share_of_3.35TBps": round(px * per / (t * 1e-3) / 3.35e12, 3)}
    st = out_stats["v"]
    res["sf_outliers_total"] = int(st["out_sf"].sum())
    res["sf_counted_total"] = int(st["n_sf"].sum())
    # the device outputs equal the restatement on one pair
    flows = np.empty((1, h, w, 2), np.float32)
    ctx.get_flow_fullres(0, 1, flows, w, h)
    ctx.sync()
    exp = preprocess.scene_flow(flows, maps[:1], maps[1:2], 1.0, CAM)
    got = out["motion"][:1].cpu().numpy()
    res["pair0_motion_bitwise"] = bool((got.view(np.uint32) == exp[2].view(np.uint32)).all())
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
