"""A/B of the lanes per patch of the P = 8 patch kernel (ofdis_set_option("patch_lanes", 8 | 4)) on the bench workload
(operating point 2, 1024x436, one stream): per batch of 1 / 8 / 64 pairs, the patch class's eager ms per step
(profile_kernels, CUDA events around each patch launch) and the graph-replayed step time, the two settings measured
alternately in three rounds (the best round is reported); the flows of every pair of the two settings are compared
bit for bit.
python tools/patch_ab.py [B ...]"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from of_dis_b200 import api, params, synth

LANES = (8, 4)
prm = params.operating_point(2, 1024)
h, w = 436, 1024
pairs = [synth.synthetic_pair(h, w, 1, seed=s, amp=6.0)[:2] for s in range(4)]
scf = 1 << prm.sc_f
W, H = (w + scf - 1) // scf * scf, (h + scf - 1) // scf * scf
for B in [int(a) for a in sys.argv[1:]] or [1, 8, 64]:
    frames = np.ascontiguousarray(np.stack([np.stack(pairs[f % len(pairs)]) for f in range(B)]))
    ctxs = {}
    for lanes in LANES:
        ctx = api.Context(prm, W, H, prm.p_samp_s, B)
        ctx.set_option("patch_lanes", lanes)
        ctx.upload_frames_u8(0, B, frames, w, h)
        ctxs[lanes] = ctx
    patch_ms = {k: 1e9 for k in LANES}
    step_ms = {k: 1e9 for k in LANES}
    for _ in range(3):
        for lanes in LANES:
            ctx = ctxs[lanes]
            ctx.set_graph_mode(False)
            prof = ctx.profile_kernels(B, steps=5)
            patch_ms[lanes] = min(patch_ms[lanes], prof["patch"]["ms_per_step"])
            ctx.set_graph_mode(True)
            for _ in range(5):
                ctx.run(B)
            ctx.sync()
            t0 = time.perf_counter()
            for _ in range(50):
                ctx.run(B)
            ctx.sync()
            step_ms[lanes] = min(step_ms[lanes], (time.perf_counter() - t0) * 1e3 / 50)
    flows = {k: np.stack([ctxs[k].get_flow(f, prm.sc_l) for f in range(B)]) for k in LANES}
    same = np.array_equal(flows[8].view(np.uint32), flows[4].view(np.uint32))
    for ctx in ctxs.values():
        ctx.close()
    print(json.dumps({"pairs": B,
                      "patch_ms_per_step": {"lanes8": round(patch_ms[8], 4), "lanes4": round(patch_ms[4], 4)},
                      "graph_ms_per_step": {"lanes8": round(step_ms[8], 4), "lanes4": round(step_ms[4], 4)},
                      "flows_bitwise_equal": bool(same)}), flush=True)
