"""SOR chain (one sweep per launch, band boundaries through global memory) against the 16-CTA cluster (all sweeps in
flight, boundaries through distributed shared memory) on the same level: 1920 x 2048 gray flow refined at level 0,
16 bands of 128 rows, one row per SOR thread.  sor_max_cluster 8 forces the chain.  Prints one JSON line per batch
with the SOR time of level 0 (CUDA events, eager profiled passes) and the whole step (graph replay).
python tools/chain_vs_cluster.py [B ...]"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from of_dis_b200 import api, params, synth


def measure(B, max_cluster, steps=10):
    prm = params.from_cli_numbers("1 0 12 12 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0".split(), noc=1)
    h, w = 2048, 1920
    i0, i1, _ = synth.synthetic_pair(h, w, 1, seed=1, amp=6.0)
    st = torch.cuda.current_stream()
    ctx = api.Context(prm, w, h, prm.p_samp_s, B, stream=st.cuda_stream)
    ctx.set_option("sor_max_cluster", max_cluster)
    ctx.upload_frames_u8(0, B, np.ascontiguousarray(np.stack([np.stack([i0, i1])] * B)), w, h)
    ctx.set_graph_mode(True)
    for _ in range(2):
        ctx.run(B)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(st)
    for _ in range(steps):
        ctx.run(B)
    b.record(st)
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / steps
    flow = ctx.get_flow(0, prm.sc_l)
    ctx.set_graph_mode(False)
    lev = ctx.profile_levels(B, steps=steps)
    ctx.close()
    return {"ms_per_step": round(ms, 3), "sor_l0_ms": round(lev[0]["sor"], 3)}, flow


if __name__ == "__main__":
    st = torch.cuda.Stream()
    torch.cuda.set_stream(st)
    for B in [int(a) for a in sys.argv[1:]] or [1, 8]:
        cl, f_cl = measure(B, 16)
        ch, f_ch = measure(B, 8)
        same = bool(np.array_equal(f_cl.view(np.uint32), f_ch.view(np.uint32)))
        print(json.dumps({"wxh": "1920x2048", "pairs": B, "cluster16": cl, "chain": ch, "flows_bitwise_equal": same}), flush=True)
