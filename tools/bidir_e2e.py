"""Bidirectional flows and consistency masks on one GPU: 64 gray 1024x436 pairs at operating point 2 in both
directions (128 slots).

    python tools/bidir_e2e.py [--reps K] [--warmup W]

First checks, exit 1 otherwise: the flows after ofdis_upload_sequence_bidir_u8 are bitwise those after
ofdis_upload_frames_u8 of the 64 forward and the 64 swapped pairs, and ofdis_consistency_fullres of both directions
equals preprocess.consistency_check on the ofdis_get_flow_fullres outputs.  Then times, after W warm-up steps,
the median of K:
  (a) upload + pyramid of the 128 slots: the two-way sequence upload against ofdis_upload_frames_u8 of the 2 x 64
      pairs, from pinned host memory (CUDA events);
  (b) ofdis_consistency_fullres of 64 pairs in both directions, into device memory and into pinned host memory
      (CUDA events);
  (c) the whole step, 8-bit frames in, both full-resolution flows and both masks on the host: two-way upload ->
      graph run -> flows and masks to pinned memory, against two pair uploads -> graph run -> flows to the host ->
      the check in numpy (host clock around steps that end in a device synchronise).
Prints one JSON line with the card name and power limit read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from of_dis_b200 import api, params, preprocess, synth  # noqa: E402

N, H, W = 64, 436, 1024


def card():
    q = "name,power.limit"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))
    except (OSError, subprocess.SubprocessError):
        return {"name": torch.cuda.get_device_name(0), "power.limit": None}


def med(xs):
    return round(statistics.median(xs), 4)


def events(fn, reps, warmup, st):
    for _ in range(warmup):
        fn()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(st)
        fn()
        b.record(st)
        b.synchronize()
        out.append(a.elapsed_time(b))
    return med(out)


def wall(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    out = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        out.append((time.perf_counter() - t) * 1e3)
    return med(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    prm = params.operating_point(2, W, noc=1)
    scf = 1 << prm.sc_f
    Wp, Hp = (W + scf - 1) // scf * scf, (H + scf - 1) // scf * scf
    alpha, beta = api.CONSISTENCY_DEFAULTS[2]
    frames = synth.synthetic_sequence(N + 1, H, W, 1, seed=5)
    seq = torch.from_numpy(frames).pin_memory()
    pairs = np.concatenate([np.stack([frames[:-1], frames[1:]], axis=1), np.stack([frames[1:], frames[:-1]], axis=1)])
    pairs = torch.from_numpy(np.ascontiguousarray(pairs)).pin_memory()
    st = torch.cuda.Stream()
    ctx = api.Context(prm, Wp, Hp, prm.p_samp_s, 2 * N, stream=st.cuda_stream)
    ctx.set_graph_mode(True)
    flows = torch.empty((2 * N, H, W, 2), dtype=torch.float32).pin_memory()
    masks = torch.empty((2, N, H, W), dtype=torch.uint8).pin_memory()
    dmask = torch.empty((2, N, H, W), dtype=torch.uint8, device="cuda")

    up_bidir = lambda: ctx.upload_sequence_bidir_u8(0, N, seq.data_ptr(), W, H)  # noqa: E731
    up_pairs = lambda: ctx.upload_frames_u8(0, 2 * N, pairs.data_ptr(), W, H)  # noqa: E731

    def check(dev):
        out = dmask if dev else masks
        kind = api.MEM_DEVICE if dev else api.MEM_HOST
        for d, (f0, b0) in enumerate(((0, N), (N, 0))):
            m = out[d].data_ptr() if dev else out[d].numpy()  # host: a numpy view of the pinned buffer
            ctx.consistency_fullres(f0, f0 + N, b0, W, H, alpha, beta, memkind=kind, mask=m)

    # ---- bitwise checks
    got = {}
    for name, up in (("bidir", up_bidir), ("pairs", up_pairs)):
        up()
        ctx.run(2 * N)
        ctx.get_flow_fullres(0, 2 * N, flows.data_ptr(), W, H)
        ctx.sync()
        got[name] = flows.numpy().copy()
    if not np.array_equal(got["bidir"].view(np.uint32), got["pairs"].view(np.uint32)):
        print("FAIL: the two-way sequence upload's flows differ from the pair upload's")
        return 1
    check(False)
    ctx.sync()
    fl = got["bidir"]
    for d, (f0, b0) in enumerate(((0, N), (N, 0))):
        for i in range(N):
            if not np.array_equal(masks[d, i].numpy(), preprocess.consistency_check(fl[f0 + i], fl[b0 + i], alpha, beta)[0]):
                print("FAIL: mask of slot %d differs from preprocess.consistency_check" % (f0 + i))
                return 1
    share = [float((masks.numpy() == v).mean()) for v in (0, 1, 2)]

    # ---- (a) upload + pyramid
    res = {"card": card(), "pairs": N, "size": [W, H], "checks": "bitwise ok",
           "mask_share_consistent_inconsistent_leaves": [round(x, 4) for x in share]}
    res["a_upload_ms"] = {"bidir_sequence": events(up_bidir, a.reps, a.warmup, st),
                          "pairs_2n": events(up_pairs, a.reps, a.warmup, st)}
    # ---- (b) the check alone
    up_bidir()
    ctx.run(2 * N)
    res["b_consistency_ms_both_directions"] = {"device_out": events(lambda: check(True), a.reps, a.warmup, st),
                                               "pinned_host_out": events(lambda: check(False), a.reps, a.warmup, st)}

    # ---- (c) the whole step
    def step_new():
        up_bidir()
        ctx.run(2 * N)
        ctx.get_flow_fullres(0, 2 * N, flows.data_ptr(), W, H)
        check(False)
        ctx.sync()

    def step_today():
        up_pairs()
        ctx.run(2 * N)
        ctx.get_flow_fullres(0, 2 * N, flows.data_ptr(), W, H)
        ctx.sync()
        f = flows.numpy()
        for d, (f0, b0) in enumerate(((0, N), (N, 0))):
            for i in range(N):
                masks[d, i].numpy()[...] = preprocess.consistency_check(f[f0 + i], f[b0 + i], alpha, beta)[0]

    res["c_step_ms"] = {"bidir_device_check": wall(step_new, a.reps, a.warmup),
                        "pair_uploads_numpy_check": wall(step_today, max(2, a.reps // 3), 1)}
    ctx.close()
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
