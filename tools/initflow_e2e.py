"""Init flow from a full-resolution flow and the warm start for video, on one GPU.

    python tools/initflow_e2e.py [--reps K] [--pairs N]

1. The preparation (ofdis_set_initflow_fullres: replicate padding, x 2^-(sc_f+1), INTER_AREA to level sc_f+1) by
   CUDA events, from pinned host memory (copy included) and from device memory, and ofdis_set_initflow_from_result
   (flow_upsample_kernel into the scratch + the preparation): 64 pairs of 1024x436 gray at operating point 2, and
   8 pairs of 1920x1080 RGB with the 20 numbers of BASELINE configs[2].  The prepared level is checked against
   preprocess.initflow_from_fullres first (exit 1 if it differs).
2. The per-pair step of a clip (N+1 frames of synthetic_sequence, 1024x436 gray, operating point 2), one pair per
   launch, graph mode: upload the pair -> [warm: ofdis_set_initflow_from_result of the previous pair] -> run ->
   ofdis_get_flow_fullres on the device.  Cold and warm start alternate; CUDA events around each whole clip.
3. EPE of both against the clip's synthetic flow (synth.synthetic_flow), mean over pairs and pixels.
Prints one JSON line with the card's name, power limit and SM clock, read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from of_dis_b200 import api, params, preprocess, synth  # noqa: E402

CASES = {
    "64x1024x436_gray_op2": dict(n=64, size=(436, 1024), ch=1, prm=lambda: params.operating_point(2, 1024, noc=1)),
    "8x1920x1080_rgb_cfg3": dict(n=8, size=(1080, 1920), ch=3, prm=lambda: params.from_cli_numbers(
        "6 2 16 16 0.05 0.95 0 12 0.75 0 1 1 1 10 10 5 1 3 1.6 0".split(), noc=3)),
}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))
    except (OSError, subprocess.SubprocessError):
        return {"name": torch.cuda.get_device_name(0), "power.limit": None, "clocks.sm": None, "clocks.max.sm": None}


def context(prm, h, w, n, stream):
    s = 2 << prm.sc_f  # the padding of a run with an init flow
    return api.Context(prm, -(-w // s) * s, -(-h // s) * s, prm.p_samp_s, n, stream=stream)


def timed(st, fn, reps):
    """Median ms of fn() over reps, CUDA events on the context's stream."""
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(st)
        fn()
        b.record(st)
        b.synchronize()
        out.append(a.elapsed_time(b))
    return round(statistics.median(out), 4)


def preparation(name, c, reps):
    n, (h, w), ch = c["n"], c["size"], c["ch"]
    prm = c["prm"]()
    st = torch.cuda.Stream()  # the context's stream: the events below are recorded on it
    ctx = context(prm, h, w, n, st.cuda_stream)
    u, v = synth.synthetic_flow(h, w, 6.0)
    rng = np.random.default_rng(1)
    flows = np.ascontiguousarray(np.stack([np.stack([u, v], -1) + rng.standard_normal((h, w, 2)) for _ in range(n)]),
                                 np.float32)
    host = torch.from_numpy(flows).pin_memory()
    dev = host.cuda()
    torch.cuda.synchronize()
    ctx.set_initflow_fullres(0, n, dev.data_ptr(), w, h, memkind=api.MEM_DEVICE)
    ctx.sync()
    for f in (0, n - 1):
        exp = preprocess.initflow_from_fullres(flows[f], prm.sc_f)
        if not np.array_equal(ctx.get_flow(f, prm.sc_f + 1).view(np.uint32), exp.view(np.uint32)):
            print("%s: the prepared init flow of pair %d differs from the restatement" % (name, f), file=sys.stderr)
            sys.exit(1)
    frames = np.ascontiguousarray(np.stack([np.stack([synth.synthetic_pair(h, w, ch, seed=2)[0]] * 2)] * n))
    ctx.upload_frames_u8(0, n, frames, w, h)
    ctx.run(n)
    for _ in range(3):  # warm-up of every call timed below
        ctx.set_initflow_fullres(0, n, host.data_ptr(), w, h)
        ctx.set_initflow_from_result(0, n, 0, w, h)
    res = dict(pairs=n, size="%dx%d" % (w, h), sc_f=prm.sc_f, block=2 << prm.sc_f,
               host_ms=timed(st, lambda: ctx.set_initflow_fullres(0, n, host.data_ptr(), w, h), reps),
               device_ms=timed(st, lambda: ctx.set_initflow_fullres(0, n, dev.data_ptr(), w, h, memkind=api.MEM_DEVICE),
                               reps),
               from_result_ms=timed(st, lambda: ctx.set_initflow_from_result(0, n, 0, w, h), reps),
               flow_mb=round(flows.nbytes / 1e6, 2))
    ctx.close()
    return res


def clip(pairs, reps):
    h, w = 436, 1024
    prm = params.operating_point(2, w, noc=1)
    st = torch.cuda.Stream()
    frames = synth.synthetic_sequence(pairs + 1, h, w, 1, seed=3, amp=6.0)
    pair_frames = [torch.from_numpy(np.ascontiguousarray(frames[t:t + 2])).pin_memory() for t in range(pairs)]
    ctx = context(prm, h, w, 1, st.cuda_stream)
    ctx.set_graph_mode(True)
    out = torch.empty((pairs, h, w, 2), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    per = h * w * 2

    def run(warm):
        for t in range(pairs):
            ctx.upload_frames_u8(0, 1, pair_frames[t].data_ptr(), w, h)
            if warm and t > 0:
                ctx.set_initflow_from_result(0, 1, 0, w, h)
            ctx.run(1, use_initflow=warm and t > 0)
            ctx.get_flow_fullres(0, 1, out.data_ptr() + 4 * per * t, w, h, memkind=api.MEM_DEVICE)

    for warm in (False, True):  # capture both graphs
        run(warm)
    times = {False: [], True: []}
    flows = {}
    for _ in range(reps):
        for warm in (False, True):
            times[warm].append(timed(st, lambda: run(warm), 1))
            ctx.sync()
            flows[warm] = out.cpu().numpy()
    u, v = synth.synthetic_flow(h, w, 6.0)
    gt = np.stack([u, v], -1)
    epe = {k: round(float(np.sqrt(((f - gt[None]) ** 2).sum(-1)).mean()), 6) for k, f in flows.items()}
    changed = float((flows[True] != flows[False]).any(-1).mean())  # share of pixels the warm start changes
    ctx.close()
    return dict(pairs=pairs, size="%dx%d" % (w, h), cold_ms_per_pair=round(statistics.median(times[False]) / pairs, 4),
                warm_ms_per_pair=round(statistics.median(times[True]) / pairs, 4), epe_cold=epe[False],
                epe_warm=epe[True], pixels_changed=round(changed, 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--pairs", type=int, default=32)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        print("no CUDA device", file=sys.stderr)
        sys.exit(2)
    res = dict(card=card())
    for name, c in CASES.items():
        res[name] = preparation(name, c, a.reps)
    res["clip"] = clip(a.pairs, max(3, a.reps // 4))
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
