"""Color-coded full-resolution flows against the float32 flow, end to end on one GPU.

    python tools/color_e2e.py [--rounds R] [--reps K]

The workload: 64 gray 1024x436 pairs at operating point 2 (bench.py's `cli` workload) from pinned 8-bit frames, one
upload per frame (ofdis_upload_sequence_u8), as tools/encode_e2e.py runs it.  The color images of
ofdis_flow_color_fullres are first checked bitwise against preprocess.flow_to_color of the float32 flow of
ofdis_get_flow_fullres, with the automatic and a fixed scale (exit 1 otherwise).  Then, alternating the outputs round
by round:
  color_device   the color call alone into device memory (CUDA events), automatic and fixed scale
  color_host     the color call into pinned host memory, copy included (CUDA events), automatic and fixed scale
  f32_host       ofdis_get_flow_fullres into pinned host memory, copy included (CUDA events)
  step           upload -> graph run -> the output in pinned host memory, on one stream and on LANES overlapping
                 streams (host clock around steps that end in a device synchronise)
and the bytes each output copies device-to-host per step.  Prints one JSON line with the card name, power limit and
SM clock, read in the same run.  Nothing is written to the tree."""
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

LANES = 4
N, H, W = 64, 436, 1024
FIXED = 8.0  # the fixed scale, px
OUTPUTS = ("f32", "color_auto", "color_fixed")


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))
    except (OSError, subprocess.SubprocessError):
        return {"name": torch.cuda.get_device_name(0), "power.limit": None, "clocks.sm": None, "clocks.max.sm": None}


def med(xs):
    return round(statistics.median(xs), 4)


def out_tensor(kind, nop, device):
    shape, dt = ((N, H, W, nop), torch.float32) if kind == "f32" else ((N, H, W, 3), torch.uint8)
    t = torch.empty(shape, dtype=dt, device=device)
    return t.pin_memory() if device == "cpu" else t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("color_e2e: no CUDA device")
    api.lib()
    info = card()
    prm = params.operating_point(2, W, noc=1)
    nop = prm.nop
    scf = 1 << prm.sc_f
    CW, CH = (W + scf - 1) // scf * scf, (H + scf - 1) // scf * scf
    seq = torch.from_numpy(synth.synthetic_sequence(N + 1, H, W, 1, seed=5)).pin_memory()
    lanes = []
    for _ in range(LANES):
        st = torch.cuda.Stream()
        ctx = api.Context(prm, CW, CH, prm.p_samp_s, N, stream=st.cuda_stream)
        ctx.set_graph_mode(True)
        lanes.append((st, ctx, {k: out_tensor(k, nop, "cpu") for k in OUTPUTS}))

    def fetch(ctx, kind, ptr, memkind):
        """The C-ABI calls, enqueued without a synchronise (Context.flow_color_fullres synchronises after a host
        copy), so that host and device results alike leave the stream free, as get_flow_fullres does."""
        if kind == "f32":
            ctx.get_flow_fullres(0, N, ptr, W, H, memkind)
        else:
            mv = 0.0 if kind == "color_auto" else FIXED
            ctx._ck(api.lib().ofdis_flow_color_fullres(ctx._h, 0, N, api._ptr(ptr), None, mv, W, H, memkind))

    def step(lane, kind):
        _, ctx, outs = lanes[lane]
        ctx.upload_sequence_u8(0, N, seq.data_ptr(), W, H)
        ctx.run(N)
        fetch(ctx, kind, outs[kind].data_ptr(), api.MEM_HOST)

    # bitwise checks first, on lane 0
    st0, ctx0, outs0 = lanes[0]
    for kind in OUTPUTS:
        step(0, kind)
    torch.cuda.synchronize()
    f32 = outs0["f32"].numpy()
    checks = {"color_auto": bool(np.array_equal(outs0["color_auto"].numpy(), preprocess.flow_to_color(f32)[0])),
              "color_fixed": bool(np.array_equal(outs0["color_fixed"].numpy(),
                                                 preprocess.flow_to_color(f32, FIXED)[0]))}
    dev = {k: out_tensor(k, nop, "cuda") for k in OUTPUTS}
    res = {"card": info.get("name"), "power_limit": info.get("power.limit"), "sm_clock_mhz": info.get("clocks.sm"),
           "sm_clock_max_mhz": info.get("clocks.max.sm"), "pairs": N, "size": [W, H], "channels": 1,
           "oppoint": 2, "fixed_scale": FIXED, "rounds": args.rounds, "reps": args.reps, "checked_bitwise": checks,
           "d2h_bytes": {k: outs0[k].numel() * outs0[k].element_size() for k in OUTPUTS}}
    if not all(checks.values()):
        print(json.dumps(res))
        sys.exit(1)

    def time_fetch(kind, memkind):
        dst = dev[kind] if memkind == api.MEM_DEVICE else outs0[kind]
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(st0)
        for _ in range(reps):
            fetch(ctx0, kind, dst.data_ptr(), memkind)
        b.record(st0)
        b.synchronize()
        return a.elapsed_time(b) / reps

    def time_step(kind, nl):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(reps * nl):
            step(i % nl, kind)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / (reps * nl)

    reps = args.reps
    for kind in OUTPUTS:  # warm-up: graphs captured on every lane, PCIe link awake
        for i in range(2 * LANES):
            step(i % LANES, kind)
        time_fetch(kind, api.MEM_DEVICE)
        time_fetch(kind, api.MEM_HOST)
    torch.cuda.synchronize()
    keys = ("fetch_device", "fetch_pinned_host", "step_1_stream", "step_%d_streams" % LANES)
    t = {k: {m: [] for m in OUTPUTS} for k in keys}
    for _ in range(args.rounds):
        for kind in OUTPUTS:
            t["fetch_device"][kind].append(time_fetch(kind, api.MEM_DEVICE))
            t["fetch_pinned_host"][kind].append(time_fetch(kind, api.MEM_HOST))
            t["step_1_stream"][kind].append(time_step(kind, 1))
            t["step_%d_streams" % LANES][kind].append(time_step(kind, LANES))
    for k, v in t.items():
        res[k + "_ms"] = {m: med(x) for m, x in v.items()}
        res[k + "_ms"]["spread_ms"] = {m: round(max(x) - min(x), 4) for m, x in v.items()}
    for _, ctx, _ in lanes:
        ctx.close()
    res["sm_clock_mhz_after"] = card().get("clocks.sm")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
