"""Full-resolution flow as float32, binary16 and KITTI 16-bit, end to end on one GPU.

    python tools/encode_e2e.py [--rounds R] [--reps K]

The workload: 64 gray 1024x436 pairs at operating point 2 (bench.py's `cli` workload) from pinned 8-bit frames, one
upload per frame (ofdis_upload_sequence_u8).  Each output is first checked bitwise: the float32 flow of
ofdis_get_flow_fullres against the restatement of the level flows (preprocess.postprocess), the encodings of
ofdis_get_flow_fullres_encoded against preprocess.encode_f16 / encode_kitti of that flow (exit 1 otherwise).  Then,
alternating the three outputs and repeating:
  step     upload -> graph run -> the full-resolution result in pinned host memory, on one stream and on LANES
           overlapping streams (host clock around steps that end in a device synchronise)
  fetch    the output call alone into a device buffer (CUDA events): flow_upsample_kernel for float32,
           flow_encode_kernel for the encodings
  copy     the device-to-host copy of each output's bytes alone, into pinned memory (CUDA events)
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
OUTPUTS = ("f32", "f16", "kitti")


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
    if kind == "f32":
        shape, dt = (N, H, W, nop), torch.float32
    elif kind == "f16":
        shape, dt = (N, H, W, nop), torch.float16
    else:
        shape, dt = (N, H, W) + ((3,) if nop == 2 else ()), torch.int16
    t = torch.empty(shape, dtype=dt, device=device)
    return t.pin_memory() if device == "cpu" else t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("encode_e2e: no CUDA device")
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
        """The C-ABI calls, enqueued without a synchronise (Context.get_flow_fullres_encoded synchronises after a
        host copy), so that host and device results alike leave the stream free, as get_flow_fullres does."""
        if kind == "f32":
            ctx.get_flow_fullres(0, N, ptr, W, H, memkind)
        else:
            ctx._ck(api.lib().ofdis_get_flow_fullres_encoded(ctx._h, 0, N, api.ENCODINGS[kind], ptr, W, H, memkind))

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
    pad_w, pad_h = CW - W, CH - H
    ref = np.stack([preprocess.postprocess(ctx0.get_flow(f, prm.sc_l), prm.sc_l, pad_w, pad_h, W, H)
                    for f in range(N)])
    f32 = outs0["f32"].numpy()
    checks = {"f32": bool(np.array_equal(f32.view(np.uint32), ref.view(np.uint32))),
              "f16": bool(np.array_equal(outs0["f16"].numpy().view(np.uint16),
                                         preprocess.encode_f16(f32).view(np.uint16))),
              "kitti": bool(np.array_equal(outs0["kitti"].numpy().view(np.uint16), preprocess.encode_kitti(f32)))}
    dev = {k: out_tensor(k, nop, "cuda") for k in OUTPUTS}
    res = {"card": info.get("name"), "power_limit": info.get("power.limit"), "sm_clock_mhz": info.get("clocks.sm"),
           "sm_clock_max_mhz": info.get("clocks.max.sm"), "pairs": N, "size": [W, H], "channels": 1,
           "oppoint": 2, "rounds": args.rounds, "reps": args.reps, "checked_bitwise": checks,
           "d2h_bytes": {k: outs0[k].numel() * outs0[k].element_size() for k in OUTPUTS}}
    if not all(checks.values()):
        print(json.dumps(res))
        sys.exit(1)

    def time_fetch(kind):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(st0)
        for _ in range(reps):
            fetch(ctx0, kind, dev[kind].data_ptr(), api.MEM_DEVICE)
        b.record(st0)
        b.synchronize()
        return a.elapsed_time(b) / reps

    def time_copy(kind):
        """The device-to-host copy of the output's bytes alone, device buffer to pinned memory."""
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(st0):
            a.record(st0)
            for _ in range(reps):
                outs0[kind].copy_(dev[kind], non_blocking=True)
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
        time_fetch(kind)
        time_copy(kind)
    torch.cuda.synchronize()
    keys = ("fetch_device", "copy_d2h", "step_1_stream", "step_%d_streams" % LANES)
    t = {k: {m: [] for m in OUTPUTS} for k in keys}
    for _ in range(args.rounds):
        for kind in OUTPUTS:
            t["fetch_device"][kind].append(time_fetch(kind))
            t["copy_d2h"][kind].append(time_copy(kind))
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
