"""Pair upload against sequence upload of consecutive frames, on one GPU.

    python tools/sequence_e2e.py [--rounds R] [--reps K]

A clip of n+1 frames gives n flows (t -> t+1).  ofdis_upload_frames_u8 takes the n pairs, so every interior frame
crosses PCIe twice and its pyramid is built twice; ofdis_upload_sequence_u8 takes the n+1 frames once.  Two cases:
64 pairs of 1024x436 gray at operating point 2 (bench.py's `cli` workload) and 8 pairs of 1920x1080 RGB with the
20 numbers of BASELINE configs[2].  For each, the flows of the two uploads are first checked to be bitwise equal
(exit 1 otherwise); then, alternating the two uploads and repeating:
  upload   upload + pyramid alone, from pinned host memory (CUDA events)
  cli      the whole step: upload -> graph run -> ofdis_get_flow_fullres into pinned memory, on one stream and on
           LANES overlapping streams (host clock around steps that end in a device synchronise)
  batch    wall time of run_OF_INT_batch on a 65-frame PNG chain list against the same pairs written as separate
           files (first case only; the output files of the two lists are checked to be byte-identical)
Prints one JSON line with the card name, power limit and SM clock, read in the same run.  Temporary files go to a
temporary directory; nothing is written to the tree."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from of_dis_b200 import api, build, params, synth  # noqa: E402

LANES = 4
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


def med(xs):
    return round(statistics.median(xs), 4)


def measure_case(name, c, rounds, reps):
    n, (h, w), ch = c["n"], c["size"], c["ch"]
    prm = c["prm"]()
    scf = 1 << prm.sc_f
    W, H = (w + scf - 1) // scf * scf, (h + scf - 1) // scf * scf
    frames = synth.synthetic_sequence(n + 1, h, w, ch, seed=5)
    seq = torch.from_numpy(frames).pin_memory()
    pairs = torch.from_numpy(np.ascontiguousarray(np.stack([frames[:-1], frames[1:]], axis=1))).pin_memory()
    lanes = []
    for _ in range(LANES):
        st = torch.cuda.Stream()
        ctx = api.Context(prm, W, H, prm.p_samp_s, n, stream=st.cuda_stream)
        ctx.set_graph_mode(True)
        lanes.append((st, ctx, torch.empty((n, h, w, prm.nop), dtype=torch.float32).pin_memory()))

    def upload(ctx, mode):
        if mode == "seq":
            ctx.upload_sequence_u8(0, n, seq.data_ptr(), w, h)
        else:
            ctx.upload_frames_u8(0, n, pairs.data_ptr(), w, h)

    def step(lane, mode):
        _, ctx, out = lanes[lane]
        upload(ctx, mode)
        ctx.run(n)
        ctx.get_flow_fullres(0, n, out.data_ptr(), w, h)

    # bitwise check first: the flows of the two uploads, on two lanes
    step(0, "pair")
    step(1, "seq")
    torch.cuda.synchronize()
    same = bool(torch.equal(lanes[0][2].view(torch.int32), lanes[1][2].view(torch.int32)))
    if not same:
        return {"result_checked_bitwise": False}

    st0, ctx0, _ = lanes[0]

    def time_upload(mode):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(st0)
        for _ in range(reps):
            upload(ctx0, mode)
        b.record(st0)
        b.synchronize()
        return a.elapsed_time(b) / reps

    def time_cli(mode, nl):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(reps * nl):
            step(i % nl, mode)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / (reps * nl)

    for mode in ("pair", "seq"):  # warm-up: graphs captured, PCIe link awake
        for i in range(2 * LANES):
            step(i % LANES, mode)
        time_upload(mode)
    torch.cuda.synchronize()
    res = {k: {"pair": [], "seq": []} for k in ("upload", "cli_1_stream", "cli_%d_streams" % LANES)}
    for _ in range(rounds):
        for mode in ("pair", "seq"):
            res["upload"][mode].append(time_upload(mode))
            res["cli_1_stream"][mode].append(time_cli(mode, 1))
            res["cli_%d_streams" % LANES][mode].append(time_cli(mode, LANES))
    out = {"pairs": n, "size": [w, h], "channels": ch, "result_checked_bitwise": same,
           "h2d_bytes": {"pair": pairs.numel(), "seq": seq.numel()}}
    for k, v in res.items():
        out[k + "_ms"] = {m: med(x) for m, x in v.items()}
        out[k + "_ms"]["spread_ms"] = {m: round(max(x) - min(x), 4) for m, x in v.items()}
    for _, ctx, _ in lanes:
        ctx.close()
    return out


def write_png(path, img):
    import struct
    import zlib

    h, w = img.shape[:2]
    raw = b"".join(b"\0" + row.tobytes() for row in np.ascontiguousarray(img).reshape(h, -1))

    def chunk(t, d):
        return struct.pack(">I", len(d)) + t + d + struct.pack(">I", zlib.crc32(t + d) & 0xFFFFFFFF)

    with open(path, "wb") as f:
        f.write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 0, 0, 0, 0)))
        f.write(chunk(b"IDAT", zlib.compress(raw, 1)) + chunk(b"IEND", b""))


def measure_batch(rounds):
    """run_OF_INT_batch, 64 pairs of 1024x436 gray at operating point 2: a 65-frame chain against 128 files."""
    exe = os.path.join(build.build_host(), "run_OF_INT_batch")
    frames = synth.synthetic_sequence(65, 436, 1024, 1, seed=5)
    with tempfile.TemporaryDirectory() as d:
        chain, split = [], []
        for t, img in enumerate(frames):
            write_png(os.path.join(d, "f%d.png" % t), img)
        for t in range(64):
            chain.append("%s %s %s" % (os.path.join(d, "f%d.png" % t), os.path.join(d, "f%d.png" % (t + 1)),
                                       os.path.join(d, "c%d.flo" % t)))
            for k in (0, 1):
                write_png(os.path.join(d, "p%d_%d.png" % (t, k)), frames[t + k])
            split.append("%s %s %s" % (os.path.join(d, "p%d_0.png" % t), os.path.join(d, "p%d_1.png" % t),
                                       os.path.join(d, "s%d.flo" % t)))
        lists = {}
        for name, lines in (("chain", chain), ("pairs", split)):
            lists[name] = os.path.join(d, name + ".txt")
            with open(lists[name], "w") as f:
                f.write("\n".join(lines) + "\n")
        wall = {"chain": [], "pairs": []}
        stdout = {}
        for r in range(rounds + 1):  # round 0: warm-up
            for name in ("pairs", "chain"):
                t0 = time.perf_counter()
                p = subprocess.run([exe, lists[name], "2"], capture_output=True, text=True)
                dt = (time.perf_counter() - t0) * 1e3
                if p.returncode:
                    raise RuntimeError(p.stdout + p.stderr)
                stdout[name] = p.stdout.strip().splitlines()
                if r:
                    wall[name].append(dt)
        same = all(open(os.path.join(d, "c%d.flo" % t), "rb").read() == open(os.path.join(d, "s%d.flo" % t), "rb").read()
                   for t in range(64))
    return {"wall_ms": {k: med(v) for k, v in wall.items()}, "spread_ms": {k: round(max(v) - min(v), 1) for k, v in wall.items()},
            "outputs_byte_identical": same, "stdout_chain": stdout["chain"], "stdout_pairs": stdout["pairs"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("sequence_e2e: no CUDA device")
    api.lib()
    info = card()
    res = {"card": info.get("name"), "power_limit": info.get("power.limit"), "sm_clock_mhz": info.get("clocks.sm"),
           "sm_clock_max_mhz": info.get("clocks.max.sm"), "rounds": args.rounds, "reps": args.reps}
    ok = True
    for name, c in CASES.items():
        res[name] = measure_case(name, c, args.rounds, args.reps)
        ok = ok and res[name]["result_checked_bitwise"]
    if ok:
        res["batch_64x1024x436"] = measure_batch(args.rounds)
        ok = res["batch_64x1024x436"]["outputs_byte_identical"]
    res["sm_clock_mhz_after"] = card().get("clocks.sm")
    print(json.dumps(res))
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
