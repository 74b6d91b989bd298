"""Fisher vectors on the device (ofdis_fisher_begin / push / take), measured: one JSON line.

    python tools/fisher_e2e.py [--pairs 64] [--reps 10] [--fit-samples 256000]

The descriptors of tools/traj_e2e.py's two workloads (operating point 2, 64 pairs with the two-way upload, the batch
command's tracker settings and the IDT defaults: 1024x436 gray synth.global_motion_clip with its camera models, and
1920x1080 RGB synth.synthetic_sequence without models) stay in device memory and are encoded with IDT's blocks
(dim_in / 2) at K = 256:
  * the device-event time of one push of all of a clip's descriptors plus the take, median of `reps` after warm-up;
  * the per-kernel device times of one push and take from torch.profiler, in a separate, profiled call;
  * the algorithmic fp32 and fp64 operations and the bytes each kernel must move, from the shapes, and each kernel's
    share of the larger of its compute bound and byte bound (data-sheet rates of the H100 SXM: 3.35 TB/s, and half of
    67 TFLOP/s fp32 and of 34 TFLOP/s fp64 for operations that are not fused multiply-adds);
  * one EM iteration of Context.fisher_fit at `fit-samples` samples and K = 256: the device E-step (begin, a host push
    of the samples, take) and the host M-step, timed with a host clock around calls that end in a synchronise.
The codebook is random: the encoder's work does not depend on its values.  The card's name and power limit are read
in the same run."""
import argparse
import json
import math
import os
import re
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from of_dis_b200 import api, params, preprocess as pp, synth

K = 256
FP32_OPS, FP64_OPS, HBM = 33.5e12, 17e12, 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def codebook(rng):
    blocks = [(o, di, di // 2) for o, di in pp.fisher_blocks(pp.TRAJ_DEFAULTS)]
    cb = {"K": K, "desc_dim": pp.traj_dim(pp.TRAJ_DEFAULTS), "blocks": blocks}
    for k in pp.FISHER_PARTS:
        cb[k] = []
    for _, di, d in blocks:
        sig = rng.uniform(0.05, 0.2, (K, d))
        cb["mean"].append(rng.uniform(0, 0.1, di).astype(np.float32))
        cb["proj"].append(rng.normal(0, 1.0 / math.sqrt(di), (d, di)).astype(np.float32))
        cb["mu"].append(rng.normal(0, 0.1, (K, d)).astype(np.float32))
        cb["isig"].append((1.0 / sig).astype(np.float32))
        cb["c"].append((math.log(1.0 / K) - np.log(sig).sum(1)).astype(np.float32))
        cb["w"].append(np.full(K, 1.0 / K, np.float32))
    return cb


def model(n, blocks, desc_dim):
    """Algorithmic operations and bytes per kernel for n descriptors (chunks of 4096)."""
    din = sum(b[1] for b in blocks)
    P = sum(b[2] for b in blocks)
    nb = len(blocks)
    proj_f32 = 2 * n * sum(b[1] * b[2] for b in blocks)  # a multiply and an add per (descriptor, d, i)
    post_f32 = n * (4 * K * P + 2 * K * nb + 21 * K * nb)  # z, z^2, q; ll; exp_f32 (17 ops), subtract, sum, divide
    stats_f32 = 2 * n * K * P  # z
    stats_f64 = 5 * n * K * P  # g*z, add, z*z, g*z^2, add
    chunks = (n + 4095) // 4096
    return {
        "project": {"f32": proj_f32, "f64": 0, "bytes": n * 4 * (din + P)},
        "post": {"f32": post_f32, "f64": 0, "bytes": n * 4 * (P + K * nb) + n * nb},
        "stats": {"f32": stats_f32, "f64": stats_f64,
                  "bytes": n * 4 * K * nb + n * 4 * sum(b[2] * math.ceil(K * b[2] / 256) for b in blocks)
                  + chunks * 8 * 2 * 2 * K * P},
    }


def share(m, ms):
    bound = max(m["f32"] / FP32_OPS + m["f64"] / FP64_OPS, m["bytes"] / HBM)
    kind = "bytes" if m["bytes"] / HBM >= m["f32"] / FP32_OPS + m["f64"] / FP64_OPS else "compute"
    return {"bound_ms": round(bound * 1e3, 4), "bound_by": kind, "share": round(bound * 1e3 / ms, 3) if ms else None}


def descriptors(h, w, ch, n, camera):
    prm = params.operating_point(2, w, noc=ch)
    if camera:
        H = synth.similarity_about_centre(h, w, 0.2, 1.002, (1.5, 0.5))
        clip, models, _ = synth.global_motion_clip(n, h, w, ch, seed=5, H=H)
        M = models.reshape(n, 9)
    else:
        clip, M = synth.synthetic_sequence(n + 1, h, w, ch, seed=5, amp=3.0), None
    scf = 1 << prm.sc_f
    ctx = api.Context(prm, (w + scf - 1) // scf * scf, (h + scf - 1) // scf * scf, prm.p_samp_s, 2 * n)
    ctx.upload_sequence_bidir_u8(0, n, clip, w, h)
    ctx.run(2 * n)
    cells = ((w + 7) // 8) * ((h + 7) // 8)
    tp = dict(capacity=4 * cells, spacing=8, alpha=0.01, beta=0.5, mb_alpha=0.01, mb_beta=0.002, min_eig=25.0)
    p = pp.TRAJ_DEFAULTS
    hwc = h * w * ch
    cap, bound, dim = tp["capacity"], pp.traj_bound(tp["capacity"], n, p["L"]), pp.traj_dim(p)
    dev = torch.from_numpy(clip.reshape(-1)).cuda()
    pts = torch.empty((n * cap * 3,), dtype=torch.int32, device="cuda")
    rec = torch.empty((bound * 7,), dtype=torch.int32, device="cuda")
    desc = torch.empty((bound * dim,), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    ctx.traj_begin(tp, p, dev.data_ptr(), w, h, memkind=api.MEM_DEVICE, points=pts.data_ptr())
    _, nd = ctx.traj_advance(0, n, n, dev.data_ptr() + hwc, w, h, models=M, memkind=api.MEM_DEVICE,
                             points=pts.data_ptr(), records=rec.data_ptr(), desc=desc.data_ptr())
    ctx.close()
    total = int(nd.sum())
    return desc[:total * dim].view(total, dim).clone()


def measure(ctx, stream, cb, desc, reps):
    n = desc.shape[0]
    sz = pp.fisher_sizes(K, cb["blocks"])
    fv = torch.empty((sz["fv"],), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    ctx.fisher_begin(cb)

    def encode():
        ctx.fisher_push(desc.data_ptr(), memkind=api.MEM_DEVICE, n=n)
        ctx.fisher_take(memkind=api.MEM_DEVICE, fv=fv.data_ptr())

    encode()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        encode()
        b.record(stream)
        b.synchronize()
        times.append(a.elapsed_time(b))
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        encode()
        torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
        if e.device_type.name == "CUDA":
            m = re.search(r"(fisher_\w+_kernel)", e.name)
            if m:
                kern[m.group(1)] = kern.get(m.group(1), 0.0) + e.device_time / 1000.0
    mod = model(n, cb["blocks"], cb["desc_dim"])
    shares = {k: share(mod[k], kern.get("fisher_%s_kernel" % k)) for k in mod}
    ops = {k: {"f32_G": round(v["f32"] / 1e9, 2), "f64_G": round(v["f64"] / 1e9, 2), "MB": round(v["bytes"] / 1e6, 1)}
           for k, v in mod.items()}
    return {"descriptors": n, "push_take_ms": round(float(np.median(times)), 3),
            "kernel_ms_profiled_call": {k: round(v, 4) for k, v in sorted(kern.items(), key=lambda kv: -kv[1])},
            "algorithmic": ops, "share_of_bound": shares}


def fit_iteration(ctx, cb, samples):
    x = np.ascontiguousarray(samples, np.float32)
    eigs = [np.ones(b[2]) for b in cb["blocks"]]
    ctx.fisher_begin(cb)
    ctx.fisher_push(x[:4096])
    ctx.fisher_take()
    t0 = time.perf_counter()
    ctx.fisher_begin(cb)
    ctx.fisher_push(x)
    stats = ctx.fisher_take(with_fv=False)[1]
    t1 = time.perf_counter()
    pp.fisher_mstep(cb, stats, eigs, 1e-3)
    t2 = time.perf_counter()
    return {"samples": int(x.shape[0]), "estep_ms": round((t1 - t0) * 1e3, 1), "mstep_ms": round((t2 - t1) * 1e3, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=64)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--fit-samples", type=int, default=256000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("fisher_e2e: no CUDA device")
    rng = np.random.default_rng(0)
    cb = codebook(rng)
    res = {"card": card(), "K": K, "pairs": a.pairs, "memory": "device"}
    stream = torch.cuda.Stream()
    prm = params.from_cli_numbers("3 1 8 8 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0".split(), noc=1, nop=2)
    ctx = api.Context(prm, 64, 64, prm.p_samp_s, 1, stream=stream.cuda_stream)  # the encoder reads no flow
    big = None
    for name, (h, w, ch, cam) in (("1024x436_gray_camera_models", (436, 1024, 1, True)),
                                  ("1920x1080_rgb_no_models", (1080, 1920, 3, False))):
        desc = descriptors(h, w, ch, a.pairs, cam)
        res[name] = measure(ctx, stream, cb, desc, a.reps)
        big = desc
    host = big.cpu().numpy()
    reps = -(-a.fit_samples // host.shape[0])
    samples = np.concatenate([host] * reps)[:a.fit_samples]
    res["fit_iteration"] = fit_iteration(ctx, cb, samples)
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
