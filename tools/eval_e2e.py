"""Evaluation against ground truth on one GPU: 64 gray 1024x436 pairs at operating point 2, run in both directions
(128 slots), evaluated against the clip's synthetic flow with the forward consistency mask as classes.

    python tools/eval_e2e.py [--reps K] [--warmup W]

First checks, exit 1 otherwise: ofdis_flow_error_fullres's stats and error map of the 64 forward slots are bitwise
preprocess.flow_error on the ofdis_get_flow_fullres output, with the device mask of ofdis_consistency_fullres as the
classes (nclasses 3).  Then times, after W warm-up calls, the median of K:
  (a) the evaluation from device ground truth and the device mask, stats only and with the error map (CUDA events);
  (b) the same from pinned host ground truth and a pinned host mask (CUDA events, the copies included);
  (c) today's way: ofdis_get_flow_fullres into pinned memory, then the same counts and sums in numpy (vectorised,
      numpy's own summation order) -- host clock around a step that starts with a device synchronise.
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


def numpy_stats(flows, gt, mask):
    """What an evaluation in numpy does today: per class the counts and the sum of the end-point errors."""
    f32 = np.float32
    lim = f32(preprocess.UNKNOWN_FLOW_THRESH)
    with np.errstate(invalid="ignore"):
        known = (np.abs(gt[..., 0]) <= lim) & (np.abs(gt[..., 1]) <= lim)
        d = flows - gt
        e = np.sqrt(d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1])
        g = np.sqrt(gt[..., 0] * gt[..., 0] + gt[..., 1] * gt[..., 1])
        out = (e > 3) & (e > f32(0.05) * g)
    res = []
    for c in range(3):
        m = known & (mask == c)
        res.append((int(m.sum()), [int((m & (e > t)).sum()) for t in (1, 3, 5)], int((m & out).sum()),
                    float(e[m].astype(np.float64).sum())))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    prm = params.operating_point(2, W, noc=1)
    scf = 1 << prm.sc_f
    Wp, Hp = (W + scf - 1) // scf * scf, (H + scf - 1) // scf * scf
    frames = synth.synthetic_sequence(N + 1, H, W, 1, seed=5)
    u, v = synth.synthetic_flow(H, W)
    gt_host = torch.from_numpy(np.ascontiguousarray(np.broadcast_to(np.stack([u, v], -1).astype(np.float32),
                                                                    (N, H, W, 2)))).pin_memory()
    gt_dev = gt_host.cuda()
    st = torch.cuda.Stream()
    ctx = api.Context(prm, Wp, Hp, prm.p_samp_s, 2 * N, stream=st.cuda_stream)
    ctx.set_graph_mode(True)
    ctx.upload_sequence_bidir_u8(0, N, torch.from_numpy(frames).pin_memory().data_ptr(), W, H)
    ctx.run(2 * N)
    flows = torch.empty((N, H, W, 2), dtype=torch.float32).pin_memory()
    dmask = torch.empty((N, H, W), dtype=torch.uint8, device="cuda")
    hmask = torch.empty((N, H, W), dtype=torch.uint8).pin_memory()
    derr = torch.empty((N, H, W), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    ctx.consistency_fullres(0, N, N, W, H, memkind=api.MEM_DEVICE, mask=dmask.data_ptr())
    ctx.sync()
    hmask.copy_(dmask)

    def dev(with_err):
        return ctx.flow_error_fullres(0, N, gt_dev.data_ptr(), W, H, classes=dmask.data_ptr(), nclasses=3,
                                      memkind=api.MEM_DEVICE, err=derr.data_ptr() if with_err else None)[0]

    def host():
        return ctx.flow_error_fullres(0, N, gt_host.numpy(), W, H, classes=hmask.numpy(), nclasses=3)[0]

    # ---- bitwise checks
    stats = dev(True)
    ctx.get_flow_fullres(0, N, flows.data_ptr(), W, H)
    ctx.sync()
    exp, exp_err = preprocess.flow_error(flows.numpy(), gt_host.numpy(), hmask.numpy(), 3)
    if stats.tobytes() != exp.tobytes() or host().tobytes() != exp.tobytes():
        print("FAIL: the device stats differ from preprocess.flow_error")
        return 1
    if not np.array_equal(derr.cpu().numpy().view(np.uint32), exp_err.view(np.uint32)):
        print("FAIL: the device error map differs from preprocess.flow_error")
        return 1
    n_c, sum_c = stats["n"].sum(axis=0), stats["sum_err"].sum(axis=0)  # per class
    n_all = int(n_c.sum())
    res = {"card": card(), "pairs": N, "size": [W, H], "checks": "bitwise ok",
           "epe_all": round(float(sum_c.sum()) / n_all, 6),
           "epe_consistent_inconsistent_leaves": [round(float(s) / max(int(n), 1), 6) for n, s in zip(n_c, sum_c)],
           "share_consistent_inconsistent_leaves": [round(int(n) / n_all, 4) for n in n_c]}

    # ---- (a), (b): the evaluation alone
    res["a_device_ms"] = {"stats": events(lambda: dev(False), a.reps, a.warmup, st),
                          "stats_and_map": events(lambda: dev(True), a.reps, a.warmup, st)}
    res["b_pinned_host_ms"] = {"stats": events(host, a.reps, a.warmup, st)}

    # ---- (c) today's way
    def today():
        ctx.get_flow_fullres(0, N, flows.data_ptr(), W, H)
        ctx.sync()
        return numpy_stats(flows.numpy(), gt_host.numpy(), hmask.numpy())

    ref = today()
    if [r[0] for r in ref] != [int(n) for n in n_c]:
        print("FAIL: numpy counts differ")
        return 1
    res["c_fullres_numpy_ms"] = wall(today, max(2, a.reps // 3), 1)
    ctx.close()
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
