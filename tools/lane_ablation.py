"""Where does a step of sor_lane_kernel go?  Timing-only builds (OFDIS_EXP_LANE; variants 2..6 compute WRONG
results) and a cycle-stamped build (OFDIS_SOR_TIMING) of the product kernel.
  python tools/lane_ablation.py --build     # here: nvcc, variants into of_dis_b200/lib/exp/
  python tools/lane_ablation.py             # on the GPU: one JSON line per variant + the chunk timeline of level 3
Variants: 0 product | 1 publish without MEMBAR | 2 no record prefetch | 3 no waits | 4 = 2+3 | 5 = 1+2+3 | 6 prefetch
never waited for."""
import ctypes, json, os, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
EXP = os.path.join(ROOT, "of_dis_b200", "lib", "exp")
VARIANTS = {0: "product", 1: "publish without MEMBAR", 2: "no record prefetch", 3: "no waits", 4: "2+3", 5: "1+2+3", 6: "prefetch never waited for"}


def build():
    from of_dis_b200 import build as B
    os.makedirs(EXP, exist_ok=True)
    procs = []
    for v in ONLY or (list(VARIANTS) + ["t"]):
        out = os.path.join(EXP, "libofdis_lane%s.so" % v)
        defs = ["-DOFDIS_SOR_TIMING"] if v == "t" else (["-DOFDIS_EXP_UNROLL=%s" % v[1:]] if str(v).startswith("u") else (["-DOFDIS_EXP_SLP=%s" % v[1:]] if str(v).startswith("p") else ["-DOFDIS_EXP_LANE=%s" % v]))
        cmd = [B._nvcc()] + B.NVCC_FLAGS + defs + [os.path.join(B.CSRC, s) for s in B.SOURCES] + ["-ldl", "-o", out]
        procs.append((v, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for v, p in procs:
        o, _ = p.communicate()
        print(v, "rc", p.returncode, o[-300:] if p.returncode else "")


def child(timeline):
    import numpy as np
    from of_dis_b200 import api, params, synth
    prm = params.operating_point(2, 1024)
    h, w = 436, 1024
    i0, i1, _ = synth.synthetic_pair(h, w, 1, seed=1)
    scf = 1 << prm.sc_f
    W, H = (w + scf - 1) // scf * scf, (h + scf - 1) // scf * scf
    out = {}
    for B in (1, 64):
        ctx = api.Context(prm, W, H, prm.p_samp_s, B)
        frames = np.ascontiguousarray(np.stack([np.stack([i0, i1])] * B))
        ctx.upload_frames_u8(0, B, frames, w, h)
        ctx.run(B)
        lev = ctx.profile_levels(B, steps=5)
        row = {}
        for lv in sorted(lev):
            g = ctx.level_info(lv)
            n_inner = prm.tv_innerit * (lv + 1)
            row[str(lv)] = {"sor_us_per_launch": round(lev[lv]["sor"] * 1e3 / n_inner, 2),
                            "cycles_per_column": round(lev[lv]["sor"] * 1e-3 / n_inner * 1.965e9 / (g["w"] + g["h"] + 6))}
        out["x%d" % B] = row
        if timeline and B == 1:
            ctx.sync()
            buf = np.zeros(64 * 8 * 16, np.int64)
            assert api.lib().ofdis_debug_sor_times(buf.ctypes.data_as(ctypes.c_void_p)) == 0
            t = buf[:16 * 32 * 4].reshape(16, 32, 4)
            t0 = t[0, 0, 0]
            tl = {}
            for wi in range(6):  # level 3 ran last: 2 bands x 3 sweeps, 20 chunks
                tl["warp%d(b=%d,k=%d)" % (wi, wi % 2, wi // 2)] = [[int(x - t0) for x in t[wi, c]] for c in range(20)]
            out["timeline_cycles[start,published,waited,end]"] = tl
        ctx.close()
    print(json.dumps(out))


ONLY = [a for a in sys.argv[1:] if not a.startswith("--")]  # e.g. 0 5 u1 u2 u4 p2 p8 (uN: product with the step loop unrolled N times; pN: progress published every N steps)

if __name__ == "__main__":
    if "--build" in sys.argv:
        build()
    elif "--child" in sys.argv:
        child("--timeline" in sys.argv)
    else:
        for v in ONLY or (list(VARIANTS) + ["t"]):
            lib = os.path.join(EXP, "libofdis_lane%s.so" % v)
            env = dict(os.environ, OFDIS_LIB=lib)
            args = [sys.executable, os.path.abspath(__file__), "--child"] + (["--timeline"] if v == "t" else [])
            r = subprocess.run(args, env=env, capture_output=True, text=True, timeout=600)
            print(json.dumps({"variant": v, "what": VARIANTS.get(v if not str(v).isdigit() else int(v), "product + cycle stamps" if v == "t" else "unroll")}), r.stdout.strip().splitlines()[-1] if r.returncode == 0 and r.stdout.strip() else ("FAILED " + r.stderr[-600:]), flush=True)
