"""Where does a SOR super-step go?  Timing-only ablation builds of sor_wave_kernel (OFDIS_EXP_ABL, results are
WRONG by construction) against the product build, per level, single pair and a batch.
  python tools/sor_ablation.py --build          # here: nvcc, variants into of_dis_b200/lib/exp/
  python tools/sor_ablation.py                  # on the GPU: one JSON line per variant
Variants: 0 product | 1 no arithmetic | 2 no record loads | 3 no operand (board) loads | 7 = 1+2+3 (stores + barrier
only) | 4 empty compute body | 5 producer does not wait for its copies | 6 producer issues no copies at all."""
import json, os, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
EXP = os.path.join(ROOT, "of_dis_b200", "lib", "exp")
VARIANTS = {0: "product", 1: "no arithmetic", 2: "no record loads", 3: "no operand loads", 7: "stores+barrier only",
            4: "empty compute body", 5: "producer never waits", 6: "no bulk copies"}


def build():
    from of_dis_b200 import build as B
    os.makedirs(EXP, exist_ok=True)
    procs = []
    for v in VARIANTS:
        out = os.path.join(EXP, "libofdis_abl%d.so" % v)
        cmd = [B._nvcc()] + B.NVCC_FLAGS + ["-DOFDIS_EXP_ABL=%d" % v] + [os.path.join(B.CSRC, s) for s in B.SOURCES] + ["-ldl", "-o", out]
        procs.append((v, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for v, p in procs:
        o, _ = p.communicate()
        print(v, "rc", p.returncode, o[-300:] if p.returncode else "")


def child():
    import numpy as np
    import torch
    from of_dis_b200 import api, params, preprocess, synth
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import big_configs
    out = {}
    for name, (h, w, prmf, ch, nop) in {
        "bench": (436, 1024, lambda: params.operating_point(2, 1024), 1, 2),
        "cfg3": (1080, 1920, big_configs.CFGS["cfg3_1920x1080_rgb_l1"]["prm"], 3, 2),
        "cfg5": (1988, 2880, big_configs.CFGS["cfg5_2880x1988_stereo_op4"]["prm"], 1, 1),
    }.items():
        prm = prmf()
        i0, i1, _ = synth.synthetic_pair(h, w, ch, seed=1, stereo=(nop == 1))
        scf = 1 << prm.sc_f
        W, H = (w + scf - 1) // scf * scf, (h + scf - 1) // scf * scf
        for B in ((1, 64) if name == "bench" else (1,)):
            ctx = api.Context(prm, W, H, prm.p_samp_s, B)
            frames = np.ascontiguousarray(np.stack([np.stack([i0, i1])] * B))
            ctx.upload_frames_u8(0, B, frames, w, h)
            ctx.run(B)
            lev = ctx.profile_levels(B, steps=5)
            row = {}
            for lv in sorted(lev):
                g = ctx.level_info(lv)
                n_inner = prm.tv_innerit * (lv + 1)
                steps = n_inner * ((g["w"] + 3) // 4 + g["h"] + 2 * prm.tv_solverit - 2 + 4)
                row[str(lv)] = {"sor_ms": round(lev[lv]["sor"], 4), "cycles_per_superstep": round(lev[lv]["sor"] * 1e-3 * 1.965e9 / steps)}
            out["%s_x%d" % (name, B)] = row
            ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    if "--build" in sys.argv:
        build()
    elif "--child" in sys.argv:
        child()
    elif "--libs" in sys.argv:  # python tools/sor_ablation.py --libs a.so b.so ...
        for lib in sys.argv[sys.argv.index("--libs") + 1:]:
            env = dict(os.environ, OFDIS_LIB=os.path.abspath(lib))
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child"], env=env, capture_output=True, text=True, timeout=900)
            print(lib, r.stdout.strip().splitlines()[-1] if r.returncode == 0 and r.stdout.strip() else ("FAILED " + r.stderr[-400:]), flush=True)
    else:
        for v, what in VARIANTS.items():
            lib = os.path.join(EXP, "libofdis_abl%d.so" % v)
            env = dict(os.environ, OFDIS_LIB=lib)
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child"], env=env, capture_output=True, text=True, timeout=600)
            line = r.stdout.strip().splitlines()[-1] if r.returncode == 0 and r.stdout.strip() else ("FAILED " + r.stderr[-400:])
            print(json.dumps({"variant": v, "what": what}), line, flush=True)
