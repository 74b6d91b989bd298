"""CPU pre-study of the per-pixel confidence, bit-exact to the device: the oracle port's stereo disparities of the
KITTI-sized synthetic clip (operating point 2, left view only, so without the forward-backward term) and of
synth.layered_stereo, ranked by preprocess.confidence and in a random order.  One JSON line: per scene the mean
|d - gt| and D1 (> 3 px) of the most confident x % of the known pixels, x = 100, 90, .., 30.

    python tools/confidence_prestudy.py [--pairs 4]"""
import argparse
import json
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from of_dis_b200 import params, preprocess, synth
from oracle import port_driver

FRACTIONS = (1.0, 0.9, 0.8, 0.7, 0.6, 0.5, 0.4, 0.3)
CP = dict(radius=2, s_fb=1.0, s_tex=100.0, min_count=5)


def disparity(left, right, prm):
    """The port's full-resolution stereo flow of one pair (the device's get_flow_fullres, bit for bit)."""
    pyr = preprocess.PairPyramids(left, right, prm.sc_f, prm.p_samp_s)
    h, w = left.shape[:2]
    lv = port_driver.port_run(pyr, prm)
    return preprocess.postprocess(lv, prm.sc_l, pyr.width - w, pyr.height - h, w, h)[..., 0]


def curves(errs, confs):
    err, conf = np.concatenate(errs), np.concatenate(confs)
    rng = np.random.default_rng(0)
    out = {}
    for name, order in (("conf", np.argsort(-conf, kind="stable")), ("random", rng.permutation(err.size))):
        e = err[order]
        sel = [e[:max(1, int(round(x * e.size)))] for x in FRACTIONS]
        out[name] = {"mean": [round(float(s.mean()), 4) for s in sel], "d1": [round(float((s > 3).mean()), 4) for s in sel]}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=4)
    a = ap.parse_args()
    figures = {}
    h, w = 120, 200
    left, right, gt, _ = synth.layered_stereo(h, w, 1, seed=7)
    prm = params.from_cli_numbers("3 1 8 8 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0".split(), noc=1, nop=1)
    F = disparity(left, right, prm)
    c, _ = preprocess.confidence(left, right, F, None, CP)
    known = gt > 0
    figures["layered"] = curves([np.abs(-F - gt)[known]], [c[known]])
    cam = dict(fx=721.5, fy=721.5, cx=609.6, cy=172.9, baseline=0.54, doffs=0.0)
    h, w, n = 375, 1242, a.pairs
    rels = [np.concatenate([synth.axis_angle((0.0, math.radians(0.3 * (k % 3 - 1)), 0.0)),
                            np.array([[0.02 * (k % 2)], [0.0], [-0.5]])], 1) for k in range(n - 1)]
    clip = synth.rigid_stereo_clip(n - 1, h, w, 1, 2, cam, rels, block={"velocity": (0.0, 0.0, 0.0)})
    prm = params.operating_point(2, w, noc=1, nop=1)
    errs, confs = [], []
    for k in range(n):
        F = disparity(clip["left"][k], clip["right"][k], prm)
        c, _ = preprocess.confidence(clip["left"][k], clip["right"][k], F, None, CP)
        g = clip["disp"][k]
        known = np.isfinite(g) & (g > 0)
        errs.append(np.abs(-F - g)[known])
        confs.append(c[known])
    figures["kitti"] = curves(errs, confs)
    print(json.dumps(figures))


if __name__ == "__main__":
    main()
