"""CPU pre-study of the monocular relative pose, bit-exact to the device: the oracle port's forward and backward flows
of the KITTI-sized synthetic clip (operating point 2, left view only) through preprocess.relpose with fb_check, and
the figures that tests/test_relpose_gpu.py bounds.  One JSON line: per pair the status, the rotation and
translation-direction errors in degrees, the share of the moving box's eroded interior at mask 1 and the AbsRel of
the median-scaled depth on the mask-0 background.

    python tools/relpose_prestudy.py"""
import json
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from scipy import ndimage

from of_dis_b200 import params, preprocess, synth
from oracle import port_driver

H, W = 375, 1242
CAM = dict(fx=721.5, fy=721.5, cx=609.6, cy=172.9, baseline=0.54, doffs=0.0)


def flow(a, b, prm):
    """The port's full-resolution flow of one pair (the device's get_flow_fullres, bit for bit)."""
    pyr = preprocess.PairPyramids(a, b, prm.sc_f, prm.p_samp_s)
    lv = port_driver.port_run(pyr, prm)
    return preprocess.postprocess(lv, prm.sc_l, pyr.width - W, pyr.height - H, W, H)


def motion(w, t):
    return np.concatenate([synth.axis_angle(w), np.asarray(t, np.float64).reshape(3, 1)], 1)


def main():
    rels = [motion((0.0, math.radians(0.5), 0.0), (0.0, 0.0, -0.9)),
            motion((math.radians(0.3), math.radians(-0.8), 0.0), (0.1, 0.0, -0.6)),
            motion((0.0, math.radians(1.0), 0.0), (0.0, 0.0, -0.3))]
    n = len(rels)
    clip = synth.rigid_stereo_clip(n, H, W, 1, 2, CAM, rels)
    prm = params.operating_point(2, W, noc=1)
    F = np.stack([flow(clip["left"][k], clip["left"][k + 1], prm) for k in range(n)])
    B = np.stack([flow(clip["left"][k + 1], clip["left"][k], prm) for k in range(n)])
    p = dict(fx=CAM["fx"], fy=CAM["fy"], cx=CAM["cx"], cy=CAM["cy"], step=4, fb_check=1, alpha=0.01, beta=0.5,
             hypotheses=1024, threshold=1.0, refine=5, min_parallax=0.5, seed=0)
    pose, stats, mask, _, depth = preprocess.relpose(F, B, p)
    r_err, t_err = preprocess.relpose_errors(pose, clip["poses"])
    fb = np.float32(np.float32(CAM["fx"]) * np.float32(CAM["baseline"]))
    out = []
    for k in range(n):
        box = clip["box"][k]
        interior = ndimage.binary_erosion(box, iterations=8)
        back = ~ndimage.binary_dilation(box, iterations=8)
        true_depth = fb / clip["disp"][k].astype(np.float64)
        d = depth[k].astype(np.float64)
        sel = back & (mask[k] == 0) & np.isfinite(d) & np.isfinite(true_depth)
        scale = np.median(true_depth[sel]) / np.median(d[sel])
        out.append(dict(status=int(stats["status"][k]), r_err=round(float(r_err[k]), 4),
                        t_dir_err=round(float(t_err[k]), 3), box_moving=round(float((mask[k][interior] == 1).mean()), 3),
                        absrel=round(float(np.mean(np.abs(d[sel] * scale - true_depth[sel]) / true_depth[sel])), 4)))
    print(json.dumps({"pairs": out}))


if __name__ == "__main__":
    main()
