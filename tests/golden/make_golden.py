"""Generates tests/golden/*.npz from the REFERENCE build (oracle/_ref, i.e. the
reference's own sources compiled in place by oracle/Makefile).  Run where the
reference sources are (oracle/Makefile's REF):

    make -C oracle ref && python tests/golden/make_golden.py

Each fixture holds the uint8 input pair, the parameters (20 CLI numbers + noc +
nop) and the reference flow at level sc_l, plus the patch-stage outputs of the
finest level (p, conv, cnt) for a fixed seeded coarser flow.

    python tests/golden/make_golden.py --digests

writes reference_digests.json instead: SHA-256 of the reference's float32 output
bits on the seeded inputs of tests/test_oracle.py (inputs the tests regenerate,
outputs too large to store as arrays).
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from of_dis_b200 import params, preprocess, synth  # noqa: E402
from oracle import ref_driver  # noqa: E402


def write_digests(out_dir):
    import test_oracle as t

    out = {}
    i0, i1, pyr, prm, fl = t.cfg1_inputs()
    out["cfg1_input"] = t.input_digest(i0, i1)
    out["cfg1_run"] = t.digest(ref_driver.ref_run(pyr, prm))
    out["cfg1_varref"] = t.digest(ref_driver.ref_level_varref(pyr, prm, prm.sc_l, fl))
    for seed in range(40):
        i0, i1, pyr, prm = t.random_config_inputs(seed)
        out["random_%d_input" % seed] = t.input_digest(i0, i1)
        out["random_%d" % seed] = t.digest(ref_driver.ref_run(pyr, prm))
    for name in t.BASELINE_CASES:
        i0, i1, pyr, prm = t.baseline_inputs(name)
        out["baseline_%s_input" % name] = t.input_digest(i0, i1)
        out["baseline_" + name] = t.digest(ref_driver.ref_run(pyr, prm))
    out.update(sor_division_digests())
    out.update(degenerate_digests())
    out.update(batched_digests())
    out.update(geometry_digests())
    with open(os.path.join(out_dir, "reference_digests.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


def degenerate_digests():
    """The degenerate image families of tests/test_degenerate_content_gpu.py on every parameter set there: input
    pair, whole run, the patch stage at sc_l without and with the coarser flow, and the refinement of sc_l."""
    import test_oracle as t
    from test_degenerate_content_gpu import CASES, degenerate_inputs

    out = {}
    for family, route in CASES:
        i0, i1, pyr, prm = degenerate_inputs(family, route)
        key = "degen_%s_%s" % (family, route)
        out[key + "_input"] = t.input_digest(i0, i1)
        out[key + "_run"] = t.digest(ref_driver.ref_run(pyr, prm))
        out[key + "_patches"], out[key + "_varref"] = t.degenerate_stage(ref_driver.ref_level_patches,
                                                                         ref_driver.ref_level_varref, pyr, prm)
    return out

def batched_digests():
    """The distinct pairs of every configuration of tests/test_batched_configs_gpu.py and those of the largest context
    of tests/test_cabi.py: input pairs, and one digest over the whole runs of the pairs."""
    import test_oracle as t

    out = {}
    for name in t.BATCHED:
        out["batched_%s_input" % name], out["batched_%s_runs" % name] = t.batched_digests(ref_driver.ref_run, name)
    out["frame_limit_input"], out["frame_limit_runs"] = t.frame_limit_digests(ref_driver.ref_run)
    return out


def geometry_digests():
    """The cases of tests/test_patch_geometry_gpu.py: paddings wider than the patch on every patch kernel (input pair,
    whole run, patch stage at sc_l, refinement of sc_l), patch sizes 2 to 52 (input pair, whole run, patch stage), the
    clips of the upload paths and the pairs of the batch of more than 16 frames (inputs, one digest over the runs)."""
    import test_oracle as t
    import test_patch_geometry as g
    from test_patch_geometry_gpu import PAD_CASES, SIZE_CASES, UPLOAD_CASES, pad_inputs, size_inputs

    out = {}
    for route, pad in PAD_CASES:
        i0, i1, pyr, _, prm = pad_inputs(route, pad)
        key = "geometry_pad_%s_%s" % (route, pad)
        run, lvl, vr = g.pad_stage(ref_driver.ref_run, ref_driver.ref_level_patches, ref_driver.ref_level_varref, pyr,
                                   prm)
        out[key + "_input"], out[key + "_run"] = t.input_digest(i0, i1), t.digest(run)
        out[key + "_patches"], out[key + "_varref"] = t.patches_digest([lvl]), t.digest(vr)
    for name in SIZE_CASES:
        i0, i1, pyr, prm = size_inputs(name)
        key = "geometry_size_%s" % name
        run, lvl = g.size_stage(ref_driver.ref_run, ref_driver.ref_level_patches, pyr, prm)
        out[key + "_input"], out[key + "_run"], out[key + "_patches"] = t.input_digest(i0, i1), t.digest(run), \
            t.patches_digest([lvl])
    for name in UPLOAD_CASES:
        out["geometry_upload_%s_input" % name], out["geometry_upload_%s_runs" % name] = g.upload_digests(ref_driver.ref_run, name)
    out["geometry_batch_input"], out["geometry_batch_runs"] = g.batch_digests(ref_driver.ref_run)
    return out


def sor_division_digests():
    """The stereo SOR's division regimes (tests/test_sor_division_gpu.py: parameters that drive A11 and B1 out of the
    range of the kernels' written-out division): whole run, and the refinement of level sc_l from the regime's
    initial disparity."""
    import test_oracle as t
    from test_sor_division_gpu import DIV_CASES, REGIMES, division_inputs, initial_disparity

    out = {}
    for case in DIV_CASES:
        for regime in REGIMES:
            i0, i1, pyr, prm = division_inputs(case, regime)
            key = "sor_div_%s_%s" % (case, regime)
            out[key + "_input"] = t.input_digest(i0, i1)
            out[key + "_run"] = t.digest(ref_driver.ref_run(pyr, prm))
            out[key + "_varref"] = t.digest(ref_driver.ref_level_varref(pyr, prm, prm.sc_l, initial_disparity(regime, pyr, prm)))
    return out


CASES = {
    # name: (h, w, channels, cli numbers, nop, amp, stereo)
    "gray_flow_l2": (128, 256, 1, "3 1 12 12 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 2, 5.0, False),
    "gray_flow_l1cost": (96, 200, 1, "3 1 16 16 0.05 0.95 0 8 0.4 0 1 1 1 10 10 5 1 3 1.6 0", 2, 5.0, False),
    "gray_flow_huber_p12": (120, 216, 1, "3 1 16 16 0.05 0.95 0 12 0.75 0 1 2 1 10 10 5 1 3 1.6 0", 2, 4.0, False),
    "rgb_flow_l1cost": (104, 184, 3, "3 1 16 16 0.05 0.95 0 12 0.75 0 1 1 1 10 10 5 1 3 1.6 0", 2, 4.0, False),
    "gray_stereo": (96, 224, 1, "3 1 24 24 0.05 0.95 0 12 0.75 0 1 0 1 10 10 5 1 3 1.6 0", 1, 4.0, True),
    "gray_flow_earlyexit": (100, 168, 1, "3 1 16 2 0.05 0.95 0.5 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 2, 5.0, False),
    "gray_flow_big_motion": (128, 256, 1, "3 1 12 12 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 2, 40.0, False),
    # forward-backward consistency (README parameter 10 = 1): second grid on the swapped images
    "gray_flow_fbcon": (120, 200, 1, "3 1 8 8 0.05 0.95 0 8 0.4 1 1 0 1 10 10 5 1 3 1.6 0", 2, 6.0, False),
    "rgb_flow_fbcon_l1cost": (104, 184, 3, "3 1 8 8 0.05 0.95 0 12 0.75 1 1 1 1 10 10 5 1 3 1.6 0", 2, 4.0, False),
    "gray_stereo_fbcon": (96, 224, 1, "3 1 12 12 0.05 0.95 0 8 0.4 1 1 0 1 10 10 5 1 3 1.6 0", 1, 4.0, True),
}


def main():
    out_dir = os.path.dirname(os.path.abspath(__file__))
    if sys.argv[1:] == ["--digests"]:
        write_digests(out_dir)
        return
    only = sys.argv[1:]  # optional: generate just these fixtures
    for name, (h, w, ch, cli, nop, amp, stereo) in CASES.items():
        if only and name not in only:
            continue
        prm = params.from_cli_numbers(cli.split(), noc=ch, nop=nop)
        i0, i1, _ = synth.synthetic_pair(h, w, ch, seed=len(name), amp=amp, stereo=stereo)
        pyr = preprocess.PairPyramids(i0, i1, prm.sc_f, prm.p_samp_s)
        flow = ref_driver.ref_run(pyr, prm)
        lv = prm.sc_l
        hh, ww = pyr.level_shape(lv + 1)
        rng = np.random.default_rng(7)
        fp = (rng.standard_normal((hh, ww, nop)) * 1.5).astype(np.float32)
        if stereo:
            fp = -np.abs(fp)
        lvl = ref_driver.ref_level_patches(pyr, prm, lv, fp)
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), img0=i0, img1=i1,
                            cli=np.array([float(x) for x in cli.split()]), noc=ch, nop=nop, flow=flow,
                            flow_prev=fp, p=lvl["p"], conv=lvl["conv"], cnt=lvl["cnt"], dense=lvl["dense"])
        print(name, flow.shape, float(np.abs(flow).max()))


if __name__ == "__main__":
    main()
