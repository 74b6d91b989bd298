"""CPU tests of the checker itself: the C restatement (oracle/dis_oracle.c) must
equal (a) the committed golden fixtures produced by the reference build -- whole
arrays, or the SHA-256 of the reference's output bits (golden/reference_digests.json)
where the output is too large to store -- and (b), where oracle/_ref exists, the
reference build itself -- bit for bit."""
import glob
import hashlib
import json
import os

import numpy as np
import pytest

from of_dis_b200 import params, preprocess, synth
from oracle import ref_driver
from test_batched_configs_gpu import CONFIGS as BATCHED, batched_inputs
from test_cabi import LIMIT_CLI, limit_pairs
from test_degenerate_content_gpu import CASE_IDS as DEGEN_IDS, CASES as DEGEN_CASES, ROUTES as DEGEN_ROUTES
from test_degenerate_content_gpu import coarser_flow, degenerate_inputs, stage_params
from test_sor_division_gpu import DIV_CASES, REGIMES, division_inputs, initial_disparity

GOLDEN_DIR = os.path.join(os.path.dirname(__file__), "golden")
GOLDEN = sorted(glob.glob(os.path.join(GOLDEN_DIR, "*.npz")))
with open(os.path.join(GOLDEN_DIR, "reference_digests.json")) as _f:
    REF_DIGESTS = json.load(_f)


def digest(a, dtype=np.float32):
    """Shape and SHA-256 of the bits of `a`: equal digests == bitwise equal arrays."""
    a = np.ascontiguousarray(a, dtype)
    return "%s:%s" % ("x".join(map(str, a.shape)), hashlib.sha256(a.tobytes()).hexdigest())


def input_digest(i0, i1):
    return digest(np.stack([i0, i1]), np.uint8)


def check_inputs(key, i0, i1):
    """The seeded 8-bit input pair must be the one the reference digest was taken on (synth.py goes through
    numpy/scipy): a mismatch here means the inputs moved, not the port."""
    assert input_digest(i0, i1) == REF_DIGESTS[key + "_input"], "%s: synthetic inputs differ from the recorded ones" % key


def _load(path):
    z = np.load(path)
    prm = params.from_cli_numbers(z["cli"], noc=int(z["noc"]), nop=int(z["nop"]))
    pyr = preprocess.PairPyramids(z["img0"], z["img1"], prm.sc_f, prm.p_samp_s)
    return z, prm, pyr


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_port_matches_golden_bitwise(path, oracle_port):
    z, prm, pyr = _load(path)
    flow = oracle_port.port_run(pyr, prm)
    assert np.array_equal(bits(flow), bits(z["flow"]))
    lvl = oracle_port.port_level_patches(pyr, prm, prm.sc_l, z["flow_prev"])
    assert np.array_equal(bits(lvl["p"]), bits(z["p"]))
    assert np.array_equal(lvl["conv"], z["conv"]) and np.array_equal(lvl["cnt"], z["cnt"])
    assert np.array_equal(bits(lvl["dense"]), bits(z["dense"]))


@pytest.mark.skipif(not ref_driver.ref_available("m1c1"), reason="oracle/_ref not built")
@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_reference_build_reproduces_golden(path):
    z, prm, pyr = _load(path)
    if not ref_driver.ref_available(prm.flavour()):
        pytest.skip("flavour not built")
    assert np.array_equal(bits(ref_driver.ref_run(pyr, prm)), bits(z["flow"]))


def cfg1_inputs():
    """BASELINE config 1 (640x480 gray, op-point 2) and an arbitrary smooth-ish flow of its finest level."""
    i0, i1, _ = synth.synthetic_pair(480, 640, 1, seed=3)
    prm = params.operating_point(2, 640)
    pyr = preprocess.PairPyramids(i0, i1, prm.sc_f, prm.p_samp_s)
    h, w = pyr.level_shape(prm.sc_l)
    rng = np.random.default_rng(0)
    fl = (rng.standard_normal((h, w, 2)) * 0.7).astype(np.float32)
    return i0, i1, pyr, prm, fl


def test_port_vs_reference_cfg1_and_stages(oracle_port):
    """BASELINE config 1 (640x480 gray, op-point 2) whole run, plus per-stage checks."""
    i0, i1, pyr, prm, fl = cfg1_inputs()
    check_inputs("cfg1", i0, i1)
    assert digest(oracle_port.port_run(pyr, prm)) == REF_DIGESTS["cfg1_run"]
    # variational refinement alone
    lv = prm.sc_l
    assert digest(oracle_port.port_level_varref(pyr, prm, lv, fl)) == REF_DIGESTS["cfg1_varref"]
    st = oracle_port.varref_stages(pyr, prm, lv, fl)
    out = np.stack([st["uu"], st["vv"]], -1)
    assert np.array_equal(bits(out), bits(oracle_port.port_level_varref(pyr, prm, lv, fl)))


def test_packet_order_sum_is_the_documented_order(oracle_port):
    import ctypes

    rng = np.random.default_rng(5)
    for n in (1, 3, 4, 7, 8, 12, 36, 64, 100, 144, 432):
        v = (rng.standard_normal(n) * 100).astype(np.float32)
        got = np.float32(oracle_port.lib().dis_sum_packet_order(v.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), n))
        n4, n8 = n // 4 * 4, n // 8 * 8
        if n4:
            a = v[0:4].copy()
            if n4 > 4:
                b = v[4:8].copy()
                for i in range(8, n8, 8):
                    a = a + v[i:i + 4]
                    b = b + v[i + 4:i + 8]
                a = a + b
                if n4 > n8:
                    a = a + v[n8:n8 + 4]
            r = np.float32(np.float32(a[0] + a[2]) + np.float32(a[1] + a[3]))
            for i in range(n4, n):
                r = np.float32(r + v[i])
        else:
            r = v[0]
            for i in range(1, n):
                r = np.float32(r + v[i])
        assert got == r


def test_properties_zero_flow_and_translation(oracle_port):
    """SURVEY section 4(iii): identical images -> zero flow; integer shift recovered."""
    i0, _, _ = synth.synthetic_pair(128, 192, 1, seed=11)
    prm = params.from_cli_numbers("3 1 12 12 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0".split())
    pyr = preprocess.PairPyramids(i0, i0, prm.sc_f, prm.p_samp_s)
    assert np.abs(oracle_port.port_run(pyr, prm)).max() == 0.0
    big, _, _ = synth.synthetic_pair(128, 192 + 8, 1, seed=12)
    a, b = np.ascontiguousarray(big[:, 4:-4]), np.ascontiguousarray(big[:, 2:-6])  # I1(x+2) = I0(x)
    pyr = preprocess.PairPyramids(a, b, prm.sc_f, prm.p_samp_s)
    fl = preprocess.postprocess(oracle_port.port_run(pyr, prm), prm.sc_l, pyr.padw, pyr.padh, 192, 128)
    inner = fl[16:-16, 16:-16]
    assert abs(np.median(inner[..., 0]) - 2.0) < 0.1 and abs(np.median(inner[..., 1])) < 0.1


# ---- the port against the reference build on everything the GPU tests use it for ----------------
def random_config_inputs(seed):
    """Inputs of tests/test_gpu_parity.py::test_random_configurations_vs_oracle[seed]."""
    from test_gpu_parity import _random_config

    rng = np.random.default_rng(1000 + seed)
    numbers, ch, nop, size, amp = _random_config(rng)
    prm = params.from_cli_numbers(numbers, noc=ch, nop=nop)
    i0, i1, _ = synth.synthetic_pair(size[0], size[1], ch, seed=200 + seed, stereo=(nop == 1), amp=amp)
    return i0, i1, preprocess.PairPyramids(i0, i1, prm.sc_f, prm.p_samp_s), prm


@pytest.mark.parametrize("seed", range(40))
def test_port_vs_reference_on_the_random_configurations_of_the_gpu_suite(seed, oracle_port):
    """The 40 seeded parameter sets of tests/test_gpu_parity.py::test_random_configurations_vs_oracle:
    the port (the GPU tests' checker) must equal the reference build on each of them."""
    i0, i1, pyr, prm = random_config_inputs(seed)
    check_inputs("random_%d" % seed, i0, i1)
    assert digest(oracle_port.port_run(pyr, prm)) == REF_DIGESTS["random_%d" % seed]


BASELINE_CASES = {
    "cfg2_seed1": (436, 1024, 1, lambda: params.operating_point(2, 1024), 1, False),
    "cfg2_seed7": (436, 1024, 1, lambda: params.operating_point(2, 1024), 7, False),
    "cfg3_1920x1080_rgb_l1": (1080, 1920, 3, lambda: params.from_cli_numbers(
        "6 2 16 16 0.05 0.95 0 12 0.75 0 1 1 1 10 10 5 1 3 1.6 0".split(), noc=3), 2, False),
    "cfg5_2880x1988_stereo_op4": (1988, 2880, 1, lambda: params.operating_point(4, 2880, noc=1, nop=1), 4, True),
}


def baseline_inputs(name):
    h, w, ch, mk, seed, stereo = BASELINE_CASES[name]
    prm = mk()
    i0, i1, _ = synth.synthetic_pair(h, w, ch, seed=seed, stereo=stereo, amp=6.0)
    return i0, i1, preprocess.PairPyramids(i0, i1, prm.sc_f, prm.p_samp_s), prm


@pytest.mark.parametrize("name", list(BASELINE_CASES))
def test_port_vs_reference_at_baseline_sizes(name, oracle_port):
    """BASELINE configs[1], [2] and [4] at full size (the inputs of the GPU suite's full-size tests)."""
    i0, i1, pyr, prm = baseline_inputs(name)
    check_inputs("baseline_" + name, i0, i1)
    assert digest(oracle_port.port_run(pyr, prm)) == REF_DIGESTS["baseline_" + name]


@pytest.mark.parametrize("regime", list(REGIMES))
@pytest.mark.parametrize("case", DIV_CASES)
def test_port_vs_reference_at_the_sor_division_regimes(case, regime, oracle_port):
    """The stereo parameter regimes of tests/test_sor_division_gpu.py, which drive the SOR's A11 and B1 out of the
    range of the GPU's written-out division (or make B1 exactly zero): whole run, and the refinement of level sc_l
    from the regime's initial disparity, bit for bit as the reference build computes them."""
    i0, i1, pyr, prm = division_inputs(case, regime)
    key = "sor_div_%s_%s" % (case, regime)
    check_inputs(key, i0, i1)
    assert digest(oracle_port.port_run(pyr, prm)) == REF_DIGESTS[key + "_run"]
    fl = initial_disparity(regime, pyr, prm)
    assert digest(oracle_port.port_level_varref(pyr, prm, prm.sc_l, fl)) == REF_DIGESTS[key + "_varref"]


# ---- degenerate content (tests/test_degenerate_content_gpu.py) ---------------------------------------------------
def patches_digest(levels):
    """SHA-256 of the bits of p, pweight, conv, cnt and dense of each patch-stage result in `levels`, in turn"""
    h = hashlib.sha256()
    for lvl in levels:
        for k in ("p", "pweight", "conv", "cnt", "dense"):
            h.update(np.ascontiguousarray(lvl[k]).tobytes())
    return h.hexdigest()


def degenerate_stage(drv_patches, drv_varref, pyr, prm):
    """The per-stage checks of a degenerate case with one driver: the patch stage at sc_l without and with the
    coarser flow, and the refinement of sc_l from the dense flow of the latter."""
    sprm = stage_params(prm)
    lv = [drv_patches(pyr, sprm, prm.sc_l, f) for f in (None, coarser_flow(pyr, prm))]
    return patches_digest(lv), digest(drv_varref(pyr, sprm, prm.sc_l, lv[1]["dense"]))


@pytest.mark.parametrize("family,route", DEGEN_CASES, ids=DEGEN_IDS)
def test_port_vs_reference_on_degenerate_content(family, route, oracle_port):
    """The inputs of tests/test_degenerate_content_gpu.py (flat, striped, checkerboard, noise, saturated and mixed
    frames): the whole run, the patch stage at sc_l and the refinement of sc_l, bit for bit as the reference build
    computes them; where oracle/_ref exists also the run against the reference build directly."""
    i0, i1, pyr, prm = degenerate_inputs(family, route)
    key = "degen_%s_%s" % (family, route)
    check_inputs(key, i0, i1)
    run = oracle_port.port_run(pyr, prm)
    assert digest(run) == REF_DIGESTS[key + "_run"]
    patches, varref = degenerate_stage(oracle_port.port_level_patches, oracle_port.port_level_varref, pyr, prm)
    assert patches == REF_DIGESTS[key + "_patches"]
    assert varref == REF_DIGESTS[key + "_varref"]
    if ref_driver.ref_available(prm.flavour()):
        assert np.array_equal(bits(ref_driver.ref_run(pyr, prm)), bits(run))


# at least this many patches of every patch kernel's parameter sets take each fallback, and stop at cnt == 0
BRANCH_FLOOR = 50


def test_degenerate_content_reaches_the_hessian_fallbacks_on_every_patch_kernel(oracle_port):
    """Without this the GPU tests of degenerate content could pass while testing nothing: per patch kernel (P = 8 gray
    at 8 and 4 lanes per patch, P = 12, generic), the cases' patches at sc_l take each Hessian fallback (flow: A
    det H == 0 with H00 == 0, B det H == 0 with H00 > 0, C Cholesky pivot <= 0; stereo: D H00 == 0) and stop at
    cnt == 0 at least BRANCH_FLOOR times.  A patch without gradients (A, D) never moves (dp == 0), so where
    min_iter < max_iter it stops at cnt == min_iter on the ratio test 0 / 0: that too, at least BRANCH_FLOOR times.
    And the mixed frame holds, in one warp's aligned group of four patches, a fallback patch beside a regular one,
    and a patch that stops at once beside one that iterates."""
    pd = oracle_port
    counts = {k[0]: dict(A=0, B=0, C=0, D=0, cnt0=0, ratio00=0) for k in DEGEN_ROUTES.values()}
    for family, route in DEGEN_CASES:
        _, _, pyr, prm = degenerate_inputs(family, route)
        br = pd.port_level_branches(pyr, prm, prm.sc_l)
        cnt = pd.port_level_patches(pyr, stage_params(prm), prm.sc_l, None, want_dense=False)["cnt"]
        c = counts[DEGEN_ROUTES[route][0]]
        c["A"] += int((br & pd.HESS_SINGULAR_ZERO != 0).sum())
        c["B"] += int((br & pd.HESS_SINGULAR != 0).sum())
        c["C"] += int((br & pd.HESS_NOT_PD != 0).sum())
        c["D"] += int((br & pd.HESS_STEREO_ZERO != 0).sum())
        c["cnt0"] += int((cnt == 0).sum())
        if 0 < prm.min_iter < prm.max_iter:
            still = (br & (pd.HESS_SINGULAR_ZERO | pd.HESS_STEREO_ZERO) != 0) & (cnt == prm.min_iter)
            c["ratio00"] += int(still.sum())
        if family == "mixed":
            n4 = br.size // 4 * 4
            g_br, g_cnt = br[:n4].reshape(-1, 4), cnt[:n4].reshape(-1, 4)
            both = ((g_br != 0).any(1) & (g_br == 0).any(1)).sum()
            stop = ((g_cnt == 0).any(1) & (g_cnt > 0).any(1)).sum()
            assert both > 0 and stop > 0, (route, both, stop)
    for kernel, c in counts.items():
        for k, v in c.items():
            assert v >= BRANCH_FLOOR, "%s: %s reached %d times only (%s)" % (kernel, k, v, c)


@pytest.mark.skipif(not ref_driver.ref_available("m1c1"), reason="oracle/_ref not built")
def test_native_thread_pool_drivers_reproduce_single_runs():
    """ofdis_ref_run_many / ofdis_ref_run_many_u8 (the CPU baseline's drivers): same flows as one
    ofdis_ref_run per pair, and the restated pyramid / upsampling equal of_dis_b200/preprocess.py
    (which tests/test_preprocess.py pins to cv2), bit for bit."""
    prm = params.from_cli_numbers("3 1 8 8 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0".split())
    pairs = [synth.synthetic_pair(121, 203, 1, seed=30 + s)[:2] for s in range(3)]  # odd size: padding + crop
    pyrs = [preprocess.PairPyramids(a, b, prm.sc_f, prm.p_samp_s) for a, b in pairs]
    _, flows = ref_driver.ref_run_many(pyrs, prm, nrep=2, threads=3)
    frames = np.stack([np.stack([a, b]) for a, b in pairs])[..., None]
    _, full = ref_driver.ref_run_many_u8(frames, prm, nrep=1, threads=2)
    for q, p in enumerate(pyrs):
        one = ref_driver.ref_run(p, prm)
        assert np.array_equal(bits(flows[q]), bits(one))
        exp = preprocess.postprocess(one, prm.sc_l, p.padw, p.padh, 203, 121)
        assert np.array_equal(bits(full[q]), bits(exp.reshape(full[q].shape)))


# ---- batched launches (tests/test_batched_configs_gpu.py) and the largest context (tests/test_cabi.py) -------------
def pairs_digests(run, prm, pairs, pyrs):
    """digest of the 8-bit input pairs, and one digest over the flows `run` computes for them, in turn"""
    return digest(np.stack([np.stack(p) for p in pairs]), np.uint8), digest(np.stack([run(p, prm) for p in pyrs]))


def batched_digests(run, name):
    prm, pairs, pyrs = batched_inputs(name)
    return pairs_digests(run, prm, pairs, pyrs)


def frame_limit_digests(run):
    prm = params.from_cli_numbers((LIMIT_CLI % 0).split())
    pairs = limit_pairs()
    return pairs_digests(run, prm, pairs, [preprocess.PairPyramids(a, b, prm.sc_f, prm.p_samp_s) for a, b in pairs])


@pytest.mark.parametrize("name", list(BATCHED))
def test_port_vs_reference_on_the_batched_configurations(name, oracle_port):
    """The distinct pairs of every configuration of the batched sweep: whole runs, bit for bit as the reference build
    computes them."""
    inp, runs = batched_digests(oracle_port.port_run, name)
    assert inp == REF_DIGESTS["batched_%s_input" % name], "%s: synthetic inputs differ from the recorded ones" % name
    assert runs == REF_DIGESTS["batched_%s_runs" % name]


def test_port_vs_reference_on_the_pairs_of_the_largest_context(oracle_port):
    inp, runs = frame_limit_digests(oracle_port.port_run)
    assert inp == REF_DIGESTS["frame_limit_input"] and runs == REF_DIGESTS["frame_limit_runs"]
