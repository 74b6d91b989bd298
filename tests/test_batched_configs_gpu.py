"""Batched launches against the oracle (pytest -m gpu).  Which kernels a launch runs depends on how many frames it
carries: above 16 internal frames (pairs, x 2 with usefbcon) the P = 8 patch kernel takes 4 lanes per patch,
programmatic dependent launch is off and sor_lane_kernel gives way to sor_wave_kernel; assemble_kernel's rows per
thread follow frames x level size.  This sweep draws parameters, geometry, frames per launch and launch options at
random (seeded), adds named cases where the draws miss a launch plan (tests/test_launch_plans.py proves that the
configurations reach every plan the planner can choose), and checks every slot of every launch bitwise against the
oracle's flow of its pair -- eager and two graph replays -- plus the patch stage and two inner refinement iterations
on a sub-range of frames that does not start at 0.

The generator is importable without a GPU: tests/test_launch_plans.py evaluates the plans of these configurations and
tests/test_oracle.py pins the oracle to the reference build's digests of their pairs."""
import functools
import zlib

import numpy as np
import pytest

from of_dis_b200 import params, preprocess, synth
from test_gpu_parity import assert_bits

N_DISTINCT = 6  # distinct pairs per configuration, cycled over the slots
N_RANDOM = 44


def _level0(h_l, w_l, sc_l):
    return h_l << sc_l, w_l << sc_l


def random_batched_config(seed):
    """One seeded configuration: dict(numbers, ch, nop, size, amp, nfr, options, stage=(f0, f1, slot))."""
    rng = np.random.default_rng(5000 + seed)
    P = int(rng.choice([4, 6, 8, 8, 10, 12, 16]))
    ch = int(rng.choice([1, 3]))
    nop = int(rng.choice([1, 2]))
    fb = int(rng.random() < 0.3)
    tall = rng.random() < 0.25
    if tall:  # tall and narrow: clusters and chains of bands
        nlev, sc_l = int(rng.integers(1, 3)), 0
        w_l = int(rng.integers(6, 19)) * 4  # 24..72 columns
        h_l = int(rng.integers(300, 2600))
        ch = 1
    else:
        nlev, sc_l = int(rng.integers(1, 4)), int(rng.integers(0, 2))
        h_l = int(np.exp(rng.uniform(np.log(4), np.log(300))))
        w_l = int(rng.integers(8, 161))
    sc_f = sc_l + nlev - 1
    # the coarsest level keeps >= 4 rows and >= 2 columns (ofdis_create); level sizes are multiples of 2^(nlev-1)
    m = 1 << (nlev - 1)
    h_l = max(4 * m, h_l // m * m)
    w_l = max(2 * m, w_l // m * m)
    max_iter = int(rng.integers(1, 16))
    numbers = [sc_f, sc_l, max_iter, int(rng.integers(0, max_iter + 1)), float(rng.choice([0.05, 0.2, 0.5])),
               float(rng.choice([0.95, 0.8, 0.5])), float(rng.choice([0.0, 0.5, 2.0])), P,
               float(rng.choice([0.0, 0.3, 0.4, 0.5, 0.75])), fb, int(rng.integers(0, 2)), int(rng.integers(0, 3)),
               int(rng.random() < 0.85), float(rng.choice([10.0, 3.0, 30.0])), float(rng.choice([10.0, 0.0, 5.0])),
               float(rng.choice([5.0, 0.0, 12.0])), int(rng.integers(1, 3)), int(rng.integers(1, 6)),
               float(rng.choice([1.6, 1.0, 1.9])), 0]
    # frames per launch: mostly 17..64, some 16 or fewer; usefbcon at 9 or more pairs is above 16 internal frames
    u = rng.random()
    nfr = int(rng.integers(1, 17)) if u < 0.2 else (int(rng.integers(9, 33)) if fb else int(rng.integers(17, 65)))
    options = dict(sor_lane=int(rng.integers(0, 3)), pdl=int(rng.integers(0, 3)),
                   patch_lanes=int(rng.choice([0, 4, 8])), sor_rows_per_thread=int(rng.choice([1, 2, 4])),
                   sor_single_max=int(rng.choice([32, 64, 128])), sor_max_cluster=int(rng.choice([1, 2, 4, 8, 16])))
    return _finish(numbers, ch, nop, _level0(h_l, w_l, sc_l), float(rng.choice([1.0, 4.0, 8.0])), nfr, options, rng)


def _finish(numbers, ch, nop, size, amp, nfr, options, rng):
    f0 = int(rng.integers(1, nfr)) if nfr > 1 else 0
    f1 = int(rng.integers(f0 + 1, nfr + 1))
    return dict(numbers=numbers, ch=ch, nop=nop, size=size, amp=amp, nfr=nfr, options=options,
                stage=(f0, f1, int(rng.integers(f0, f1))))


def _named(seed, cli, ch, nop, level, nfr, options):
    """A named case: `cli` the 20 numbers, `level` (rows, columns) of level sc_l."""
    numbers = [float(x) if "." in x else int(x) for x in cli.split()]
    o = dict(sor_lane=2, pdl=2, patch_lanes=0, sor_rows_per_thread=1, sor_single_max=128, sor_max_cluster=8)
    o.update(options)
    rng = np.random.default_rng(9000 + seed)
    return _finish(numbers, ch, nop, _level0(level[0], level[1], numbers[1]), 4.0, nfr, o, rng)


# Plans the random draws miss (tests/test_launch_plans.py::test_the_sweep_reaches_every_launch_plan names them)
NAMED = {
    "assemble_c1_nop2_rows2_mode2": ("0 0 8 4 0.05 0.95 0 12 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 1, 2, (24, 48), 64, dict(sor_lane=1, sor_rows_per_thread=1, sor_single_max=128, sor_max_cluster=8)),
    "assemble_c1_nop2_rows4_mode2": ("0 0 8 4 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 1, 2, (4, 160), 64, dict(sor_lane=1, sor_rows_per_thread=1, sor_single_max=128, sor_max_cluster=8, patch_lanes=8)),
    "assemble_c3_nop1_rows2_mode0": ("0 0 8 4 0.05 0.95 0 6 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 3, 1, (24, 48), 64, dict(sor_lane=0, sor_rows_per_thread=1, sor_single_max=128, sor_max_cluster=8)),
    "assemble_c3_nop1_rows2_mode2": ("0 0 8 4 0.05 0.95 0 6 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 3, 1, (24, 48), 64, dict(sor_lane=1, sor_rows_per_thread=1, sor_single_max=128, sor_max_cluster=8)),
    "assemble_c3_nop1_rows4_mode2": ("0 0 8 4 0.05 0.95 0 6 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 3, 1, (4, 160), 64, dict(sor_lane=1, sor_rows_per_thread=1, sor_single_max=128, sor_max_cluster=8)),
    "assemble_c3_nop2_rows4_mode2": ("0 0 8 4 0.05 0.95 0 12 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 3, 2, (4, 160), 64, dict(sor_lane=1, sor_rows_per_thread=1, sor_single_max=128, sor_max_cluster=8)),
    "wave_nop1_hpad128_rt1_cluster": ("0 0 8 4 0.05 0.95 0 6 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 1, 1, (129, 48), 17, dict(sor_lane=0, sor_rows_per_thread=1, sor_single_max=128, sor_max_cluster=2)),
    "wave_nop1_hpad128_rt1_single": ("0 0 8 4 0.05 0.95 0 6 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 1, 1, (65, 48), 17, dict(sor_lane=0, sor_rows_per_thread=1, sor_single_max=128, sor_max_cluster=8)),
    "wave_nop1_hpad128_rt2_cluster": ("0 0 8 4 0.05 0.95 0 6 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 1, 1, (257, 48), 17, dict(sor_lane=0, sor_rows_per_thread=2, sor_single_max=128, sor_max_cluster=2)),
    "wave_nop1_hpad128_rt2_single": ("0 0 8 4 0.05 0.95 0 6 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 1, 1, (129, 48), 17, dict(sor_lane=0, sor_rows_per_thread=2, sor_single_max=128, sor_max_cluster=1)),
    "wave_nop1_hpad256_rt1_cluster": ("0 0 8 4 0.05 0.95 0 6 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 1, 1, (257, 48), 17, dict(sor_lane=0, sor_rows_per_thread=1, sor_single_max=128, sor_max_cluster=2)),
    "wave_nop1_hpad32_rt2_cluster": ("0 0 8 4 0.05 0.95 0 6 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 1, 1, (65, 48), 17, dict(sor_lane=0, sor_rows_per_thread=2, sor_single_max=32, sor_max_cluster=8)),
    "wave_nop1_hpad64_rt1_cluster": ("0 0 8 4 0.05 0.95 0 6 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 1, 1, (65, 48), 17, dict(sor_lane=0, sor_rows_per_thread=1, sor_single_max=64, sor_max_cluster=2)),
    "wave_nop1_hpad64_rt1_single": ("0 0 8 4 0.05 0.95 0 6 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 1, 1, (33, 48), 17, dict(sor_lane=0, sor_rows_per_thread=1, sor_single_max=128, sor_max_cluster=8)),
    "wave_nop1_hpad64_rt2_cluster": ("0 0 8 4 0.05 0.95 0 6 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 1, 1, (129, 48), 17, dict(sor_lane=0, sor_rows_per_thread=2, sor_single_max=128, sor_max_cluster=2)),
    "wave_nop1_hpad64_rt4_cluster": ("0 0 8 4 0.05 0.95 0 6 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 1, 1, (257, 48), 17, dict(sor_lane=0, sor_rows_per_thread=4, sor_single_max=128, sor_max_cluster=2)),
    "wave_nop1_hpad64_rt4_single": ("0 0 8 4 0.05 0.95 0 6 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 1, 1, (129, 48), 17, dict(sor_lane=0, sor_rows_per_thread=4, sor_single_max=128, sor_max_cluster=1)),
    "wave_nop2_hpad128_rt1_chain": ("0 0 8 4 0.05 0.95 0 6 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 1, 2, (33, 48), 17, dict(sor_lane=0, sor_rows_per_thread=1, sor_single_max=32, sor_max_cluster=1)),
    "wave_nop2_hpad128_rt1_cluster": ("0 0 8 4 0.05 0.95 0 6 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 1, 2, (129, 48), 17, dict(sor_lane=0, sor_rows_per_thread=1, sor_single_max=128, sor_max_cluster=2)),
    "wave_nop2_hpad128_rt2_chain": ("0 0 8 4 0.05 0.95 0 6 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 1, 2, (65, 48), 17, dict(sor_lane=0, sor_rows_per_thread=2, sor_single_max=32, sor_max_cluster=1)),
    "wave_nop2_hpad128_rt2_cluster": ("0 0 8 4 0.05 0.95 0 6 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 1, 2, (257, 48), 17, dict(sor_lane=0, sor_rows_per_thread=2, sor_single_max=128, sor_max_cluster=2)),
    "wave_nop2_hpad128_rt2_single": ("0 0 8 4 0.05 0.95 0 6 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 1, 2, (129, 48), 17, dict(sor_lane=0, sor_rows_per_thread=2, sor_single_max=128, sor_max_cluster=1)),
    "wave_nop2_hpad32_rt4_cluster": ("0 0 8 4 0.05 0.95 0 6 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 1, 2, (129, 48), 17, dict(sor_lane=0, sor_rows_per_thread=4, sor_single_max=128, sor_max_cluster=8)),
    "wave_nop2_hpad64_rt1_cluster": ("0 0 8 4 0.05 0.95 0 6 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 1, 2, (65, 48), 17, dict(sor_lane=0, sor_rows_per_thread=1, sor_single_max=64, sor_max_cluster=2)),
    "wave_nop2_hpad64_rt2_single": ("0 0 8 4 0.05 0.95 0 6 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 1, 2, (65, 48), 17, dict(sor_lane=0, sor_rows_per_thread=2, sor_single_max=128, sor_max_cluster=8)),
    "wave_nop2_hpad64_rt4_cluster": ("0 0 8 4 0.05 0.95 0 6 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 1, 2, (257, 48), 17, dict(sor_lane=0, sor_rows_per_thread=4, sor_single_max=128, sor_max_cluster=2)),
    "wave_nop2_hpad64_rt4_single": ("0 0 8 4 0.05 0.95 0 6 0.4 0 1 0 1 10 10 5 1 3 1.6 0", 1, 2, (129, 48), 17, dict(sor_lane=0, sor_rows_per_thread=4, sor_single_max=128, sor_max_cluster=1)),
}

CONFIGS = {"random_%d" % s: random_batched_config(s) for s in range(N_RANDOM)}
CONFIGS.update({name: _named(i, *args) for i, (name, args) in enumerate(NAMED.items())})


def config_params(cfg):
    return params.from_cli_numbers(cfg["numbers"], noc=cfg["ch"], nop=cfg["nop"])


@functools.lru_cache(maxsize=None)
def batched_inputs(name):
    """(prm, [(i0, i1)] * N_DISTINCT, [PairPyramids]) of configuration `name`."""
    cfg = CONFIGS[name]
    prm = config_params(cfg)
    h, w = cfg["size"]
    seed0 = zlib.crc32(name.encode()) % 100000
    pairs = [synth.synthetic_pair(h, w, cfg["ch"], seed=seed0 + d, stereo=(cfg["nop"] == 1), amp=cfg["amp"])[:2]
             for d in range(N_DISTINCT)]
    return prm, pairs, [preprocess.PairPyramids(a, b, prm.sc_f, prm.p_samp_s) for a, b in pairs]


@functools.lru_cache(maxsize=None)
def oracle_flows(name, oracle_port):
    """the oracle's flows of the distinct pairs of configuration `name`"""
    prm, _, pyrs = batched_inputs(name)
    return [oracle_port.port_run(p, prm) for p in pyrs]


def slot_pair(f):
    """distinct pair of slot f: neighbouring slots differ"""
    return f % N_DISTINCT


@pytest.fixture(scope="module")
def api():
    from of_dis_b200 import api as _api

    _api.lib()
    return _api


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CONFIGS))
def test_batched_configuration_vs_oracle(name, api, oracle_port):
    cfg = CONFIGS[name]
    prm, _, pyrs = batched_inputs(name)
    nfr, lv = cfg["nfr"], prm.sc_l
    ctx = api.Context(prm, pyrs[0].width, pyrs[0].height, pyrs[0].imgpadding, nfr)
    try:
        for k, v in cfg["options"].items():
            if k.startswith("sor_") and not prm.usetvref:
                continue  # no refinement, no SOR
            try:
                ctx.set_option(k, v)
            except api.OfdisError:
                if k == "sor_max_cluster" and v == 16:
                    pytest.skip("device grants no 16-CTA clusters")
                raise
        exp = oracle_flows(name, oracle_port)
        if prm.usefbcon:
            for f in range(nfr):
                ctx.upload_pyramids(f, pyrs[slot_pair(f)])
        else:
            ctx.upload_packed(0, nfr, np.stack([ctx.pack_frame(pyrs[slot_pair(f)]) for f in range(nfr)]))
        out = np.empty((nfr,) + exp[0].shape, np.float32)
        for graph, reps in ((False, 1), (True, 2)):
            ctx.set_graph_mode(graph)
            for rep in range(reps):
                out[:] = np.nan
                ctx.run(nfr)
                ctx.get_flow_batch(0, nfr, out)
                ctx.sync()
                for f in range(nfr):
                    assert_bits(out[f], exp[slot_pair(f)], "graph=%s replay %d slot %d" % (graph, rep, f))
        ctx.set_graph_mode(False)

        # stage operators on frames [f0, f1), f0 > 0: the patch stage of sc_l from a seeded coarser flow (from zero
        # where sc_l is the only level: an init flow needs frames padded to multiples of 2^(sc_f+1)) ...
        f0, f1, slot = cfg["stage"]
        rng = np.random.default_rng(11)
        fp = None
        if lv < prm.sc_f:
            hh, ww = pyrs[0].level_shape(lv + 1)
            fp = (rng.standard_normal((hh, ww, prm.nop)) * 1.5).astype(np.float32)
            if prm.nop == 1:
                fp = -np.abs(fp)
            for f in range(f0, f1):
                ctx.set_flow(f, lv + 1, fp)
        ctx.patgrid_optimize(lv, f0, f1, fp is not None)
        ctx.patgrid_aggregate(lv, f0, f1)
        for d in sorted({slot_pair(f) for f in range(f0, f1)}):
            f = next(f for f in range(f0, f1) if slot_pair(f) == d)
            ref = oracle_port.port_level_patches(pyrs[d], prm, lv, fp, want_dense=not prm.usefbcon)
            got = ctx.get_patches(f, lv)
            for k in ("p", "pweight", "conv", "cnt"):
                assert_bits(got[k], ref[k], "patch.%s slot %d" % (k, f))
            if not prm.usefbcon:  # with usefbcon the densification merges both grids (the whole run checks it)
                assert_bits(ctx.get_flow(f, lv), ref["dense"], "dense slot %d" % f)
        # ... and two inner iterations of the refinement of sc_l from a seeded dense flow in one slot
        if prm.usetvref:
            h, w = pyrs[0].level_shape(lv)
            dense = (rng.standard_normal((h, w, prm.nop)) * 1.5).astype(np.float32)
            if prm.nop == 1:
                dense = -np.abs(dense)
            ctx.set_flow(slot, lv, dense)
            ctx.varref_refine(lv, f0, f1, n_inner=2)
            it = oracle_port.varref_stages(pyrs[slot_pair(slot)], prm, lv, dense, n_iters=2)["iters"][1]
            dudv = ctx.debug_get("dudv", slot, lv)
            assert_bits(dudv[..., 0], it["du"], "du")
            if prm.nop == 2:
                assert_bits(dudv[..., 1], it["dv"], "dv")
            rec = ctx.debug_get("rec", slot, lv)
            assert_bits(rec[..., 3 if prm.nop == 2 else 1], it["b1"], "rec.b1")
    finally:
        ctx.close()
