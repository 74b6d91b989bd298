"""The launch plans of the refinement and the patch stage (CPU: ofdis_debug_sor_plan makes no CUDA call).

The planner (sor_plan) and assemble_kernel's rows-per-thread rule decide, per level and launch, which kernel
instances run.  This test enumerates everything they can choose over a grid of level sizes, sweep counts, frame
counts and option values, and checks that the batched sweep of tests/test_batched_configs_gpu.py reaches every item
of that set, level by level and launch by launch, so that no instance escapes the GPU comparison with the oracle.

    python tests/test_launch_plans.py    lists the reachable set and the configurations that reach each item
"""
import os
import sys

import pytest

_TESTS = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [p for p in (_TESTS, os.path.dirname(_TESTS)) if p not in sys.path]
from test_batched_configs_gpu import CONFIGS, config_params  # noqa: E402

AUTO_FRAMES = 16  # SOR_LANE_AUTO_FRAMES: launches of more internal frames switch the defaults


@pytest.fixture(scope="module")
def api():
    from of_dis_b200 import api as _api

    _api.lib()
    return _api


def plan_items(plan, h, nop, noc, asm_rows=None):
    """The kernel instances and launch shapes of one level's refinement launch"""
    kind = plan["kind"]
    items = set()
    if kind.startswith("wave_"):
        items.add(("sor_wave_kernel", nop, plan["hpad"], plan["rt"], kind[5:]))
        if kind == "wave_single" and -(-h // plan["rt"]) > plan["ml"]:
            items.add(("stage copy wraps", nop))  # more lanes than stage slots: the producer's copy wraps
    elif kind == "lane":
        items.add(("sor_lane_kernel", nop, "bands" if plan["nb"] > 1 else "one band"))
    else:
        items.add(("sor_redblack_kernel", nop))
    if plan["tail_sweeps"]:
        items.add(("shorter last launch", kind))
    rows = plan["assemble_rows"] if asm_rows is None else asm_rows
    items.add(("assemble_kernel", noc, nop, rows, plan["assemble_mode"]))
    return items


def patch_item(prm, internal_frames, patch_lanes):
    """Kernel of launch_patch_optimize (patch_kernels.cu) for these parameters (imgpadding = P)"""
    if prm.p_samp_s == 8 and prm.noc == 1:
        lanes = patch_lanes or (4 if internal_frames > AUTO_FRAMES else 8)
        return ("patch_p8c1", prm.nop, lanes)
    if prm.p_samp_s == 12:
        return ("patch_p12", prm.nop, prm.noc)
    return ("patch_generic", prm.nop)


def _heights():
    hs = {4, 5, 7, 8, 9, 16, 24, 31, 32, 33, 40, 48, 56, 16383, 16384}
    for k in (1, 1.5, 2, 3, 4, 6, 8, 12, 16, 24, 32, 48, 64, 96, 128, 192, 256, 384, 512):
        for d in (-1, 0, 1):
            hs.add(int(32 * k) + d)
    return sorted(h for h in hs if 4 <= h <= 16384)


def reachable_items(api):
    """Everything the planner can choose (exact mode; the red-black solver is tests/test_fast_mode.py's)"""
    items = set()
    for h in _heights():
        for w in (8, 512):
            for nop in (1, 2):
                for K in (1, 2, 3, 4, 5, 6, 9):
                    for lane, frames in ((0, 1), (1, 1), (2, 1), (2, 17)):
                        for rt in (1, 2, 4):
                            for sm in (32, 64, 128):
                                for mc in (1, 2, 4, 8, 16):
                                    p = api.debug_sor_plan(w, h, nop, 1, K, frames, lane, 0, rt, sm, mc)
                                    if p:
                                        items |= {i for i in plan_items(p, h, nop, 1) if i[0] != "assemble_kernel"}
    for h in (4, 64, 300):
        for w in (8, 512):
            for frames in (1, 17, 64):
                for nop in (1, 2):
                    for noc in (1, 3):
                        for lane in (0, 1):
                            p = api.debug_sor_plan(w, h, nop, noc, 3, frames, lane, 0, 1, 128, 8)
                            items |= {i for i in plan_items(p, h, nop, noc) if i[0] == "assemble_kernel"}
    items |= {("patch_p8c1", nop, lanes) for nop in (1, 2) for lanes in (4, 8)}
    items |= {("patch_p12", nop, c) for nop in (1, 2) for c in (1, 3)}
    items |= {("patch_generic", nop) for nop in (1, 2)}
    return items


def sweep_items(api, configs=CONFIGS):
    """{item: [configuration names]} of the launches the batched sweep runs: ofdis_run of all its frames, then the
    patch stage and the refinement of sc_l on its sub-range"""
    got = {}
    for name, cfg in configs.items():
        prm = config_params(cfg)
        H, W = cfg["size"]
        o = cfg["options"]
        D = 2 if prm.usefbcon else 1
        f0, f1, _ = cfg["stage"]
        launches = [(lv, cfg["nfr"]) for lv in range(prm.sc_f, prm.sc_l - 1, -1)] + [(prm.sc_l, f1 - f0)]
        found = set()
        for lv, n in launches:
            found.add(patch_item(prm, n * D, o["patch_lanes"]))
            if not prm.usetvref:
                continue
            w, h = W >> lv, H >> lv
            p = api.debug_sor_plan(w, h, prm.nop, prm.noc, prm.tv_solverit, n * D, o["sor_lane"], 0,
                                   o["sor_rows_per_thread"], o["sor_single_max"], o["sor_max_cluster"])
            assert p is not None, (name, lv)
            # the last level with usefbcon refines the forward frames only: the plan is made for n * 2 frames,
            # assemble_kernel launches n
            rows = None
            if D == 2 and lv == prm.sc_l:
                rows = api.debug_sor_plan(w, h, prm.nop, prm.noc, prm.tv_solverit, n, o["sor_lane"], 0,
                                          o["sor_rows_per_thread"], o["sor_single_max"],
                                          o["sor_max_cluster"])["assemble_rows"]
            found |= plan_items(p, h, prm.nop, prm.noc, rows)
        for i in found:
            got.setdefault(i, []).append(name)
    return got


def test_hook_follows_the_planner_on_known_levels(api):
    """Plans the GPU suite's docstrings and DESIGN state"""
    p = api.debug_sor_plan(128, 56, 2, 1, 3, 64, 2, 0, 1, 128, 16)  # the bench workload's finest level
    assert (p["kind"], p["hpad"], p["ml"], p["sweeps"], p["assemble_rows"]) == ("wave_single", 64, 32, 3, 4)
    p = api.debug_sor_plan(128, 56, 2, 1, 3, 1, 2, 0, 1, 128, 16)  # one pair: sor_lane_kernel, two bands
    assert (p["kind"], p["nb"], p["assemble_mode"]) == ("lane", 2, 2)
    # 650 x 72 with sor_max_cluster 1: chains of 6 bands of 128 x 1 rows (flow), 3 of 256 x 1 (stereo)
    p = api.debug_sor_plan(72, 650, 2, 1, 3, 3, 0, 0, 1, 128, 1)
    assert (p["kind"], p["hpad"], p["nb"], p["sweeps"]) == ("wave_chain", 128, 6, 1)
    p = api.debug_sor_plan(72, 650, 1, 1, 3, 3, 0, 0, 1, 128, 1)
    assert (p["kind"], p["hpad"], p["nb"]) == ("wave_chain", 256, 3)
    assert api.debug_sor_plan(72, 650, 1, 1, 3, 3, 0, 1, 1, 128, 1)["assemble_mode"] == 1
    assert api.debug_sor_plan(72, 650, 1, 1, 50, 3, 0, 1, 1, 128, 1) is None  # red-black halo beyond shared memory
    with pytest.raises(api.OfdisError):
        api.debug_sor_plan(72, 650, 3, 1, 3, 3, 0, 0, 1, 128, 1)


def test_reachable_set_names_every_instance(api):
    items = reachable_items(api)
    waves = {i for i in items if i[0] == "sor_wave_kernel"}
    assert {i[4] for i in waves} == {"single", "cluster", "chain"}
    assert {i[2] for i in waves} == {32, 64, 128, 256} and {i[3] for i in waves} == {1, 2, 4}
    assert {i[2] for i in waves if i[4] == "single"} <= {32, 64, 128}
    assert len({(i[1], i[3]) for i in waves if i[4] == "chain"}) == 6  # one chain instantiation per (mode, rt)
    assert {i for i in items if i[0] == "sor_lane_kernel"} == {("sor_lane_kernel", n, b) for n in (1, 2)
                                                               for b in ("one band", "bands")}
    assert {i for i in items if i[0] == "assemble_kernel"} == {("assemble_kernel", c, n, r, m) for c in (1, 3)
                                                               for n in (1, 2) for r in (1, 2, 4) for m in (0, 2)}
    assert ("stage copy wraps", 1) in items and ("stage copy wraps", 2) in items
    assert {i[1] for i in items if i[0] == "shorter last launch"} == {"wave_single", "wave_cluster", "lane"}


def test_the_sweep_reaches_every_launch_plan(api):
    missing = reachable_items(api) - set(sweep_items(api))
    assert not missing, "the batched sweep misses %s: add a named case" % sorted(missing, key=str)


def main():
    from of_dis_b200 import api as _api

    got = sweep_items(_api)
    for i in sorted(reachable_items(_api), key=str):
        names = got.get(i, [])
        print("%-60s %3d  %s" % (i, len(names), " ".join(names[:4])))


if __name__ == "__main__":
    main()
