"""Contexts that share a device (run on an H100: pytest -m gpu).  Every other GPU test runs one context at a time; the
library is used with many: bench.py's lanes (one context and stream per lane, graph replays overlapping), the command
line's and ShardedEngine's caller streams, and callers that drive contexts from several host threads.  Here contexts of
different configurations -- every patch kernel route, every SOR plan, forward-backward, init flow, the red-black mode --
are alive together, interleaved on one thread, on overlapping streams, on one shared stream with programmatic
dependent launch, and on concurrent threads; every flow is compared BITWISE with the oracle (sor_fast, which is not
exact, with the same context's own output from a run with no other context at work).

Process-wide state the contexts share is the kernels' dynamic shared-memory attribute: the generic patch kernel opts in
to 163,840 bytes at P = 16 gray, 122,880 at P = 16 RGB and 66,560 at P = 10 gray, so a context that set the attribute to
its own launch's size could lower it under another context's launch or captured graph."""
import threading
import time

import numpy as np
import pytest

from of_dis_b200 import params, preprocess, synth
from test_gpu_parity import CASES, assert_bits

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def api():
    from of_dis_b200 import api as _api

    _api.lib()
    return _api


def _cli(numbers, noc=1, nop=2):
    return lambda: params.from_cli_numbers(numbers.split(), noc=noc, nop=nop)


def _case(name, frames, distinct, options=None):
    return CASES[name] + (frames, distinct, options or {})


GENERIC = "3 1 8 8 0.05 0.95 0 %d 0.5 0 1 0 1 10 10 5 1 3 1.6 0"
# name: (h, w, ch, params, amp, stereo, frames per run, distinct pairs (slot f holds pair f % distinct), options)
CONFIGS = {
    # patch_p8c1_kernel with 8 lanes per patch (launches of up to 16 frames); sor_lane_kernel and PDL by default
    "p8_lanes8_op2": _case("cfg2_1024x436_gray_op2", 2, 2),
    # 4 lanes per patch (more than 16 frames); block-wavefront SOR in one CTA, no PDL
    "p8_lanes4_op2": (128, 256, 1, lambda: params.operating_point(2, 256), 6.0, False, 18, 3, {}),
    # patch_p12_kernel: gray stereo (single-CTA SOR), RGB flow (SOR in a cluster)
    "p12_stereo": _case("stereo_op4_small", 2, 2),
    "p12_rgb": _case("rgb_op3_l1cost_small", 2, 2),
    # patch_optimize_kernel<2> at three shared-memory sizes (5 NK threads floats): 163,840, 66,560, 122,880 bytes
    "generic_p16_gray": (200, 320, 1, _cli(GENERIC % 16), 6.0, False, 2, 2, {}),
    "generic_p10_gray": (200, 320, 1, _cli(GENERIC % 10), 6.0, False, 2, 2, {}),
    "generic_p16_rgb": (200, 320, 3, _cli(GENERIC % 16, noc=3), 6.0, False, 2, 2, {}),
    # SOR plans: the lane kernel on four bands, a cluster of 32-lane bands, a chain of bands (P = 6 generic kernel)
    "sor_lane_forced": _case("stereo_sor1_rows100", 2, 2, {"sor_lane": 1}),
    "sor_cluster": _case("gray_sor2_rows70", 2, 2, {"sor_single_max": 32}),
    "sor_chain": _case("gray_p6_nopatnorm_sor5", 2, 2, {"sor_single_max": 32, "sor_max_cluster": 1}),
    # forward-backward consistency (4 internal frames)
    "fbcon": (120, 200, 1, _cli("3 1 8 8 0.05 0.95 0 8 0.4 1 1 0 1 10 10 5 1 3 1.6 0"), 3.0, False, 2, 2, {}),
    # a run from an init flow (level sc_f + 1); RGB P = 8 takes the generic kernel at 122,880 bytes
    "initflow_rgb_p8": (192, 320, 3, _cli("3 1 12 12 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0", noc=3), 6.0, False,
                        2, 2, {}),
    # red-black SOR: checked against its own output from a run with no other context at work
    "sor_fast": (200, 320, 1, _cli("3 1 8 8 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0"), 6.0, False, 2, 2,
                 {"sor_fast": 1}),
}

_INPUTS = {}


def _inputs(name, oracle_port):
    """(params, distinct pyramids, init flows or None, expected flows or None for sor_fast), computed once."""
    if name not in _INPUTS:
        h, w, ch, mk, amp, stereo, _, distinct, opts = CONFIGS[name]
        prm = mk()
        pyrs, inits = [], None
        for s in range(distinct):
            i0, i1, _ = synth.synthetic_pair(h, w, ch, seed=700 + 10 * s, amp=amp, stereo=stereo)
            pyrs.append(preprocess.PairPyramids(i0, i1, prm.sc_f, prm.p_samp_s))
        if name.startswith("initflow"):
            hh, ww = pyrs[0].level_shape(prm.sc_f + 1)
            rng = np.random.default_rng(7)
            inits = [(rng.standard_normal((hh, ww, prm.nop)) * 1.5).astype(np.float32) for _ in range(distinct)]
        exp = None
        if "sor_fast" not in opts:
            exp = [oracle_port.port_run(p, prm, None if inits is None else inits[k]) for k, p in enumerate(pyrs)]
        _INPUTS[name] = (prm, pyrs, inits, exp)
    return _INPUTS[name]


class Lane:
    """One context of a configuration with its slots uploaded; `exp[f % len(exp)]` is slot f's flow."""

    def __init__(self, api, name, oracle_port, stream=None):
        self.name = name
        self.n = CONFIGS[name][6]
        self.prm, pyrs, self.init, self.exp = _inputs(name, oracle_port)
        self.shape = pyrs[0].level_shape(self.prm.sc_l) + (self.prm.nop,)  # of a slot's flow
        self.ctx = api.Context(self.prm, pyrs[0].width, pyrs[0].height, pyrs[0].imgpadding, self.n, stream=stream)
        for k, v in CONFIGS[name][8].items():
            self.ctx.set_option(k, v)
        for f in range(self.n):
            self.ctx.upload_pyramids(f, pyrs[f % len(pyrs)])
            if self.init is not None:
                self.ctx.set_flow(f, self.prm.sc_f + 1, self.init[f % len(pyrs)])

    @property
    def frames(self):  # internal frames of a launch
        return self.n * (2 if self.prm.usefbcon else 1)

    def run(self):
        self.ctx.run(self.n, use_initflow=self.init is not None)

    def flows(self):
        return [self.ctx.get_flow(f, self.prm.sc_l) for f in range(self.n)]

    def check(self, what, flows=None):
        for f, got in enumerate(self.flows() if flows is None else flows):
            assert_bits(got, self.exp[f % len(self.exp)], "%s: %s slot %d" % (what, self.name, f))


def _sor_kinds(api, name, oracle_port):
    """SOR kinds of every level of a configuration under its options (the planner's own answer, no device).
    ofdis_create's default sor_max_cluster is the largest cluster the device grants, 8 or 16: the plans are worked out
    for both and must agree, so that they are the ones the context runs on either kind of device."""
    prm, pyrs = _inputs(name, oracle_port)[:2]
    if not prm.usetvref:
        return set()
    keys = {"sor_lane": "lane", "sor_fast": "fast", "sor_rows_per_thread": "rt", "sor_single_max": "single_max",
            "sor_max_cluster": "max_cluster"}
    frames = CONFIGS[name][6] * (2 if prm.usefbcon else 1)
    plans = []
    for dev_cluster in (8, 16):
        o = dict(lane=2, fast=0, rt=2 if prm.nop == 1 else 1, single_max=128, max_cluster=dev_cluster)  # ofdis_create
        o.update({keys[k]: v for k, v in CONFIGS[name][8].items() if k in keys})
        plans.append([api.debug_sor_plan(w, h, prm.nop, prm.noc, prm.tv_solverit, frames, **o)
                      for h, w in (pyrs[0].level_shape(lv) for lv in range(prm.sc_l, prm.sc_f + 1))])
    assert plans[0] == plans[1], "%s: the SOR plans depend on the device's largest cluster" % name
    return {p["kind"] for p in plans[0]}


def _check_all(lanes, what):
    for lane in lanes.values():
        lane.check(what)


def test_interleaved_contexts_on_one_thread(api, oracle_port):
    """All configurations alive together on their own streams: eager round robin, then the generic patch kernel's
    graph captured at the largest shared-memory size replayed after smaller launches of other contexts, graph
    replays, an option changed between two enqueued replays, and a context destroyed while the others have work in
    flight -- every context's flows after every step."""
    for name in CONFIGS:
        _inputs(name, oracle_port)
    assert set().union(*(_sor_kinds(api, n, oracle_port) for n in CONFIGS)) == set(api.SOR_KINDS)
    fast = Lane(api, "sor_fast", oracle_port)  # its reference: a run while no other context exists
    fast.run()
    fast.exp = fast.flows()
    lanes = {name: Lane(api, name, oracle_port) for name in CONFIGS if name != "sor_fast"}
    lanes["sor_fast"] = fast
    try:
        # eager, round robin; every flow read only after the whole round
        for lane in lanes.values():
            lane.run()
        _check_all(lanes, "eager round")

        # graph of the P = 16 gray context (163,840 bytes), then eager launches of the same kernel at 66,560 and
        # 122,880 bytes from other contexts, then the graph again
        big = lanes["generic_p16_gray"]
        big.ctx.set_graph_mode(True)
        big.run()
        lanes["generic_p10_gray"].run()
        lanes["generic_p16_rgb"].run()
        big.run()
        for name in ("generic_p16_gray", "generic_p10_gray", "generic_p16_rgb"):
            lanes[name].check("P = 16 gray graph replayed after smaller generic launches")

        for lane in lanes.values():
            lane.ctx.set_graph_mode(True)
        for rep in range(2):
            for lane in lanes.values():
                lane.run()
            _check_all(lanes, "graph round %d" % rep)

        # replay, option change (the context's graphs are destroyed while one is in flight), capture and replay
        for lane in lanes.values():
            lane.run()
            lane.ctx.set_option("pdl", 0 if lane.frames <= 16 else 1)
            lane.run()
        _check_all(lanes, "replay, set_option, replay")

        # a context destroyed while every other one has work enqueued, and a new one in its place
        for lane in lanes.values():
            lane.run()
        lanes.pop("p12_rgb").ctx.close()
        fresh = Lane(api, "p12_rgb", oracle_port)
        fresh.ctx.set_graph_mode(True)
        fresh.run()
        lanes["p12_rgb"] = fresh
        _check_all(lanes, "after destroy and create")
    finally:
        for lane in lanes.values():
            lane.ctx.close()


BENCH_LANES, BENCH_DISTINCT = 4, 16
_BENCH = {}


def _bench_lane_inputs(lane, oracle_port):
    """Operating point 2 at 1024 x 436: the lane's own 16 distinct pairs and their oracle flows."""
    if lane not in _BENCH:
        prm = params.operating_point(2, 1024)
        pyrs = []
        for k in range(BENCH_DISTINCT):
            i0, i1, _ = synth.synthetic_pair(436, 1024, 1, seed=800 + BENCH_DISTINCT * lane + k)
            pyrs.append(preprocess.PairPyramids(i0, i1, prm.sc_f, prm.p_samp_s))
        _BENCH[lane] = (prm, pyrs, [oracle_port.port_run(p, prm) for p in pyrs])
    return _BENCH[lane]


@pytest.mark.parametrize("pairs,mixed", [(64, False), (8, False), (64, True), (8, True)],
                         ids=["64_pairs", "8_pairs", "64_pairs_mixed", "8_pairs_mixed"])
def test_overlapping_streams_like_the_benchmark(api, oracle_port, pairs, mixed):
    """bench.py's `value` in miniature: four lanes, each a context on its own torch stream in graph mode, steps dealt
    round robin without a synchronisation between them.  64 pairs per lane (4 lanes per patch, block-wavefront SOR)
    and 8 (8 lanes per patch, sor_lane_kernel, PDL); mixed: one lane's SOR chained, one lane's red-black (sor_fast,
    checked against its own output from before the other lanes ran)."""
    import torch

    inputs = [_bench_lane_inputs(lane, oracle_port) for lane in range(BENCH_LANES)]
    prm = inputs[0][0]
    options = [{}, {"sor_single_max": 32, "sor_max_cluster": 1}, {"sor_fast": 1}, {}] if mixed else [{}] * BENCH_LANES
    streams = [torch.cuda.Stream() for _ in range(BENCH_LANES)]
    ctxs, exp = [], []
    try:
        for lane, (_, pyrs, flows) in enumerate(inputs):
            p0 = pyrs[0]
            ctx = api.Context(prm, p0.width, p0.height, p0.imgpadding, pairs, stream=streams[lane].cuda_stream)
            ctxs.append(ctx)
            for k, v in options[lane].items():
                ctx.set_option(k, v)
            ctx.upload_packed(0, pairs, np.stack([ctx.pack_frame(pyrs[f % BENCH_DISTINCT]) for f in range(pairs)]))
            ctx.set_graph_mode(True)
            if "sor_fast" in options[lane]:
                ctx.run(pairs)
                flows = [ctx.get_flow(f, prm.sc_l) for f in range(pairs)]
            exp.append(flows)
        for step in range(3 * BENCH_LANES):
            ctxs[step % BENCH_LANES].run(pairs)
        for lane, ctx in enumerate(ctxs):
            h, w = inputs[lane][1][0].level_shape(prm.sc_l)
            out = np.empty((pairs, h, w, prm.nop), np.float32)
            ctx.get_flow_batch(0, pairs, out)
            ctx.sync()
            for f in range(pairs):
                assert_bits(out[f], exp[lane][f % len(exp[lane])], "lane %d %s, slot %d" % (lane, options[lane], f))
    finally:
        for ctx in ctxs:
            ctx.close()


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_contexts_sharing_one_caller_stream_with_pdl(api, oracle_port, graph):
    """Three configurations on one torch stream with programmatic dependent launch forced on, run back to back in each
    round with nothing enqueued between them.  Eager, the P = 8 kernel that starts the second and the third context is
    launched as a programmatic dependent of the previous context's last kernel (flow_update_kernel, itself launched
    with the attribute).  After each round every context's flows are copied on the same stream to a torch tensor and
    cloned by torch there -- the first context's after the later contexts' dependent kernels -- so the stream's later
    work must see every context's finished result.  In graph mode each run is its own graph launch, so no programmatic
    edge joins two contexts; that case checks captures and replays of several contexts on one stream."""
    import torch

    names = ["sor_chain", "p8_lanes8_op2", "fbcon"]
    for name in names:
        _inputs(name, oracle_port)
    stream = torch.cuda.Stream()
    lanes = []
    try:
        for name in names:
            lane = Lane(api, name, oracle_port, stream=stream.cuda_stream)
            lane.ctx.set_option("pdl", 1)
            lane.ctx.set_graph_mode(graph)
            lanes.append(lane)
        snaps = []
        with torch.cuda.stream(stream):
            for rep in range(3):
                for lane in lanes:
                    lane.run()
                for lane in lanes:
                    dev = torch.empty((lane.n,) + lane.shape, dtype=torch.float32, device="cuda")
                    lane.ctx.get_flow_batch(0, lane.n, dev.data_ptr(), memkind=api.MEM_DEVICE)
                    snaps.append((lane, rep, dev.clone()))
        stream.synchronize()
        for lane, rep, snap in snaps:
            lane.check("shared stream, %s, round %d" % ("graph" if graph else "eager", rep), list(snap.cpu().numpy()))
    finally:
        for lane in lanes:
            lane.ctx.close()


def test_contexts_driven_from_concurrent_threads(api, oracle_port):
    """Five threads, each with its own context on its own stream (contexts that share a stream are used from one
    thread at a time in graph mode: ofdis_b200.h) -- the generic patch kernel at three shared-memory sizes, a chained
    and a clustered SOR -- start together and run three rounds of an eager run and two graph replays, with one set_option
    after the first round; the main thread compares every flow they read with the oracle.  A fixed, small amount of
    work: this checks results, it does not hunt for a race."""
    names = ["generic_p16_gray", "generic_p10_gray", "generic_p16_rgb", "sor_chain", "sor_cluster"]
    for name in names:
        _inputs(name, oracle_port)
    barrier = threading.Barrier(len(names))
    results, errors = {}, []

    def work(name):
        try:
            lane = Lane(api, name, oracle_port)
            try:
                barrier.wait(timeout=120)
                got = []
                for rnd in range(3):
                    lane.ctx.set_graph_mode(False)
                    lane.run()
                    got.append(("eager, round %d" % rnd, lane.flows()))
                    lane.ctx.set_graph_mode(True)
                    lane.run()
                    lane.run()
                    got.append(("graph, round %d" % rnd, lane.flows()))
                    if rnd == 0:
                        lane.ctx.set_option("pdl", 0)
                results[name] = (lane, got)
            finally:
                lane.ctx.close()
        except BaseException as e:  # noqa: BLE001 -- reported by the main thread
            errors.append("%s: %r" % (name, e))
            barrier.abort()

    threads = [threading.Thread(target=work, args=(name,), name=name, daemon=True) for name in names]
    for t in threads:
        t.start()
    deadline = time.time() + 300
    for t in threads:
        t.join(max(0.0, deadline - time.time()))
    alive = [t.name for t in threads if t.is_alive()]
    if alive:
        pytest.fail("threads still running after 300 s: %s" % ", ".join(alive))
    assert not errors, "; ".join(errors)
    for name in names:
        lane, got = results[name]
        for what, flows in got:
            lane.check("thread " + what, flows)
