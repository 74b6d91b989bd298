"""Init flow from a full-resolution flow on the device (ofdis_set_initflow_fullres, ofdis_set_initflow_from_result) and
the command lines' `hasinfile infile` and `--warm-start`.  The prepared level sc_f+1 must be BITWISE
preprocess.initflow_from_fullres, and every run from it bitwise the oracle's run from the same init flow."""
import os
import re
import subprocess

import numpy as np
import pytest

from of_dis_b200 import build, params, preprocess, synth
from test_initflow import CASES, fullres_flow, initflow_inputs
from test_sequence_gpu import assert_bits, write_png

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def api():
    from of_dis_b200 import api as _api

    _api.lib()
    return _api


def context(api, prm, h, w, n, div=1):
    s = 1 << (prm.sc_f + div)
    return api.Context(prm, -(-w // s) * s, -(-h // s) * s, prm.p_samp_s, n)


def set_direction(api, ctx, d):
    assert api.lib().ofdis_set_direction(ctx._h, d) == 0


def _status(api, fn, *args):
    try:
        fn(*args)
    except api.OfdisError as e:
        return int(re.match(r"status (-?\d+)", str(e)).group(1))
    return 0


@pytest.mark.parametrize("fb", [0, 1], ids=["fb0", "fb1"])
@pytest.mark.parametrize("nop,ch,sc_f", [(2, 1, 3), (1, 1, 0), (2, 3, 1), (1, 3, 5), (2, 1, 5)])
def test_prepared_level_equals_the_restatement(api, nop, ch, sc_f, fb):
    """Host and device input, f0 > 0, slots outside [f0, f1) untouched, and with usefbcon the backward grid's level
    sc_f+1 zero even after set_direction(1) + set_flow put values there."""
    import torch

    h, w, cap, f0, n = 100, 150, 5, 1, 3
    prm = params.from_cli_numbers(("%d 0 8 8 0.05 0.95 0 8 0.4 %d 1 0 0 10 10 5 1 3 1.6 0" % (sc_f, fb)).split(),
                                  noc=ch, nop=nop)
    ctx = context(api, prm, h, w, cap)
    lv = prm.sc_f + 1
    H, W = ctx.height >> lv, ctx.width >> lv
    junk = np.full((H, W, nop), 7.5, np.float32)
    for f in range(cap):
        ctx.set_flow(f, lv, junk)
        if fb:
            set_direction(api, ctx, 1)
            ctx.set_flow(f, lv, junk)
            set_direction(api, ctx, -1)
    flows = np.stack([fullres_flow(h, w, nop, seed=k) for k in range(n)])
    flows[0, :40, :40] = -0.0  # blocks that sum to -0
    ctx.set_initflow_fullres(f0, f0 + n, flows, w, h)
    for f in range(cap):
        got = ctx.get_flow(f, lv)
        exp = preprocess.initflow_from_fullres(flows[f - f0], prm.sc_f) if f0 <= f < f0 + n else junk
        assert_bits(got, exp, "slot %d" % f)
        if fb:
            set_direction(api, ctx, 1)
            back = ctx.get_flow(f, lv)
            set_direction(api, ctx, -1)
            assert_bits(back, np.zeros_like(junk) if f0 <= f < f0 + n else junk, "backward slot %d" % f)
    dev = torch.from_numpy(flows[::-1].copy()).cuda()
    torch.cuda.synchronize()
    ctx.set_initflow_fullres(f0, f0 + n, dev.data_ptr(), w, h, memkind=api.MEM_DEVICE)
    for k in range(n):
        assert_bits(ctx.get_flow(f0 + k, lv), preprocess.initflow_from_fullres(flows[n - 1 - k], prm.sc_f), "device %d" % k)
    ctx.close()


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("name", list(CASES))
def test_runs_from_the_init_flow_equal_the_oracle(api, oracle_port, name, graph):
    i0, i1, pyr, prm, fl, init = initflow_inputs(name)
    h, w = i0.shape[:2]
    exp = oracle_port.port_run(pyr, prm, init)
    ctx = context(api, prm, h, w, 2)
    ctx.set_graph_mode(graph)
    frames = np.ascontiguousarray(np.stack([np.stack([i0, i1])] * 2))
    for _ in range(2 if graph else 1):  # graph: capture, then replay
        ctx.upload_frames_u8(0, 2, frames, w, h)
        ctx.set_initflow_fullres(0, 2, np.stack([fl, fl]), w, h)
        ctx.run(2, use_initflow=True)
        for f in range(2):
            assert_bits(ctx.get_flow(f, prm.sc_l), exp, "%s pair %d" % (name, f))
    # full resolution: the oracle's flow upsampled and cropped
    out = np.empty((2, h, w, prm.nop), np.float32)
    ctx.get_flow_fullres(0, 2, out, w, h)
    ctx.sync()
    assert_bits(out[1], preprocess.postprocess(exp, prm.sc_l, pyr.padw, pyr.padh, w, h), "fullres")
    ctx.close()


def test_64_pairs_at_operating_point_2(api, oracle_port):
    h, w, n = 436, 1024, 64
    prm = params.operating_point(2, w, noc=1)
    frames = synth.synthetic_sequence(n + 1, h, w, 1, seed=60)
    flows = np.stack([fullres_flow(h, w, 2, seed=k) for k in range(n)])
    ctx = context(api, prm, h, w, n)
    ctx.set_graph_mode(True)
    ctx.upload_sequence_u8(0, n, frames, w, h)
    ctx.set_initflow_fullres(0, n, flows, w, h)
    ctx.run(n, use_initflow=True)
    for t in range(n):
        pyr = preprocess.PairPyramids(frames[t], frames[t + 1], prm.sc_f, prm.p_samp_s, div_level=prm.sc_f + 1)
        init = preprocess.initflow_from_fullres(flows[t], prm.sc_f)
        assert_bits(ctx.get_flow(t, prm.sc_f + 1), init, "init %d" % t)
        assert_bits(ctx.get_flow(t, prm.sc_l), oracle_port.port_run(pyr, prm, init), "pair %d" % t)
    ctx.close()


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("name", ["flow_gray_fb1", "stereo_rgb_fb0", "stereo_gray_s2"])
def test_zero_init_flow_equals_no_init_flow(api, name, graph):
    i0, i1, pyr, prm, fl, init = initflow_inputs(name)
    h, w = i0.shape[:2]
    ctx = context(api, prm, h, w, 1)
    ctx.set_graph_mode(graph)
    frames = np.ascontiguousarray(np.stack([i0, i1])[None])
    res = []
    for use in (False, True, False, True):
        ctx.upload_frames_u8(0, 1, frames, w, h)
        if use:
            ctx.set_initflow_fullres(0, 1, np.zeros_like(fl), w, h)
        ctx.run(1, use_initflow=use)
        res.append(ctx.get_flow(0, prm.sc_l))
    for k in range(1, 4):
        assert_bits(res[k], res[0], "run %d" % k)
    ctx.close()


@pytest.mark.parametrize("fb", [0, 1], ids=["fb0", "fb1"])
@pytest.mark.parametrize("nop,ch", [(2, 1), (1, 3)])
def test_init_flow_from_result_equals_the_composition(api, nop, ch, fb):
    import torch

    h, w, n = 120, 200, 4
    prm = params.from_cli_numbers(("3 1 8 8 0.05 0.95 0 8 0.4 %d 1 0 1 10 10 5 1 3 1.6 0" % fb).split(), noc=ch, nop=nop)
    frames = synth.synthetic_sequence(n + 1, h, w, ch, seed=61, amp=3.0, stereo=(nop == 1))
    a, b = context(api, prm, h, w, n), context(api, prm, h, w, n)
    lv = prm.sc_f + 1
    for ctx in (a, b):
        ctx.upload_sequence_u8(0, n, frames, w, h)
        ctx.run(n)
    for f0, f1, src in ((0, 4, 0), (1, 3, 2), (0, 3, 1), (3, 4, 0)):  # src == dst, src > dst, src < dst
        a.set_initflow_from_result(f0, f1, src, w, h)
        full = torch.empty((f1 - f0, h, w, nop), dtype=torch.float32, device="cuda")
        b.get_flow_fullres(src, src + f1 - f0, full.data_ptr(), w, h, memkind=1)
        b.set_initflow_fullres(f0, f1, full.data_ptr(), w, h, memkind=1)
        b.sync()
        for f in range(n):
            assert_bits(a.get_flow(f, lv), b.get_flow(f, lv), "(%d, %d, %d) slot %d" % (f0, f1, src, f))
            if fb:
                for c in (a, b):
                    set_direction(api, c, 1)
                assert_bits(a.get_flow(f, lv), b.get_flow(f, lv), "backward slot %d" % f)
                for c in (a, b):
                    set_direction(api, c, -1)
    # the warm-started run continues from it like the composition's
    for ctx in (a, b):
        ctx.run(n, use_initflow=True)
    for f in range(n):
        assert_bits(a.get_flow(f, prm.sc_l), b.get_flow(f, prm.sc_l), "run pair %d" % f)
    a.close()
    b.close()


def test_status_codes(api):
    h, w, n = 120, 200, 3
    prm = params.from_cli_numbers("3 1 8 8 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0".split(), noc=1, nop=2)
    ctx = context(api, prm, h, w, n)
    fl = np.zeros((n, h, w, 2), np.float32)
    cases = {"f0 < 0": (-1, 2, w, h), "f1 > max_frames": (0, n + 1, w, h), "f0 == f1": (1, 1, w, h),
             "f0 > f1": (2, 1, w, h), "null": (0, n, w, h), "width": (0, n, w + 17, h), "height": (0, n, w, h - 64)}
    for name, (f0, f1, ww, hh) in cases.items():
        got = _status(api, ctx.set_initflow_fullres, f0, f1, None if name == "null" else fl, ww, hh)
        exp = _status(api, ctx.upload_frames_u8, f0, f1, None if name == "null" else np.zeros((n, 2, h, w), np.uint8),
                      ww, hh)
        assert got == exp == -1, (name, got, exp)
        if name != "null":
            assert _status(api, ctx.set_initflow_from_result, f0, f1, 0, ww, hh) == -1, name
    assert _status(api, ctx.set_initflow_from_result, 0, 2, 2, w, h) == -1  # source past max_frames
    assert _status(api, ctx.set_initflow_from_result, 0, 1, -1, w, h) == -1
    assert _status(api, ctx.set_initflow_fullres, 0, n, fl, w, h) == 0
    ctx.close()
    # a context padded only to 2^sc_f (200 x 120 at sc_f = 3) cannot take an init flow
    ctx = context(api, prm, h, w, n, div=0)
    assert (ctx.width, ctx.height) == (200, 120)
    assert _status(api, ctx.set_initflow_fullres, 0, n, fl, w, h) == -1
    assert _status(api, ctx.set_initflow_from_result, 0, n, 0, w, h) == -1
    ctx.close()
    # the 8-bit uploads and the output stage accept both paddings, and the crop is floor(pad/2) either way
    ctx = context(api, prm, h, w, n)
    assert (ctx.width, ctx.height) == (208, 128)
    assert _status(api, ctx.upload_frames_u8, 0, 1, np.zeros((1, 2, h, w), np.uint8), w, h) == 0
    assert _status(api, ctx.upload_frames_u8, 0, 1, np.zeros((1, 2, 128, 208), np.uint8), 208, 128) == 0
    ctx.close()


# ---- command lines --------------------------------------------------------------------------------------------------
def _write_pair(tmp_path, i0, i1, ch):
    paths = []
    for k, img in enumerate((i0, i1)):
        paths.append(str(tmp_path / ("p%d.png" % k)))
        write_png(paths[-1], img if ch == 1 else img[..., ::-1])  # files store RGB, the pipeline works in BGR
    return paths


def _write_init(path, fl):
    if fl.shape[2] == 2:
        preprocess.write_flo(path, fl)
    else:
        preprocess.write_pfm(path, fl)


@pytest.mark.parametrize("exe,ch,nop,args", [
    ("run_OF_INT", 1, 2, "3 1 12 12 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0"),
    ("run_DE_INT", 1, 1, "3 1 12 12 0.05 0.95 0 8 0.4 1 1 0 1 10 10 5 1 3 1.6 0"),
    ("run_OF_RGB", 3, 2, "2 1 16 16 0.05 0.95 0 12 0.75 1 1 1 1 10 10 5 1 3 1.6 0"),
])
def test_cli_with_infile_writes_the_python_pipelines_bytes(tmp_path, oracle_port, exe, ch, nop, args):
    bindir = build.build_host()
    h, w = 150, 250  # pads differently to 2^lv_f and 2^(lv_f+1)
    i0, i1, _ = synth.synthetic_pair(h, w, ch, seed=62, amp=4.0, stereo=(nop == 1))
    pa, pb = _write_pair(tmp_path, i0, i1, ch)
    fl = fullres_flow(h, w, nop, seed=63)
    ext = "flo" if nop == 2 else "pfm"
    infile = str(tmp_path / ("init." + ext))
    _write_init(infile, fl)
    nums = args.split()
    outs = {}
    for key, extra, env in (("dev", ["1", infile], {}), ("host", ["1", infile], {"OFDIS_HOST_PYRAMID": "1"}),
                            ("plain", [], {}), ("hasinfile0", ["0"], {})):
        outs[key] = str(tmp_path / ("%s.%s" % (key, ext)))
        r = subprocess.run([os.path.join(bindir, exe), pa, pb, outs[key]] + nums + extra, capture_output=True,
                           text=True, env=dict(os.environ, **env))
        assert r.returncode == 0, r.stdout + r.stderr
    data = {k: open(p, "rb").read() for k, p in outs.items()}
    assert data["dev"] == data["host"]
    assert data["hasinfile0"] == data["plain"]
    prm = params.from_cli_numbers(nums, noc=ch, nop=nop)
    pyr = preprocess.PairPyramids(i0, i1, prm.sc_f, prm.p_samp_s, div_level=prm.sc_f + 1)
    init = preprocess.initflow_from_fullres(fl, prm.sc_f)
    exp = preprocess.postprocess(oracle_port.port_run(pyr, prm, init), prm.sc_l, pyr.padw, pyr.padh, w, h)
    ref = str(tmp_path / ("py." + ext))
    _write_init(ref, exp)
    assert data["dev"] == open(ref, "rb").read()
    assert data["dev"] != data["plain"]


@pytest.mark.parametrize("exe,ch,nop,args", [
    # operating point 2 at 500 columns, spelled out: lv_f 4, lv_l 2
    ("run_OF_INT", 1, 2, "4 2 12 12 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 1".split()),
    ("run_DE_RGB", 3, 1, "3 1 8 8 0.05 0.95 0 8 0.4 1 1 0 1 10 10 5 1 3 1.6 1".split()),
])
def test_warm_start_writes_the_files_of_chained_single_pair_calls(tmp_path, exe, ch, nop, args):
    """A 4-frame chain, a 3-frame chain of another size, and a chain that resumes the first clip's size."""
    bindir = build.build_host()
    ext = "flo" if nop == 2 else "pfm"
    clips = []
    for name, n_frames, (h, w), seed in (("a", 4, (218, 500), 64), ("b", 3, (150, 250), 65), ("c", 2, (218, 500), 66)):
        frames = synth.synthetic_sequence(n_frames, h, w, ch, seed=seed, amp=3.0, stereo=(nop == 1))
        paths = []
        for t, img in enumerate(frames):
            paths.append(str(tmp_path / ("%s%d.png" % (name, t))))
            write_png(paths[-1], img if ch == 1 else img[..., ::-1])
        clips.append((paths, h, w))
    pairs = [(p[t], p[t + 1], h, w) for p, h, w in clips for t in range(len(p) - 1)]
    outs = [str(tmp_path / ("warm%d.%s" % (k, ext))) for k in range(len(pairs))]
    lst = tmp_path / "list.txt"
    lst.write_text("".join("%s %s %s\n" % (p, q, o) for (p, q, _, _), o in zip(pairs, outs)))
    r = subprocess.run([os.path.join(bindir, exe + "_batch"), str(lst), "--warm-start"] + args, capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "WARM START (3 of 6 pairs" in r.stdout, r.stdout
    prev = None
    for k, (p, q, h, w) in enumerate(pairs):
        if prev is None or p != pairs[k - 1][1]:  # first pair of a chain: an all-zero init flow
            prev = str(tmp_path / ("zero%d.%s" % (k, ext)))
            _write_init(prev, np.zeros((h, w, nop), np.float32))
        single = outs[k] + ".single"
        r = subprocess.run([os.path.join(bindir, exe), p, q, single] + args + ["1", prev], capture_output=True,
                           text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        assert open(single, "rb").read() == open(outs[k], "rb").read(), k
        prev = single
