"""CPU-side checks of the drop-in boundary: the shared library loads without a GPU
and exports every symbol include/ofdis_b200.h declares; argument validation that
does not need a device."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built_lib():
    from of_dis_b200 import build

    return ctypes.CDLL(build.build())


def test_every_declared_symbol_is_exported(built_lib):
    hdr = open(os.path.join(ROOT, "include", "ofdis_b200.h")).read()
    declared = sorted(set(re.findall(r"\b(ofdis_[a-z_0-9]+)\s*\(", hdr)))
    assert len(declared) >= 20
    for name in declared:
        assert hasattr(built_lib, name), name
    from of_dis_b200 import api

    assert sorted(api.EXPORTS) == declared


def test_create_rejects_bad_arguments_without_touching_the_gpu(built_lib):
    from of_dis_b200 import params

    prm = params.operating_point(2, 1024)
    h = ctypes.c_void_p()
    cp = prm.to_c()
    # width not divisible by 2^sc_f (oflow.h:87)
    assert built_lib.ofdis_create(ctypes.byref(h), 0, None, ctypes.byref(cp), 2, 1000, 448, 8, 1) == -1
    # a refinement level taller than the largest SOR cluster can hold (16 bands of ~256 rows): valid in the reference, not built
    assert built_lib.ofdis_create(ctypes.byref(h), 0, None, ctypes.byref(cp), 2, 1024, 131104, 8, 1) == -3
    cp.noc = 2
    assert built_lib.ofdis_create(ctypes.byref(h), 0, None, ctypes.byref(cp), 2, 1024, 448, 8, 1) == -1
    # patches whose generic patch kernel needs more shared memory than a CTA can opt in to (RGB P = 32: 245,760
    # bytes, gray P = 54: 233,600): valid in the reference, not built.  The largest sizes that fit (RGB P = 30, gray
    # P = 52: 216,320 bytes) are accepted: created on a GPU; without one the first CUDA call fails
    for noc, P, refused in ((3, 32, True), (1, 54, True), (3, 30, False), (1, 52, False)):
        cp = params.from_cli_numbers(("2 0 4 4 0.05 0.95 0 %d 0.4 0 1 0 1 10 10 5 1 3 1.6 0" % P).split(), noc=noc).to_c()
        for nop in (1, 2):
            rc = built_lib.ofdis_create(ctypes.byref(h), 0, None, ctypes.byref(cp), nop, 64, 32, P, 1)
            if refused:
                assert rc == -3 and not h.value, (noc, P, nop, rc)
            else:
                assert rc not in (-1, -3), (noc, P, nop, rc)
                built_lib.ofdis_destroy(h)
    assert built_lib.ofdis_destroy(None) == 0


def test_missing_library_fails_loudly(monkeypatch):
    from of_dis_b200 import api

    monkeypatch.setattr(api, "_lib", None)
    monkeypatch.setattr(api, "LIB_PATH", "/nonexistent/libofdis_b200.so")
    with pytest.raises(api.OfdisError):
        api.lib()


def test_reference_arm_prints_the_contract_line(tmp_path):
    """bench.py --impl reference (the reference CPU build, or the oracle port when oracle/_ref is not built)
    prints one JSON line with the keys the driver reads."""
    import json
    import os
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "1",
                        "--batch", "2"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    for key in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
                "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert key in line, key
    assert line["impl"] == "reference" and line["value"] > 0 and line["higher_is_better"] is True
    assert line["e2e"]["h2d_bytes_per_step"] == 0 and line["e2e"]["d2h_bytes_per_step"] == 0
    assert line["cpu_baseline"]["kind"] in ("reference", "port") and line["cpu_baseline"]["cores"] >= 1


# Frames sit in gridDim.y / gridDim.z (at most 65535) of several launches: the derivative kernels take
# max_frames x dirs x noc, the pyramid kernels 2 x max_frames.  Largest accepted max_frames per (noc, usefbcon):
FRAME_BOUNDS = [(1, 0, 32767), (3, 0, 21845), (1, 1, 32767), (3, 1, 10922)]
LIMIT_CLI = "2 0 8 8 0.05 0.95 0 4 0.4 %d 1 0 1 10 10 5 1 3 1.6 0"


@pytest.mark.parametrize("noc,fb,bound", FRAME_BOUNDS)
def test_create_refuses_more_frames_than_a_grid_dimension_holds(noc, fb, bound, built_lib):
    from of_dis_b200 import params

    cp = params.from_cli_numbers((LIMIT_CLI % fb).split(), noc=noc).to_c()
    h = ctypes.c_void_p()
    assert built_lib.ofdis_create(ctypes.byref(h), 0, None, ctypes.byref(cp), 2, 32, 16, 4, bound + 1) == -3
    assert not h.value
    rc = built_lib.ofdis_create(ctypes.byref(h), 0, None, ctypes.byref(cp), 2, 32, 16, 4, bound)
    assert rc != -3  # created on a GPU; without one the first CUDA call fails
    built_lib.ofdis_destroy(h)


def limit_pairs():
    """the 4 distinct 32 x 16 gray pairs of test_largest_frame_count_vs_oracle"""
    from of_dis_b200 import synth

    return [synth.synthetic_pair(16, 32, 1, seed=400 + d, amp=2.0)[:2] for d in range(4)]


@pytest.mark.gpu
def test_largest_frame_count_vs_oracle(oracle_port):
    """The largest gray flow context without usefbcon (32767 pairs of 32 x 16, three levels): the 8-bit upload, the
    run, the batch download and the full-resolution output all take it, and every slot equals the oracle's flow of
    its pair (4 distinct pairs, cycled)."""
    import numpy as np

    from of_dis_b200 import api, params, preprocess

    prm = params.from_cli_numbers((LIMIT_CLI % 0).split())
    n = FRAME_BOUNDS[0][2]
    pairs = limit_pairs()
    pyrs = [preprocess.PairPyramids(a, b, prm.sc_f, prm.p_samp_s) for a, b in pairs]
    exp = np.stack([oracle_port.port_run(p, prm) for p in pyrs])
    full = np.stack([preprocess.postprocess(e, prm.sc_l, p.padw, p.padh, 32, 16) for e, p in zip(exp, pyrs)])
    slots = np.arange(n) % len(pairs)
    frames = np.ascontiguousarray(np.stack([np.stack(pairs[d]) for d in range(len(pairs))])[slots])
    ctx = api.Context(prm, 32, 16, prm.p_samp_s, n)
    try:
        ctx.upload_frames_u8(0, n, frames, 32, 16)
        ctx.run(n)
        out = np.empty((n,) + exp.shape[1:], np.float32)
        ctx.get_flow_batch(0, n, out)
        ctx.sync()
        bad = np.flatnonzero((out.view(np.uint32) != exp[slots].view(np.uint32)).reshape(n, -1).any(1))
        assert bad.size == 0, "%d slots differ from the oracle, first %d" % (bad.size, bad[0])
        fr = np.empty((n,) + full.shape[1:], np.float32)
        ctx.get_flow_fullres(0, n, fr, 32, 16)
        ctx.sync()
        bad = np.flatnonzero((fr.view(np.uint32) != full[slots].view(np.uint32)).reshape(n, -1).any(1))
        assert bad.size == 0, "%d full-resolution slots differ, first %d" % (bad.size, bad[0])
    finally:
        ctx.close()
