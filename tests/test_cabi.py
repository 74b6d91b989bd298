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
