"""ctypes driver for oracle/_ref/libofdis_ref_*.so -- TEST INFRASTRUCTURE ONLY.

The shared objects are the reference's own sources compiled in place (see
oracle/Makefile); this module only marshals numpy arrays into them.  It may be
imported by tests/, __graft_entry__.smoke() and bench.py's CPU-baseline leg,
never by the product package.
"""
from __future__ import annotations

import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_FP = ctypes.POINTER(ctypes.c_float)
_IP = ctypes.POINTER(ctypes.c_int)
_LIBS = {}


def ref_available(flavour: str = "m1c1") -> bool:
    return os.path.exists(os.path.join(_HERE, "_ref", "libofdis_ref_%s.so" % flavour))


def _lib(flavour: str):
    if flavour not in _LIBS:
        path = os.path.join(_HERE, "_ref", "libofdis_ref_%s.so" % flavour)
        if not os.path.exists(path):
            raise FileNotFoundError("%s missing: run `make -C oracle ref` where the reference sources are (oracle/Makefile REF)" % path)
        # RTLD_LOCAL: the four flavours export the same symbol names.
        _LIBS[flavour] = ctypes.CDLL(path, mode=ctypes.RTLD_LOCAL)
    return _LIBS[flavour]


def _fp(a):
    return a.ctypes.data_as(_FP) if a is not None else None


def _pyr_ptrs(levels):
    arr = (_FP * len(levels))()
    for i, a in enumerate(levels):
        assert a.dtype == np.float32 and a.flags["C_CONTIGUOUS"]
        arr[i] = _fp(a)
    return arr


def ref_run(pyr, prm) -> np.ndarray:
    """OFClass ctor on one pair: returns the flow at level sc_l, (h, w, nop)."""
    lib = _lib(prm.flavour())
    h, w = pyr.level_shape(prm.sc_l)
    out = np.zeros((h, w, prm.nop), dtype=np.float32)
    cp = prm.to_c()
    ptrs = [_pyr_ptrs(x) for x in (pyr.i0, pyr.i0x, pyr.i0y, pyr.i1, pyr.i1x, pyr.i1y)]
    lib.ofdis_ref_run(*ptrs, ctypes.c_int(pyr.imgpadding), _fp(out), None,
                      ctypes.c_int(pyr.width), ctypes.c_int(pyr.height), ctypes.byref(cp))
    return out


def ref_time_run(pyr, prm, reps: int) -> np.ndarray:
    """Per-run wall times (ms) of the OFClass ctor, timed inside the shared object."""
    lib = _lib(prm.flavour())
    h, w = pyr.level_shape(prm.sc_l)
    out = np.zeros((h, w, prm.nop), dtype=np.float32)
    cp = prm.to_c()
    ms = np.zeros(reps, dtype=np.float64)
    ptrs = [_pyr_ptrs(x) for x in (pyr.i0, pyr.i0x, pyr.i0y, pyr.i1, pyr.i1x, pyr.i1y)]
    lib.ofdis_ref_time_run(*ptrs, ctypes.c_int(pyr.imgpadding), _fp(out),
                           ctypes.c_int(pyr.width), ctypes.c_int(pyr.height), ctypes.byref(cp),
                           ctypes.c_int(reps), ms.ctypes.data_as(ctypes.POINTER(ctypes.c_double)))
    return ms


def ref_level_patches(pyr, prm, level: int, flow_prev=None, want_dense: bool = True):
    """PatGridClass at one level.  Returns dict(p, pweight, conv, cnt, dense)."""
    lib = _lib(prm.flavour())
    h, w = pyr.level_shape(level)
    steps = prm.steps
    nopw, noph = -(-w // steps), -(-h // steps)
    n_p = nopw * noph
    novals = prm.noc * prm.p_samp_s ** 2
    p = np.zeros((n_p, prm.nop), np.float32)
    pw = np.zeros((n_p, novals), np.float32)
    conv = np.zeros(n_p, np.int32)
    cnt = np.zeros(n_p, np.int32)
    dense = np.zeros((h, w, prm.nop), np.float32) if want_dense else None
    cp = prm.to_c()
    if flow_prev is not None:
        flow_prev = np.ascontiguousarray(flow_prev, dtype=np.float32)
    lib.ofdis_ref_level_patches.restype = ctypes.c_int
    got = lib.ofdis_ref_level_patches(
        _fp(pyr.i0[level]), _fp(pyr.i0x[level]), _fp(pyr.i0y[level]),
        _fp(pyr.i1[level]), _fp(pyr.i1x[level]), _fp(pyr.i1y[level]),
        ctypes.c_int(pyr.width), ctypes.c_int(pyr.height), ctypes.c_int(level),
        ctypes.c_int(pyr.imgpadding), ctypes.byref(cp), _fp(flow_prev), _fp(p), _fp(pw),
        conv.ctypes.data_as(_IP), cnt.ctypes.data_as(_IP), _fp(dense))
    assert got == n_p, (got, n_p)
    return dict(p=p, pweight=pw, conv=conv, cnt=cnt, dense=dense, nopw=nopw, noph=noph)


def ref_level_varref(pyr, prm, level: int, flow: np.ndarray) -> np.ndarray:
    """VarRefClass at one level; returns the refined copy of `flow` (h, w, nop)."""
    lib = _lib(prm.flavour())
    out = np.ascontiguousarray(flow, dtype=np.float32).copy()
    cp = prm.to_c()
    lib.ofdis_ref_level_varref(
        _fp(pyr.i0[level]), _fp(pyr.i0x[level]), _fp(pyr.i0y[level]),
        _fp(pyr.i1[level]), _fp(pyr.i1x[level]), _fp(pyr.i1y[level]),
        ctypes.c_int(pyr.width), ctypes.c_int(pyr.height), ctypes.c_int(level),
        ctypes.c_int(pyr.imgpadding), ctypes.byref(cp), _fp(out))
    return out


def ref_run_many(pyrs, prm, nrep: int = 1, threads: int = 1):
    """OFClass ctor over `pyrs` x nrep on a native std::thread pool (no Python inside the timed
    region).  Returns (wall seconds, flows [(h, w, nop)] of the last pass)."""
    lib = _lib(prm.flavour())
    h, w = pyrs[0].level_shape(prm.sc_l)
    out = np.zeros((len(pyrs), h, w, prm.nop), dtype=np.float32)
    cp = prm.to_c()
    PP = ctypes.POINTER(_FP)
    tables = []  # keep the per-pair pointer tables alive
    ptrs = (PP * (6 * len(pyrs)))()
    for q, pyr in enumerate(pyrs):
        for k, x in enumerate((pyr.i0, pyr.i0x, pyr.i0y, pyr.i1, pyr.i1x, pyr.i1y)):
            t = _pyr_ptrs(x)
            tables.append(t)
            ptrs[q * 6 + k] = ctypes.cast(t, PP)
    lib.ofdis_ref_run_many.restype = ctypes.c_double
    sec = lib.ofdis_ref_run_many(ptrs, ctypes.c_int(len(pyrs)), ctypes.c_int(nrep), ctypes.c_int(threads),
                                 ctypes.c_int(pyrs[0].imgpadding), _fp(out), ctypes.c_size_t(h * w * prm.nop),
                                 ctypes.c_int(pyrs[0].width), ctypes.c_int(pyrs[0].height), ctypes.byref(cp))
    return float(sec), out


def ref_run_many_u8(frames: np.ndarray, prm, nrep: int = 1, threads: int = 1):
    """8-bit frames [pair][2][h][w][noc] -> full-resolution flow [pair][h][w][nop]: pyramid construction,
    OFClass and the final upsampling/crop per pair on a native thread pool (what one run_OF_INT call
    computes between imread and SaveFlowFile).  Returns (wall seconds, flows)."""
    lib = _lib(prm.flavour())
    frames = np.ascontiguousarray(frames, dtype=np.uint8)
    n, _, h, w = frames.shape[:4]
    out = np.zeros((n, h, w, prm.nop), dtype=np.float32)
    cp = prm.to_c()
    lib.ofdis_ref_run_many_u8.restype = ctypes.c_double
    sec = lib.ofdis_ref_run_many_u8(frames.ctypes.data_as(ctypes.c_void_p), ctypes.c_int(n), ctypes.c_int(nrep),
                                    ctypes.c_int(threads), ctypes.c_int(w), ctypes.c_int(h), _fp(out), ctypes.byref(cp))
    return float(sec), out
