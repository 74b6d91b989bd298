"""ctypes driver for oracle/libdis_oracle.so (the plain-C restatement) --
TEST INFRASTRUCTURE ONLY.  Importable from tests/, smoke() and bench.py's
cpu_baseline leg; never from the product package.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_FP = ctypes.POINTER(ctypes.c_float)
_IP = ctypes.POINTER(ctypes.c_int)
_LIB = None


class CLevel(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in
                ("w", "h", "pad", "tmp_w", "noc", "nop", "P", "steps", "nopw", "noph", "offw", "offh",
                 "level", "camlr")] + [(n, ctypes.c_float) for n in ("lb", "ubw", "ubh", "outlierthresh")]


def build(force: bool = False) -> str:
    so = os.path.join(_HERE, "libdis_oracle.so")
    src = os.path.join(_HERE, "dis_oracle.c")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "port"], stdout=subprocess.DEVNULL)
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = ctypes.CDLL(build())
        _LIB.dis_sum_packet_order.restype = ctypes.c_float
    return _LIB


def _fp(a):
    return a.ctypes.data_as(_FP) if a is not None else None


def make_level(pyr, prm, level: int, camlr: int = 0) -> CLevel:
    L = CLevel()
    cp = prm.to_c()
    lib().dis_make_level(ctypes.byref(L), pyr.width, pyr.height, level, pyr.imgpadding, ctypes.byref(cp),
                         prm.nop, camlr)
    return L


def port_level_patches(pyr, prm, level: int, flow_prev=None, want_dense=True):
    L = make_level(pyr, prm, level)
    cp = prm.to_c()
    n_p = L.nopw * L.noph
    novals = prm.noc * prm.p_samp_s ** 2
    p = np.zeros((n_p, prm.nop), np.float32)
    pw = np.zeros((n_p, novals), np.float32)
    conv = np.zeros(n_p, np.int32)
    cnt = np.zeros(n_p, np.int32)
    if flow_prev is not None:
        flow_prev = np.ascontiguousarray(flow_prev, dtype=np.float32)
    lib().dis_patches_level(ctypes.byref(L), ctypes.byref(cp), _fp(pyr.i0[level]), _fp(pyr.i0x[level]),
                            _fp(pyr.i0y[level]), _fp(pyr.i1[level]), _fp(flow_prev), _fp(p), _fp(pw),
                            conv.ctypes.data_as(_IP), cnt.ctypes.data_as(_IP))
    dense = None
    if want_dense:
        dense = np.zeros((L.h, L.w, prm.nop), np.float32)
        lib().dis_densify(ctypes.byref(L), ctypes.byref(cp), _fp(p), _fp(pw), _fp(dense))
    return dict(p=p, pweight=pw, conv=conv, cnt=cnt, dense=dense, nopw=L.nopw, noph=L.noph)


# bits of dis_patches_level_branches (oracle/dis_oracle.h): the Hessian fallbacks of the patch stage
HESS_SINGULAR_ZERO, HESS_SINGULAR, HESS_NOT_PD, HESS_STEREO_ZERO = 1, 2, 4, 8


def port_level_branches(pyr, prm, level: int) -> np.ndarray:
    """Per patch of the level (ip order), the HESS_* bits of the Hessian fallbacks its template takes."""
    L = make_level(pyr, prm, level)
    cp = prm.to_c()
    out = np.zeros(L.nopw * L.noph, np.int32)
    lib().dis_patches_level_branches(ctypes.byref(L), ctypes.byref(cp), _fp(pyr.i0[level]), _fp(pyr.i0x[level]),
                                     _fp(pyr.i0y[level]), out.ctypes.data_as(_IP))
    return out


def port_densify(pyr, prm, level: int, p, pweight):
    L = make_level(pyr, prm, level)
    cp = prm.to_c()
    dense = np.zeros((L.h, L.w, prm.nop), np.float32)
    p = np.ascontiguousarray(p, np.float32)
    pweight = np.ascontiguousarray(pweight, np.float32)
    lib().dis_densify(ctypes.byref(L), ctypes.byref(cp), _fp(p), _fp(pweight), _fp(dense))
    return dense


def port_level_varref(pyr, prm, level: int, flow: np.ndarray) -> np.ndarray:
    L = make_level(pyr, prm, level)
    cp = prm.to_c()
    out = np.ascontiguousarray(flow, dtype=np.float32).copy()
    lib().dis_varref_level(ctypes.byref(L), ctypes.byref(cp), _fp(pyr.i0[level]), _fp(pyr.i1[level]), _fp(out))
    return out


def _pyr_ptrs(levels):
    arr = (_FP * len(levels))()
    for i, a in enumerate(levels):
        arr[i] = _fp(a)
    return arr


def port_run(pyr, prm, initflow=None) -> np.ndarray:
    h, w = pyr.level_shape(prm.sc_l)
    out = np.zeros((h, w, prm.nop), np.float32)
    cp = prm.to_c()
    rc = lib().dis_run_fb(_pyr_ptrs(pyr.i0), _pyr_ptrs(pyr.i0x), _pyr_ptrs(pyr.i0y), _pyr_ptrs(pyr.i1),
                          _pyr_ptrs(pyr.i1x), _pyr_ptrs(pyr.i1y), pyr.imgpadding, _fp(out), _fp(initflow), pyr.width,
                          pyr.height, ctypes.byref(cp), prm.nop)
    assert rc == 0
    return out


def varref_stages(pyr, prm, level: int, flow: np.ndarray, n_iters=None):
    """Runs the refinement step by step and returns every intermediate plane of
    each inner iteration (for per-kernel parity tests)."""
    L = make_level(pyr, prm, level)
    w, h, C, nop = L.w, L.h, prm.noc, prm.nop
    n = w * h
    f32 = np.float32
    flow = np.ascontiguousarray(flow, f32)
    wx = np.ascontiguousarray(flow[..., 0]).reshape(n).copy()
    wy = np.ascontiguousarray(flow[..., 1]).reshape(n).copy() if nop == 2 else np.zeros(n, f32)
    warped = np.zeros(C * n, f32)
    mask = np.zeros(n, f32)
    lib().dis_warp(ctypes.byref(L), _fp(pyr.i1[level]), _fp(wx), _fp(wy), _fp(warped), _fp(mask))
    D = {k: np.zeros(C * n, f32) for k in ("Ix", "Iy", "Iz", "Ixx", "Ixy", "Iyy", "Ixz", "Iyz")}
    lib().dis_derivatives(ctypes.byref(L), _fp(pyr.i0[level]), _fp(warped), *[_fp(D[k]) for k in
                          ("Ix", "Iy", "Iz", "Ixx", "Ixy", "Iyy", "Ixz", "Iyz")])
    out = dict(warped=warped.reshape(C, h, w), mask=mask.reshape(h, w), iters=[],
               **{k: v.reshape(C, h, w) for k, v in D.items()})
    du, dv = np.zeros(n, f32), np.zeros(n, f32)
    uu, vv = wx.copy(), wy.copy()
    qa = f32(0.25) * f32(prm.tv_alpha)
    hgo3 = f32(prm.tv_gamma) * f32(0.5) / f32(3.0)
    hdo3 = f32(prm.tv_delta) * f32(0.5) / f32(3.0)
    n_inner = prm.tv_innerit * (level + 1) if n_iters is None else n_iters
    cf = ctypes.c_float
    for _ in range(n_inner):
        sh, sv = np.zeros(n, f32), np.zeros(n, f32)
        a11, a12, a22, b1, b2 = (np.zeros(n, f32) for _ in range(5))
        lib().dis_smoothness(w, h, _fp(uu), _fp(vv), cf(qa), _fp(sh), _fp(sv))
        lib().dis_data_term(ctypes.byref(L), _fp(mask), _fp(du), _fp(dv), *[_fp(D[k]) for k in
                            ("Ix", "Iy", "Iz", "Ixx", "Ixy", "Iyy", "Ixz", "Iyz")], cf(hdo3), cf(hgo3),
                            _fp(a11), _fp(a12), _fp(a22), _fp(b1), _fp(b2))
        lib().dis_sub_laplacian(w, h, _fp(b1), _fp(wx), _fp(sh), _fp(sv))
        rec = dict(sh=sh.reshape(h, w).copy(), sv=sv.reshape(h, w).copy(), b1=b1.reshape(h, w).copy(),
                   a11_pre=a11.reshape(h, w).copy(), du_in=du.reshape(h, w).copy(), dv_in=dv.reshape(h, w).copy())
        if nop == 2:
            lib().dis_sub_laplacian(w, h, _fp(b2), _fp(wy), _fp(sh), _fp(sv))
            rec.update(b2=b2.reshape(h, w).copy(), a12_pre=a12.reshape(h, w).copy(), a22_pre=a22.reshape(h, w).copy())
            lib().dis_sor_coupled(w, h, _fp(du), _fp(dv), _fp(a11), _fp(a12), _fp(a22), _fp(b1), _fp(b2),
                                  _fp(sh), _fp(sv), prm.tv_solverit, cf(prm.tv_sor))
            rec.update(a11_inv=a11.reshape(h, w).copy(), a12_inv=a12.reshape(h, w).copy(),
                       a22_inv=a22.reshape(h, w).copy())
            uu = wx + du
            vv = wy + dv
        else:
            lib().dis_sor_de(w, h, _fp(du), _fp(a11), _fp(b1), _fp(sh), _fp(sv), prm.tv_solverit, cf(prm.tv_sor))
            t = wx + du
            uu = np.where(t < 0, t, f32(0)).astype(f32)
        rec.update(du=du.reshape(h, w).copy(), dv=dv.reshape(h, w).copy())
        out["iters"].append(rec)
    out["uu"], out["vv"] = uu.reshape(h, w), vv.reshape(h, w)
    return out
