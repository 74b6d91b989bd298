"""Run parameters of the DIS hot path: the reference's 20 positional CLI numbers
and its four operating-point presets.

Mirrors run_dense.cpp:225-294 (argument grammar, presets) and
run_dense.cpp:180-183 (AutoFirstScaleSelect).  Field names follow
oflow.h:31-76 (optparam).
"""
from __future__ import annotations

import ctypes
import dataclasses
import math


class CParams(ctypes.Structure):
    """Binary layout shared by include/ofdis_b200.h (ofdis_params) and
    oracle/ref_wrapper.cpp (ofdis_ref_params)."""

    _fields_ = [
        ("sc_f", ctypes.c_int), ("sc_l", ctypes.c_int),
        ("max_iter", ctypes.c_int), ("min_iter", ctypes.c_int),
        ("dp_thresh", ctypes.c_float), ("dr_thresh", ctypes.c_float), ("res_thresh", ctypes.c_float),
        ("p_samp_s", ctypes.c_int), ("patove", ctypes.c_float),
        ("usefbcon", ctypes.c_int), ("costfct", ctypes.c_int), ("noc", ctypes.c_int),
        ("patnorm", ctypes.c_int), ("usetvref", ctypes.c_int),
        ("tv_alpha", ctypes.c_float), ("tv_gamma", ctypes.c_float), ("tv_delta", ctypes.c_float),
        ("tv_innerit", ctypes.c_int), ("tv_solverit", ctypes.c_int), ("tv_sor", ctypes.c_float),
        ("verbosity", ctypes.c_int),
    ]


@dataclasses.dataclass
class DisParams:
    sc_f: int
    sc_l: int
    max_iter: int = 12
    min_iter: int = 12
    dp_thresh: float = 0.05
    dr_thresh: float = 0.95
    res_thresh: float = 0.0
    p_samp_s: int = 8
    patove: float = 0.4
    usefbcon: int = 0
    costfct: int = 0
    noc: int = 1
    patnorm: int = 1
    usetvref: int = 1
    tv_alpha: float = 10.0
    tv_gamma: float = 10.0
    tv_delta: float = 5.0
    tv_innerit: int = 1
    tv_solverit: int = 3
    tv_sor: float = 1.6
    verbosity: int = 0
    nop: int = 2  # 2 = optical flow (SELECTMODE 1), 1 = stereo depth (SELECTMODE 2)

    def to_c(self) -> CParams:
        c = CParams()
        for name, _ in CParams._fields_:
            setattr(c, name, getattr(self, name))
        return c

    @property
    def steps(self) -> int:
        """oflow.cpp:91 -- float arithmetic on purpose (0.4f etc.)."""
        import numpy as np

        return max(1, int(math.floor(np.float32(self.p_samp_s) * (np.float32(1) - np.float32(self.patove)))))

    @property
    def mode(self) -> int:
        return 1 if self.nop == 2 else 2

    def flavour(self) -> str:
        return "m%dc%d" % (self.mode, self.noc)


def auto_first_scale(imgwidth: int, fratio: int, patchsize: int) -> int:
    """run_dense.cpp:180-183."""
    return max(0, int(math.floor(math.log2((2.0 * imgwidth) / (float(fratio) * float(patchsize))))))


def operating_point(op: int, width_org: int, noc: int = 1, nop: int = 2, verbosity: int = 0) -> DisParams:
    """run_dense.cpp:225-268: presets selected by one digit (default 2)."""
    fratio = 5
    if op == 1:
        patchsz, poverl, dl, it, tv = 8, 0.3, 2, 16, 0
    elif op == 3:
        patchsz, poverl, dl, it, tv = 12, 0.75, 4, 16, 1
    elif op == 4:
        patchsz, poverl, dl, it, tv = 12, 0.75, 5, 128, 1
    else:
        patchsz, poverl, dl, it, tv = 8, 0.4, 2, 12, 1
    lv_f = auto_first_scale(width_org, fratio, patchsz)
    lv_l = max(lv_f - dl, 0)
    return DisParams(sc_f=lv_f, sc_l=lv_l, max_iter=it, min_iter=it, p_samp_s=patchsz, patove=poverl,
                     usetvref=tv, noc=noc, nop=nop, verbosity=verbosity)


def from_cli_numbers(vals, noc: int = 1, nop: int = 2) -> DisParams:
    """run_dense.cpp:269-294: the 20-number explicit form, in CLI order
    (note: CLI order is patnorm, costfct; the class API order is costfct, noc, patnorm)."""
    v = list(vals)
    if len(v) != 20:
        raise ValueError("need exactly 20 numbers (README.md:66-88)")
    return DisParams(sc_f=int(v[0]), sc_l=int(v[1]), max_iter=int(v[2]), min_iter=int(v[3]),
                     dp_thresh=float(v[4]), dr_thresh=float(v[5]), res_thresh=float(v[6]),
                     p_samp_s=int(v[7]), patove=float(v[8]), usefbcon=int(v[9]), patnorm=int(v[10]),
                     costfct=int(v[11]), usetvref=int(v[12]), tv_alpha=float(v[13]), tv_gamma=float(v[14]),
                     tv_delta=float(v[15]), tv_innerit=int(v[16]), tv_solverit=int(v[17]),
                     tv_sor=float(v[18]), verbosity=int(v[19]), noc=noc, nop=nop)
