"""Fits a Fisher-vector codebook on the device from the batch command's descriptor file.

    python -m of_dis_b200.fisher_fit DESCFILE OUT [--k 256] [--samples 256000] [--iters 10] [--seed 0]
                                     [--var-floor 1e-3]

DESCFILE is what `run_OF_*_batch --tracks ... --descriptors DESCFILE` writes: a header line, then per segment `clip id
start mean_x mean_y sd_x sd_y length` and the IDT defaults' 426 floats.  Every ceil(n / samples)-th segment is a
sample; the blocks are IDT's (shape, HOG, HOF, MBHx, MBHy) with dim_in // 2 PCA outputs each.  The E-step runs on
the device (Context.fisher_fit; there is no CPU fallback) and OUT gets the codebook file that
preprocess.read_fisher_codebook and ofdis_fisher_begin read."""
from __future__ import annotations

import argparse
import sys

import numpy as np

from . import params, preprocess as pp

RECORD_COLUMNS = 8  # clip id start mean_x mean_y sd_x sd_y length


def read_samples(path: str, samples: int) -> np.ndarray:
    dim = pp.traj_dim(pp.TRAJ_DEFAULTS)
    with open(path) as f:
        lines = f.read().splitlines()[1:]
    lines = [ln for ln in lines if ln.strip()]
    step = max(1, -(-len(lines) // max(1, samples)))
    rows = [np.array(ln.split()[RECORD_COLUMNS:], np.float32) for ln in lines[::step]]
    if not rows or any(r.size != dim for r in rows):
        raise ValueError("%s: expected lines of %d + %d columns" % (path, RECORD_COLUMNS, dim))
    return np.stack(rows)


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(prog="python -m of_dis_b200.fisher_fit", description=__doc__.splitlines()[0])
    ap.add_argument("descfile")
    ap.add_argument("out")
    ap.add_argument("--k", type=int, default=256)
    ap.add_argument("--samples", type=int, default=256000)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--var-floor", type=float, default=1e-3)
    a = ap.parse_args(argv)
    x = read_samples(a.descfile, a.samples)
    blocks = pp.fisher_blocks(pp.TRAJ_DEFAULTS)
    from . import api

    prm = params.from_cli_numbers("3 1 8 8 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0".split(), noc=1, nop=2)
    ctx = api.Context(prm, 64, 64, prm.p_samp_s, 1)  # the encoder reads no flow: the smallest context serves
    try:
        cb = ctx.fisher_fit(x, blocks, [di // 2 for _, di in blocks], a.k, a.iters, a.seed, a.var_floor)
    finally:
        ctx.close()
    pp.write_fisher_codebook(a.out, cb)
    print("fisher_fit: %d samples, K %d, %d iterations -> %s" % (x.shape[0], a.k, a.iters, a.out))
    return 0


if __name__ == "__main__":
    sys.exit(main())
