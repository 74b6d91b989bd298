"""CPU pins of tests/test_patch_geometry_gpu.py: its cases reach what they claim to reach (every patch kernel at a
padding other than P; every thread count and fold of the generic patch kernel, by generic_launch, which restates the
launcher), the oracle port equals the reference build on every one of its inputs (golden/reference_digests.json, and
the reference build itself where oracle/_ref exists), and the port's results do not depend on the padding."""
import numpy as np
import pytest

from oracle import ref_driver
from test_oracle import REF_DIGESTS, bits, check_inputs, digest, patches_digest
from test_patch_geometry_gpu import (BATCH_FRAMES, PAD_CASES, PAD_IDS, PAD_ROUTES, PADS, SIZE_CASES, UPLOAD_CASES,
                                     batch_inputs, coarser_flow, generic_launch, pad_inputs, patch_kernel, size_inputs,
                                     stage_params, upload_inputs)

SMEM_OPTIN_MAX = 232448  # dynamic shared memory one CTA can opt in to on sm_90 (227 KB)


def test_size_cases_reach_every_generic_launch():
    """Threads per CTA 256, 128, 64 and 32, both residues of noc * P^2 mod 8, and the tail-only fold (nk == 0)."""
    launches = {name: generic_launch(ch, int(numbers.split()[7])) for name, (_, ch, numbers, _) in SIZE_CASES.items()}
    for name, (_, ch, numbers, _) in SIZE_CASES.items():
        assert patch_kernel(ch, int(numbers.split()[7])) == "generic", name
    assert {t for t, _, _, _ in launches.values()} == {256, 128, 64, 32}
    assert {r for _, _, r, _ in launches.values()} == {0, 4}
    assert any(nk == 0 for _, _, _, nk in launches.values())
    # both residues at every thread count but 256, where the residue 0 is gray P = 4 and 16 of the random sweeps
    for t in (256, 128, 64, 32):
        assert {r for tt, _, r, _ in launches.values() if tt == t} == ({4} if t == 256 else {0, 4}), t
    assert max(s for _, s, _, _ in launches.values()) <= SMEM_OPTIN_MAX


def test_largest_patch_sizes_that_fit_the_generic_kernel():
    """RGB P = 30 and gray P = 52 (216,320 bytes at 32 threads) are the largest sizes whose launch fits the opt-in
    ceiling; RGB P = 32 (245,760) and gray P = 54 (233,600) exceed it: ofdis_create refuses those
    (tests/test_cabi.py)."""
    assert generic_launch(3, 30) == (32, 216320, 4, 337) and generic_launch(1, 52) == (32, 216320, 0, 338)
    assert generic_launch(3, 32)[:2] == (32, 245760) and generic_launch(1, 54)[:2] == (32, 233600)
    for noc, largest in ((3, 30), (1, 52)):
        sizes = [P for P in range(2, 80, 2) if (noc * P * P) % 4 == 0 and generic_launch(noc, P)[1] <= SMEM_OPTIN_MAX]
        assert max(sizes) == largest and sizes == list(range(2, largest + 1, 2)), noc


def test_pad_cases_reach_every_patch_kernel_with_usefbcon_and_an_odd_width():
    seen = set()
    for route, (kernel, nop, ch, numbers, opts, (h, w)) in PAD_ROUTES.items():
        P, sc_f, fb = int(numbers.split()[7]), int(numbers.split()[0]), int(numbers.split()[9])
        assert patch_kernel(ch, P) == kernel.split("_")[0], route
        if kernel.startswith("p8c1"):
            assert dict(opts)["patch_lanes"] == int(kernel[-1]), route
        seen.add((kernel, ch if kernel == "p12" else 0, nop, fb))
    kernels = {"p8c1_l8", "p8c1_l4", "p12", "generic"}
    assert {k for k, _, _, _ in seen} == kernels
    assert {(k, c) for k, c, _, _ in seen if k == "p12"} == {("p12", 1), ("p12", 3)}
    assert {k for k, _, _, fb in seen if fb} == kernels  # usefbcon on every kernel
    assert {nop for _, _, nop, _ in seen} == {1, 2}
    assert {PADS[p](8) - 8 for p in PADS} == {1, 2, 3, 8}
    assert any((w >> int(n.split()[0])) % 2 for _, _, _, n, _, (h, w) in PAD_ROUTES.values())


def pad_stage(run, patches, varref, pyr, prm):
    """the GPU checks of a padding case with one driver: whole run, patch stage at sc_l from coarser_flow, the
    refinement of sc_l from its dense flow"""
    sprm = stage_params(prm)
    lvl = patches(pyr, sprm, prm.sc_l, coarser_flow(pyr, prm))
    return run(pyr, prm), lvl, varref(pyr, sprm, prm.sc_l, lvl["dense"])


@pytest.mark.parametrize("route,pad", PAD_CASES, ids=PAD_IDS)
def test_port_vs_reference_at_wider_paddings(route, pad, oracle_port):
    i0, i1, pyr, _, prm = pad_inputs(route, pad)
    key = "geometry_pad_%s_%s" % (route, pad)
    check_inputs(key, i0, i1)
    run, lvl, vr = pad_stage(oracle_port.port_run, oracle_port.port_level_patches, oracle_port.port_level_varref,
                              pyr, prm)
    assert digest(run) == REF_DIGESTS[key + "_run"]
    assert patches_digest([lvl]) == REF_DIGESTS[key + "_patches"]
    assert digest(vr) == REF_DIGESTS[key + "_varref"]
    if ref_driver.ref_available(prm.flavour()):
        assert np.array_equal(bits(ref_driver.ref_run(pyr, prm)), bits(run))


@pytest.mark.parametrize("route", list(PAD_ROUTES))
def test_port_is_invariant_under_the_padding(route, oracle_port):
    """The flow, the patch stage and the refinement at paddings P+1, P+3 and 2P are bitwise those at padding P."""
    _, _, _, pyr_p, prm = pad_inputs(route, "P+1")
    ref = pad_stage(oracle_port.port_run, oracle_port.port_level_patches, oracle_port.port_level_varref, pyr_p, prm)
    for pad in ("P+1", "P+3", "2P"):
        pyr = pad_inputs(route, pad)[2]
        assert pyr.imgpadding > prm.p_samp_s
        got = pad_stage(oracle_port.port_run, oracle_port.port_level_patches, oracle_port.port_level_varref, pyr, prm)
        assert np.array_equal(bits(got[0]), bits(ref[0])), (pad, "run")
        assert patches_digest([got[1]]) == patches_digest([ref[1]]), (pad, "patches")
        assert np.array_equal(bits(got[2]), bits(ref[2])), (pad, "varref")


def size_stage(run, patches, pyr, prm):
    return run(pyr, prm), patches(pyr, stage_params(prm), prm.sc_l, coarser_flow(pyr, prm))


@pytest.mark.parametrize("name", list(SIZE_CASES))
def test_port_vs_reference_at_patch_sizes(name, oracle_port):
    i0, i1, pyr, prm = size_inputs(name)
    key = "geometry_size_%s" % name
    check_inputs(key, i0, i1)
    run, lvl = size_stage(oracle_port.port_run, oracle_port.port_level_patches, pyr, prm)
    assert digest(run) == REF_DIGESTS[key + "_run"]
    assert patches_digest([lvl]) == REF_DIGESTS[key + "_patches"]
    if ref_driver.ref_available(prm.flavour()):
        assert np.array_equal(bits(ref_driver.ref_run(pyr, prm)), bits(run))


def upload_digests(run, name):
    """digest of the clip, and one digest over the runs of its forward and (flow only) backward pairs"""
    prm, _, frames, fwd, bwd = upload_inputs(name)
    pyrs = fwd + (bwd if prm.nop == 2 else [])
    return digest(frames, np.uint8), digest(np.stack([run(p, prm) for p in pyrs]))


def batch_digests(run):
    prm, pairs, pyrs = batch_inputs()
    return digest(np.stack([np.stack(p) for p in pairs]), np.uint8), digest(np.stack([run(p, prm) for p in pyrs]))


@pytest.mark.parametrize("name", list(UPLOAD_CASES))
def test_port_vs_reference_on_the_upload_clips(name, oracle_port):
    inp, runs = upload_digests(oracle_port.port_run, name)
    assert inp == REF_DIGESTS["geometry_upload_%s_input" % name], "%s: synthetic inputs differ from the recorded ones" % name
    assert runs == REF_DIGESTS["geometry_upload_%s_runs" % name]


def test_port_vs_reference_on_the_batch_pairs(oracle_port):
    assert BATCH_FRAMES > 16
    inp, runs = batch_digests(oracle_port.port_run)
    assert inp == REF_DIGESTS["geometry_batch_input"], "synthetic inputs differ from the recorded ones"
    assert runs == REF_DIGESTS["geometry_batch_runs"]
