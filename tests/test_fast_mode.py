"""The opt-in "fast" refinement (ofdis_set_option "sor_fast": red-black instead of lexicographic SOR, SURVEY 8f
rank 4).  It is NOT bit-identical to the reference and never covered by the parity claim; these tests pin what it
is: (1) exactly a red-black SOR of the same linear system (numpy restatement, bitwise, on a level of several
tiles: the temporal-blocking halo must not show), (2) close to the exact mode and as accurate against the ground
truth of the synthetic pairs, (3) deterministic and off by default."""
import numpy as np
import pytest

from of_dis_b200 import params, preprocess, synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def api():
    from of_dis_b200 import api as _api

    _api.lib()
    return _api


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def redblack_numpy(it, K, omega):
    """K red-black sweeps from du = dv = 0 on the records of one inner iteration (flow)."""
    f32 = np.float32
    a11, a12, a22, b1, b2, sh, sv = (np.asarray(it[k], f32) for k in ("a11_inv", "a12_inv", "a22_inv", "b1", "b2", "sh", "sv"))
    h, w = b1.shape
    shl = np.zeros_like(sh); shl[:, 1:] = sh[:, :-1]
    svt = np.zeros_like(sv); svt[1:, :] = sv[:-1, :]
    yy, xx = np.mgrid[0:h, 0:w]
    du, dv = np.zeros((h, w), f32), np.zeros((h, w), f32)
    om = f32(omega)

    def nb(a):
        l = np.zeros_like(a); l[:, 1:] = a[:, :-1]
        r = np.zeros_like(a); r[:, :-1] = a[:, 1:]
        t = np.zeros_like(a); t[1:, :] = a[:-1, :]
        b = np.zeros_like(a); b[:-1, :] = a[1:, :]
        return l, r, t, b

    for s in range(2 * K):
        m = ((xx + yy) & 1) == (s & 1)
        ul, ur, ut, ub = nb(du)
        vl, vr, vt, vb = nb(dv)
        B1 = b1 + (((shl * ul + sh * ur) + svt * ut) + sv * ub)
        B2 = b2 + (((shl * vl + sh * vr) + svt * vt) + sv * vb)
        nu = du + om * (a11 * B1 + a12 * B2 - du)
        nv = dv + om * (a12 * B1 + a22 * B2 - dv)
        du, dv = np.where(m, nu, du), np.where(m, nv, dv)
    return du, dv


def redblack_stereo_numpy(it, K, omega):
    """K red-black sweeps from du = 0 on the records of one inner iteration (stereo): A11 = a11 + the smoothness
    weights of the pixel's neighbours (solver.c:438-460, summed top, left, bottom, right as assemble_kernel does), then
    du = (1 - omega) du + omega (B1 / A11) on the pixels of one colour (solver.c:458).  Returns (A11, du)."""
    f32 = np.float32
    a11, b1, sh, sv = (np.asarray(it[k], f32) for k in ("a11_pre", "b1", "sh", "sv"))
    h, w = b1.shape
    shl = np.zeros_like(sh); shl[:, 1:] = sh[:, :-1]
    svt = np.zeros_like(sv); svt[1:, :] = sv[:-1, :]
    yy, xx = np.mgrid[0:h, 0:w]
    s = np.zeros((h, w), f32)
    s = np.where(yy > 0, s + svt, s)
    s = np.where(xx > 0, s + shl, s)
    s = np.where(yy < h - 1, s + sv, s)
    s = np.where(xx < w - 1, s + sh, s)
    A11 = a11 + s
    du = np.zeros((h, w), f32)
    om = f32(omega)
    for k in range(2 * K):
        m = ((xx + yy) & 1) == (k & 1)
        ul = np.zeros_like(du); ul[:, 1:] = du[:, :-1]
        ur = np.zeros_like(du); ur[:, :-1] = du[:, 1:]
        ut = np.zeros_like(du); ut[1:, :] = du[:-1, :]
        ub = np.zeros_like(du); ub[:-1, :] = du[1:, :]
        B1 = b1 + (((shl * ul + sh * ur) + svt * ut) + sv * ub)
        du = np.where(m, (f32(1.0) - om) * du + om * (B1 / A11), du)
    return A11, du


def rb_max_sweeps(nop):
    """the largest K whose red-black tile (32 + 2 x 2K pixels square, 7 + 2 planes for flow, 4 + 1 for stereo)
    fits the 227 KB of shared memory a CTA can opt in to on sm_90"""
    K = 1
    while (32 + 4 * (K + 1)) ** 2 * ((7 if nop == 2 else 4) + nop) * 4 <= 227 * 1024:
        K += 1
    return K


# (size, frames, sweeps, rows): assemble_kernel MODE 1 at 1, 2 and 4 rows per thread (2, 8 and 20 frames of the
# 100 x 160 level), and the largest sweep count
RB_CASES = [((200, 320), 2, None, 1), ((200, 320), 8, None, 2), ((200, 320), 20, None, 4), ((200, 320), 2, "max", 1)]


@pytest.mark.parametrize("size,nfr,sweeps,rows", RB_CASES, ids=["rows1", "rows2", "rows4_batch20", "max_sweeps"])
@pytest.mark.parametrize("nop,ch", [(2, 1), (1, 1), (2, 3), (1, 3)], ids=["gray_flow", "gray_stereo", "rgb_flow",
                                                                        "rgb_stereo"])
def test_fast_mode_is_a_red_black_sor_in_every_mode(nop, ch, size, nfr, sweeps, rows, api, oracle_port):
    """sor_redblack_kernel<NOP> and assemble_kernel<C, NOP, R, 1> against the restatements, bitwise: the records
    and (du,dv) after one inner iteration in the last frame of a launch of `nfr` frames; at the largest sweep count
    the halo still fits, and one sweep more is refused."""
    import dataclasses

    prm = params.from_cli_numbers("3 1 8 8 0.05 0.95 0 6 0.5 0 0 0 1 10 10 5 2 5 1.5 0".split(), noc=ch, nop=nop)
    if sweeps == "max":
        prm = dataclasses.replace(prm, tv_solverit=rb_max_sweeps(nop))
    i0, i1, _ = synth.synthetic_pair(size[0], size[1], ch, seed=1, stereo=(nop == 1))
    pyr = preprocess.PairPyramids(i0, i1, prm.sc_f, prm.p_samp_s)
    lv = prm.sc_l
    hh, ww = pyr.level_shape(lv)
    dense = (np.random.default_rng(3).standard_normal((hh, ww, nop)) * 1.5).astype(np.float32)
    if nop == 1:
        dense = -np.abs(dense)
    it = oracle_port.varref_stages(pyr, prm, lv, dense, n_iters=1)["iters"][0]
    K = prm.tv_solverit
    plan = api.debug_sor_plan(ww, hh, nop, ch, K, nfr, fast=1)
    assert plan["kind"] == "redblack" and plan["assemble_mode"] == 1
    assert plan["assemble_rows"] == rows
    ctx = api.Context(prm, pyr.width, pyr.height, pyr.imgpadding, nfr)
    try:
        ctx.set_option("sor_fast", 1)
        for f in range(nfr):
            ctx.upload_pyramids(f, pyr)
        ctx.set_flow(nfr - 1, lv, dense)
        ctx.varref_refine(lv, 0, nfr, n_inner=1)
        rec, dudv = ctx.debug_get("rec", nfr - 1, lv), ctx.debug_get("dudv", nfr - 1, lv)
        if nop == 2:
            for idx, key in enumerate(("a11_inv", "a12_inv", "a22_inv", "b1", "b2", "sh", "sv")):
                assert np.array_equal(bits(rec[..., idx]), bits(it[key])), key
            exp = redblack_numpy(it, K, prm.tv_sor)
        else:
            A11, du = redblack_stereo_numpy(it, K, prm.tv_sor)
            for idx, (key, e) in enumerate((("A11", A11), ("b1", it["b1"]), ("sh", it["sh"]), ("sv", it["sv"]))):
                assert np.array_equal(bits(rec[..., idx]), bits(e)), key
            exp = (du,)
        for c, e in enumerate(exp):
            assert np.array_equal(bits(dudv[..., c]), bits(e)), (c, float(np.abs(dudv[..., c] - e).max()))
        if sweeps == "max":
            assert api.debug_sor_plan(ww, hh, nop, ch, K + 1, nfr, fast=1) is None
            ctx.close()
            ctx = api.Context(dataclasses.replace(prm, tv_solverit=K + 1), pyr.width, pyr.height, pyr.imgpadding, 1)
            with pytest.raises(api.OfdisError, match="status -3"):
                ctx.set_option("sor_fast", 1)
    finally:
        ctx.close()


@pytest.mark.parametrize("size,numbers", [((436, 1024), None), ((200, 320), "3 1 8 8 0.05 0.95 0 6 0.5 0 0 0 1 10 10 5 2 5 1.5 0")])
def test_fast_mode_is_a_red_black_sor_of_the_same_system(size, numbers, api, oracle_port):
    prm = params.operating_point(2, size[1]) if numbers is None else params.from_cli_numbers(numbers.split())
    i0, i1, _ = synth.synthetic_pair(size[0], size[1], 1, seed=1)
    pyr = preprocess.PairPyramids(i0, i1, prm.sc_f, prm.p_samp_s)
    lv = prm.sc_l
    hh, ww = pyr.level_shape(lv)
    rng = np.random.default_rng(3)
    dense = (rng.standard_normal((hh, ww, 2)) * 1.5).astype(np.float32)
    st = oracle_port.varref_stages(pyr, prm, lv, dense, n_iters=1)
    exp_du, exp_dv = redblack_numpy(st["iters"][0], prm.tv_solverit, prm.tv_sor)
    ctx = api.Context(prm, pyr.width, pyr.height, pyr.imgpadding, 2)
    ctx.set_option("sor_fast", 1)
    for f in range(2):
        ctx.upload_pyramids(f, pyr)
        ctx.set_flow(f, lv, dense)
    ctx.varref_refine(lv, 0, 2, n_inner=1)
    rec = ctx.debug_get("rec", 1, lv)
    for idx, key in enumerate(("a11_inv", "a12_inv", "a22_inv", "b1", "b2", "sh", "sv")):
        assert np.array_equal(bits(rec[..., idx]), bits(st["iters"][0][key])), key  # the system itself is the reference's
    dudv = ctx.debug_get("dudv", 1, lv)
    assert np.array_equal(bits(dudv[..., 0]), bits(exp_du)), float(np.abs(dudv[..., 0] - exp_du).max())
    assert np.array_equal(bits(dudv[..., 1]), bits(exp_dv)), float(np.abs(dudv[..., 1] - exp_dv).max())
    ctx.close()


@pytest.mark.parametrize("nop,ch", [(2, 1), (1, 1), (2, 3)])
def test_fast_mode_stays_close_to_the_exact_mode(nop, ch, api):
    prm = params.operating_point(2, 1024, noc=ch, nop=nop)
    errs = {}
    flows = {}
    for fast in (0, 1):
        out = []
        for seed in (5, 6):
            i0, i1, gt = synth.synthetic_pair(436, 1024, ch, seed=seed, stereo=(nop == 1))
            pyr = preprocess.PairPyramids(i0, i1, prm.sc_f, prm.p_samp_s)
            ctx = api.Context(prm, pyr.width, pyr.height, pyr.imgpadding, 1)
            if fast:
                ctx.set_option("sor_fast", 1)
            ctx.upload_pyramids(0, pyr)
            ctx.set_graph_mode(True)
            ctx.run(1)
            ctx.run(1)  # replay must give the same result
            a = ctx.get_flow(0, prm.sc_l)
            ctx.close()
            full = preprocess.postprocess(a, prm.sc_l, pyr.padw, pyr.padh, 1024, 436)
            gtf = gt if nop == 2 else gt[..., :1]
            out.append((full, float(np.sqrt(((full - gtf) ** 2).sum(-1)).mean())))
        flows[fast] = [o[0] for o in out]
        errs[fast] = np.mean([o[1] for o in out])
    delta = np.mean([np.abs(a - b).mean() for a, b in zip(flows[0], flows[1])])
    assert 0 < delta < 0.05, delta            # different iterate, a few hundredths of a pixel (full resolution)
    assert errs[1] < errs[0] * 1.05 + 0.01, errs  # as accurate against the ground truth as the exact mode


def test_fast_mode_is_off_by_default_and_needs_the_refinement(api):
    prm = params.operating_point(1, 1024)  # operating point 1: no refinement
    ctx = api.Context(prm, 1024, 448, 8, 1)
    with pytest.raises(api.OfdisError):
        ctx.set_option("sor_fast", 1)
    ctx.close()
