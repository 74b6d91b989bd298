"""Fisher vectors on the device: ofdis_fisher_begin / ofdis_fisher_push / ofdis_fisher_take.  Every vector float,
statistic and counter must be BITWISE what preprocess.FisherStream gives on the same descriptors, whatever the pushes,
memory kinds and streams, and the device fit must return preprocess.fisher_fit's codebook bytes."""
import ctypes
import math

import numpy as np
import pytest

from of_dis_b200 import params, preprocess as pp, synth

pytestmark = pytest.mark.gpu

f32 = np.float32
CHUNK = 4096  # FISHER_CHUNK: descriptors per internal chunk of a push
IDT = pp.TRAJ_DEFAULTS
IDT_DIM = pp.traj_dim(IDT)


@pytest.fixture(scope="module")
def api():
    from of_dis_b200 import api as _api

    _api.lib()
    return _api


def context(api, stream=None):
    prm = params.from_cli_numbers("3 1 8 8 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0".split(), noc=1, nop=2)
    return api.Context(prm, 64, 64, prm.p_samp_s, 2, stream=stream)


def random_codebook(rng, K, blocks, desc_dim):
    cb = {"K": K, "desc_dim": desc_dim, "blocks": blocks}
    for k in pp.FISHER_PARTS:
        cb[k] = []
    for _, di, d in blocks:
        w = rng.uniform(0.2, 1.0, K)
        w /= w.sum()
        sig = rng.uniform(0.3, 1.5, (K, d))
        cb["mean"].append(rng.normal(0, 0.1, di).astype(f32))
        cb["proj"].append(rng.normal(0, 1.0 / math.sqrt(di), (d, di)).astype(f32))
        cb["mu"].append(rng.normal(0, 0.3, (K, d)).astype(f32))
        cb["isig"].append((1.0 / sig).astype(f32))
        cb["c"].append((np.log(w) - np.log(sig).sum(1)).astype(f32))
        cb["w"].append(w.astype(f32))
    return cb


def idt_codebook(rng, K):
    return random_codebook(rng, K, [(o, di, di // 2) for o, di in pp.fisher_blocks(IDT)], IDT_DIM)


def same(a, b):
    a, b = np.atleast_1d(a), np.atleast_1d(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def assert_take(got, exp, name=""):
    assert same(got[0], exp[0]), "%s: vector differs" % name
    assert same(got[1], exp[1]), "%s: statistics differ" % name
    assert got[2]["pushed"] == exp[2]["pushed"], name
    assert np.array_equal(got[2]["n"], exp[2]["n"]), (name, got[2]["n"], exp[2]["n"])
    assert np.array_equal(got[2]["skipped"], exp[2]["skipped"]), name


def descriptors(rng, n, dim, bad=True):
    x = np.abs(rng.normal(0, 0.3, (n, dim))).astype(f32)
    if bad and n > 10:
        x[3, 40] = np.nan
        x[5, 200] = np.inf
        x[7, 1] = -np.inf
        x[9, 300] = 3e38
    return x


CASES = [  # K, n
    (256, CHUNK + 37),
    (8, 2 * CHUNK + 1),
    (1, 500),
]


@pytest.mark.parametrize("K,n", CASES, ids=["K%d-n%d" % c for c in CASES])
def test_idt_blocks_equal_the_restatement(K, n, api):
    rng = np.random.default_rng(K + n)
    cb = idt_codebook(rng, K)
    x = descriptors(rng, n, IDT_DIM)
    exp = pp.fisher_encode(x, cb)
    ctx = context(api)
    ctx.fisher_begin(cb)
    before = ctx.launch_count
    ctx.fisher_push(x)
    assert ctx.launch_count - before == 3 * ((n + CHUNK - 1) // CHUNK)
    before = ctx.launch_count
    got = ctx.fisher_take()
    assert ctx.launch_count - before == 1
    assert_take(got, exp, "one push")
    assert got[0].size == 2 * K * 213
    # many pushes across the chunk boundary, n = 0 and n = 1 among them
    cuts = [0, 1, 1, 2, CHUNK - 1, CHUNK + 5, n]
    for a, b in zip(cuts[:-1], cuts[1:]):
        ctx.fisher_push(x[a:b])
    assert_take(ctx.fisher_take(), exp, "many pushes")
    ctx.close()


def test_odd_blocks_and_dims(api):
    """K = 3, dim = dim_in, dim = 1, overlapping blocks, the largest dim_in."""
    rng = np.random.default_rng(4)
    blocks = [(0, 7, 7), (3, 5, 1), (10, 512, 33), (0, 1, 1)]
    cb = random_codebook(rng, 3, blocks, 600)
    x = rng.normal(0, 1.0, (300, 600)).astype(f32)
    x[10, 4] = np.nan
    ctx = context(api)
    ctx.fisher_begin(cb)
    ctx.fisher_push(x)
    assert_take(ctx.fisher_take(), pp.fisher_encode(x, cb))
    ctx.close()


def test_device_memory_on_a_caller_stream(api):
    import torch

    rng = np.random.default_rng(8)
    cb = idt_codebook(rng, 16)
    x = descriptors(rng, CHUNK + 100, IDT_DIM)
    exp = pp.fisher_encode(x, cb)
    sz = pp.fisher_sizes(16, cb["blocks"])
    stream = torch.cuda.Stream()
    ctx = context(api, stream=stream.cuda_stream)
    dx = torch.from_numpy(x).cuda()
    fv = torch.full((sz["fv"],), -7.0, dtype=torch.float32, device="cuda")
    st = torch.full((sz["stats"],), -7.0, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    ctx.fisher_begin(cb)
    ctx.fisher_push(dx[:100].data_ptr(), memkind=api.MEM_DEVICE, n=100)
    ctx.fisher_push(dx[100:].data_ptr(), memkind=api.MEM_DEVICE, n=CHUNK)
    cnt = ctx.fisher_take(memkind=api.MEM_DEVICE, fv=fv.data_ptr(), stats=st.data_ptr())
    stream.synchronize()
    assert_take((fv.cpu().numpy(), st.cpu().numpy(), cnt), exp, "device")
    # host output on the same stream, the vector alone, then the statistics alone
    ctx.fisher_push(x)
    got_fv, got_st, cnt = ctx.fisher_take(with_stats=False)
    assert got_st is None and same(got_fv, exp[0]) and cnt["pushed"] == x.shape[0]
    ctx.fisher_push(x)
    got_fv, got_st, _ = ctx.fisher_take(with_fv=False)
    assert got_fv is None and same(got_st, exp[1])
    ctx.close()


def test_clips_begin_and_other_stages(api):
    """A second clip after a take, a run between calls (its flows unchanged by the encoder), and a begin that resets a
    live encoder with half a clip in it."""
    rng = np.random.default_rng(12)
    cb = idt_codebook(rng, 4)
    a, b = descriptors(rng, 700, IDT_DIM), descriptors(rng, 300, IDT_DIM, bad=False)
    ctx = context(api)
    pair = synth.synthetic_sequence(2, 64, 64, 1, seed=2, amp=3.0)
    ctx.upload_frames_u8(0, 1, np.ascontiguousarray(pair[None]), 64, 64)
    ctx.run(1)
    flow0 = np.empty((1, 64, 64, 2), f32)
    ctx.get_flow_fullres(0, 1, flow0, 64, 64)
    ctx.fisher_begin(cb)
    ctx.fisher_push(a[:300])
    ctx.run(1)
    ctx.fisher_push(a[300:])
    assert_take(ctx.fisher_take(), pp.fisher_encode(a, cb), "clip a")
    ctx.fisher_push(b)
    assert_take(ctx.fisher_take(), pp.fisher_encode(b, cb), "clip b")
    ctx.fisher_push(a)
    cb2 = idt_codebook(rng, 6)
    ctx.fisher_begin(cb2)
    ctx.fisher_push(b)
    assert_take(ctx.fisher_take(), pp.fisher_encode(b, cb2), "after a second begin")
    flow1 = np.empty_like(flow0)
    ctx.get_flow_fullres(0, 1, flow1, 64, 64)
    assert same(flow0, flow1)
    ctx.close()


def test_descriptors_of_traj_advance(api):
    """The descriptor stage's output on gray and RGB clips, taken from the host and straight from a device buffer;
    the tracks and descriptors stay what the stage gives without the encoder."""
    import torch

    for ch in (1, 3):
        h, w, n = 96, 128, 2 * IDT["L"] + 2
        prm = params.from_cli_numbers("3 1 8 8 0.05 0.95 0 8 0.4 0 1 0 1 10 10 5 1 3 1.6 0".split(), noc=ch, nop=2)
        clip = synth.synthetic_sequence(n + 1, h, w, ch, seed=21 + ch, amp=3.0)
        ctx = api.Context(prm, w, h, prm.p_samp_s, 2 * n)
        ctx.upload_sequence_bidir_u8(0, n, clip, w, h)
        ctx.run(2 * n)
        tpp = dict(capacity=4000, spacing=6, alpha=0.01, beta=0.5, mb_alpha=0.01, mb_beta=0.002, min_eig=25.0)
        ctx.traj_begin(tpp, IDT, clip[0], w, h)
        _, _, desc, n_desc = ctx.traj_advance(0, n, n, clip[1:], w, h)
        assert desc.shape[0] > 0
        rng = np.random.default_rng(ch)
        cb = idt_codebook(rng, 32)
        exp = pp.fisher_encode(desc, cb)
        ctx.fisher_begin(cb)
        ctx.fisher_push(desc)
        assert_take(ctx.fisher_take(), exp, "host, %d channels" % ch)
        # the same clip with the descriptors left in device memory
        bound = pp.traj_bound(tpp["capacity"], n, IDT["L"])
        dclip = torch.from_numpy(clip.reshape(-1)).cuda()
        pts = torch.empty((n * tpp["capacity"] * 3,), dtype=torch.int32, device="cuda")
        rec = torch.empty((bound * 7,), dtype=torch.int32, device="cuda")
        ddesc = torch.empty((bound * IDT_DIM,), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        hwc = h * w * ch
        ctx.traj_begin(tpp, IDT, dclip.data_ptr(), w, h, memkind=api.MEM_DEVICE, points=pts.data_ptr())
        _, nd = ctx.traj_advance(0, n, n, dclip.data_ptr() + hwc, w, h, frame_stride=hwc, memkind=api.MEM_DEVICE,
                                 points=pts.data_ptr(), records=rec.data_ptr(), desc=ddesc.data_ptr())
        assert np.array_equal(nd, n_desc)
        ctx.fisher_push(ddesc.data_ptr(), memkind=api.MEM_DEVICE, n=int(nd.sum()))
        assert_take(ctx.fisher_take(), exp, "device, %d channels" % ch)
        got = ddesc[:int(nd.sum()) * IDT_DIM].cpu().numpy().reshape(-1, IDT_DIM)
        assert same(got, desc)
        ctx.close()


def test_fit_on_the_device_equals_the_restatement(api):
    rng = np.random.default_rng(6)
    centres = rng.normal(0, 2.0, (8, IDT_DIM))
    x = np.abs(centres[rng.integers(0, 8, 3000)] + rng.normal(0, 0.3, (3000, IDT_DIM))).astype(f32)
    blocks = pp.fisher_blocks(IDT)
    dims = [di // 2 for _, di in blocks]
    exp = pp.fisher_fit(x, blocks, dims, K=8, iters=3, seed=1)
    ctx = context(api)
    got = ctx.fisher_fit(x, blocks, dims, K=8, iters=3, seed=1)
    assert same(pp.fisher_pack(got), pp.fisher_pack(exp))
    ctx.close()


def test_bad_arguments(api):
    import torch

    rng = np.random.default_rng(1)
    cb = random_codebook(rng, 2, [(0, 4, 2)], 6)
    ctx = context(api)
    L = api.lib()
    body = np.ascontiguousarray(pp.fisher_pack(cb))
    x = rng.normal(0, 1, (5, 6)).astype(f32)
    # no live encoder yet
    assert L.ofdis_fisher_push(ctx._h, api._ptr(x), 5, api.MEM_HOST) == -1
    assert L.ofdis_fisher_take(ctx._h, None, None, None, api.MEM_HOST) == -1

    def begin(**kw):
        c = api.FisherCodebook()
        c.K, c.desc_dim, c.nblocks = kw.get("K", 2), kw.get("desc_dim", 6), kw.get("nblocks", 1)
        c.blocks[0] = api.FisherBlock(*kw.get("block", (0, 4, 2)))
        p = kw.get("body", body)
        c.params = None if p is None else p.ctypes.data
        return L.ofdis_fisher_begin(ctx._h, ctypes.byref(c))

    assert begin() == 0
    assert L.ofdis_fisher_begin(ctx._h, None) == -1
    for kw in (dict(K=0), dict(K=257), dict(nblocks=0), dict(nblocks=9), dict(desc_dim=0), dict(block=(0, 4, 5)),
               dict(block=(0, 0, 0)), dict(block=(3, 4, 2)), dict(block=(-1, 4, 2)), dict(block=(0, 513, 2)),
               dict(body=None)):
        assert begin(**kw) == -1, kw
    for part, val in (("isig", 0.0), ("isig", -1.0), ("w", 0.0), ("c", np.inf), ("mu", np.nan), ("proj", np.inf),
                      ("mean", np.nan), ("isig", np.inf), ("w", np.nan)):
        bad = dict(cb, **{k: [a.copy() for a in cb[k]] for k in pp.FISHER_PARTS})
        bad[part][0].flat[0] = val
        assert begin(body=np.ascontiguousarray(pp.fisher_pack(bad))) == -1, part
    # a refused begin leaves the live encoder as it was
    ctx.fisher_begin(cb)
    ctx.fisher_push(x[:2])
    assert begin(K=0) == -1
    ctx.fisher_push(x[2:])
    assert_take(ctx.fisher_take(), pp.fisher_encode(x, cb))
    dev = torch.zeros((64,), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    assert L.ofdis_fisher_push(ctx._h, None, 1, api.MEM_HOST) == -1
    assert L.ofdis_fisher_push(ctx._h, api._ptr(x), -1, api.MEM_HOST) == -1
    assert L.ofdis_fisher_push(ctx._h, ctypes.c_void_p(dev.data_ptr() + 2), 1, api.MEM_DEVICE) == -1
    assert L.ofdis_fisher_push(ctx._h, None, 0, api.MEM_HOST) == 0
    assert L.ofdis_fisher_take(ctx._h, ctypes.c_void_p(dev.data_ptr() + 2), None, None, api.MEM_DEVICE) == -1
    assert L.ofdis_fisher_take(ctx._h, None, ctypes.c_void_p(dev.data_ptr() + 4), None, api.MEM_DEVICE) == -1
    # the encoder is still live and empty after the refusals
    ctx.fisher_push(x)
    assert_take(ctx.fisher_take(), pp.fisher_encode(x, cb))
    ctx.close()


def _read_fisher(path, nblocks):
    lines = open(path).read().splitlines()
    assert lines[0].startswith("# clip n_desc n_0 .. n_%d fv0 .. fv" % (nblocks - 1))
    out = {}
    for ln in lines[1:]:
        f = ln.split()
        out[int(f[0])] = (int(f[1]), [int(v) for v in f[2:2 + nblocks]],
                          np.array([f32(float(v)) for v in f[2 + nblocks:]], f32))
    return out


@pytest.mark.parametrize("exe,ch,gm", [("run_OF_INT", 1, False), ("run_OF_RGB", 3, True)],
                         ids=["gray", "rgb-global-motion"])
def test_batch_command_fisher(tmp_path, exe, ch, gm, api):
    """A 17-frame clip (16 pairs, split by batches of 5) and a one-pair clip.  --fisher writes, clip for clip, what
    Context.fisher_begin / push / take give on the Python descriptor stage's descriptors, with and without
    --descriptors (whose file keeps its bytes); the tracks and the flows keep theirs."""
    import os
    import subprocess

    from of_dis_b200 import build

    from test_traj_desc import _write_png

    bindir = build.build_host()
    h, w = 96, 160
    clip = synth.global_motion_clip(16, h, w, ch, seed=98, H=synth.similarity_about_centre(h, w, 0.2, 1.0, (1.2, 0.4)))[0]
    other = synth.synthetic_sequence(2, h, w, ch, seed=99, amp=3.0)
    paths, imgs = {}, {}
    for name, fr in (("a", clip), ("b", other)):
        for t, img in enumerate(fr):
            paths[name, t] = str(tmp_path / ("%s%d.png" % (name, t)))
            imgs[name, t] = img
            _write_png(paths[name, t], img)
    pairs = [("a", t) for t in range(16)] + [("b", 0)]
    clips = [list(range(16)), [16]]
    rng = np.random.default_rng(ch)
    cb = idt_codebook(rng, 16)
    pp.write_fisher_codebook(str(tmp_path / "cb.fv"), cb)
    logs = {}
    for tag in ("desc", "fisher", "both"):
        outs = [str(tmp_path / ("%s%d.flo" % (tag, k))) for k in range(len(pairs))]
        lst = tmp_path / ("%s.txt" % tag)
        lst.write_text("".join("%s %s %s\n" % (paths[nm, t], paths[nm, t + 1], outs[k])
                               for k, (nm, t) in enumerate(pairs)))
        opts = ["--tracks", str(tmp_path / ("tracks_%s.txt" % tag))]
        opts += ["--global-motion", "homography", str(tmp_path / ("gm_%s.txt" % tag))] if gm else []
        opts += ["--descriptors", str(tmp_path / ("desc_%s.txt" % tag))] if tag != "fisher" else []
        opts += ["--fisher", str(tmp_path / "cb.fv"), str(tmp_path / ("fv_%s.txt" % tag))] if tag != "desc" else []
        r = subprocess.run([os.path.join(bindir, exe + "_batch"), str(lst), "--batch", "5"] + opts + ["2"],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        logs[tag] = r.stdout
    prm = params.operating_point(2, w, noc=ch, nop=2)
    bgr = (lambda a: a[..., ::-1]) if ch == 3 else (lambda a: a)  # the decoder holds BGR
    tp = dict(capacity=4 * ((w + 7) // 8) * ((h + 7) // 8), spacing=8, alpha=0.01, beta=0.5, mb_alpha=0.01,
              mb_beta=0.002, min_eig=25.0)
    got = {tag: _read_fisher(str(tmp_path / ("fv_%s.txt" % tag)), 5) for tag in ("fisher", "both")}
    pushed, skipped = 0, np.zeros(5, np.int64)
    for c, ks in enumerate(clips):
        fr = [bgr(imgs[pairs[ks[0]]])] + [bgr(imgs[pairs[k][0], pairs[k][1] + 1]) for k in ks]
        fr = np.ascontiguousarray(np.stack(fr))
        n = len(ks)
        scf = 1 << prm.sc_f
        ctx = api.Context(prm, (w + scf - 1) // scf * scf, (h + scf - 1) // scf * scf, prm.p_samp_s, 2 * n)
        ctx.upload_sequence_bidir_u8(0, n, fr, w, h)
        ctx.run(2 * n)
        M = None
        if gm:
            mp = dict(model=3, step=8, fb_check=0, alpha=0.01, beta=0.5, hypotheses=1024, threshold=1.0, refine=3,
                      seed=0)
            M = ctx.global_motion_fullres(0, n, mp, width_org=w, height_org=h, b0=n)[0].reshape(n, 9)
        ctx.traj_begin(tp, IDT, fr[0], w, h)
        _, _, desc, _ = ctx.traj_advance(0, n, n, fr[1:], w, h, models=M)
        ctx.fisher_begin(cb)
        ctx.fisher_push(desc)
        fv, _, cnt = ctx.fisher_take()
        ctx.close()
        pushed += cnt["pushed"]
        skipped += cnt["skipped"]
        for tag in ("fisher", "both"):
            g = got[tag][c]
            assert g[0] == cnt["pushed"] and g[1] == list(cnt["n"]), (tag, c)
            assert same(g[2], fv), (tag, c)
    assert pushed > 0
    for tag in ("fisher", "both"):
        line = [ln for ln in logs[tag].splitlines() if ln.startswith("FISHER")]
        assert line == ["FISHER clips 2 descriptors %d skipped %s" % (pushed, " ".join(map(str, skipped)))], logs[tag]
    # the tracks, the descriptors and the flows keep their bytes
    rd = lambda q: open(tmp_path / q, "rb").read()  # noqa: E731
    assert rd("tracks_desc.txt") == rd("tracks_fisher.txt") == rd("tracks_both.txt")
    assert rd("desc_desc.txt") == rd("desc_both.txt")
    for k in range(len(pairs)):
        assert rd("desc%d.flo" % k) == rd("fisher%d.flo" % k) == rd("both%d.flo" % k), k
