"""Fisher vectors of descriptors, restated on the CPU: preprocess.fisher_encode / FisherStream against a per-descriptor,
per-Gaussian loop written from ofdis_fisher_begin's header comment, exp_f32 against float64 exp, the skip rule, the
normalisation, the fit and the codebook file.  No GPU."""
import math

import numpy as np
import pytest

from of_dis_b200 import preprocess as pp

f32 = np.float32


def random_codebook(rng, K, blocks, desc_dim):
    """blocks: [(offset, dim_in, dim)]; a valid codebook with well-spread parameters."""
    cb = {"K": K, "desc_dim": desc_dim, "blocks": blocks}
    for k in pp.FISHER_PARTS:
        cb[k] = []
    for _, di, d in blocks:
        w = rng.uniform(0.2, 1.0, K)
        w /= w.sum()
        sig = rng.uniform(0.5, 2.0, (K, d))
        cb["mean"].append(rng.normal(0, 0.5, di).astype(f32))
        cb["proj"].append(rng.normal(0, 1.0 / math.sqrt(di), (d, di)).astype(f32))
        cb["mu"].append(rng.normal(0, 1.0, (K, d)).astype(f32))
        cb["isig"].append((1.0 / sig).astype(f32))
        cb["c"].append((np.log(w) - np.log(sig).sum(1)).astype(f32))
        cb["w"].append(w.astype(f32))
    return cb


def loop_encode(desc, cb):
    """The header's contract, one descriptor, block and Gaussian at a time, with float32 / float64 scalars."""
    K = cb["K"]
    fv, stats = [], []
    n_b, skipped = [], []
    for b, (o, di, d) in enumerate(cb["blocks"]):
        mean, proj, mu, isig, c, w = (cb[k][b] for k in pp.FISHER_PARTS)
        S0, S1, S2 = [0.0] * K, [[0.0] * d for _ in range(K)], [[0.0] * d for _ in range(K)]
        N = sk = 0
        with np.errstate(all="ignore"):
            for x in np.asarray(desc, f32):
                y = []
                for j in range(d):
                    acc = f32(0.0)
                    for i in range(di):
                        acc = f32(acc + f32(proj[j, i] * f32(x[o + i] - mean[i])))
                    y.append(acc)
                ll, zs, q_ok = [], [], True
                for k in range(K):
                    q = f32(0.0)
                    zk = []
                    for j in range(d):
                        z = f32(f32(y[j] - mu[k, j]) * isig[k, j])
                        zk.append(z)
                        q = f32(q + f32(z * z))
                    q_ok = q_ok and math.isfinite(float(q))
                    ll.append(f32(c[k] - f32(f32(0.5) * q)))
                    zs.append(zk)
                m = max(ll)
                if not all(math.isfinite(float(v)) for v in y) or not q_ok or not math.isfinite(float(m)):
                    sk += 1
                    continue
                e = [pp.exp_f32(f32(v - m))[()] for v in ll]
                s = f32(0.0)
                for v in e:
                    s = f32(s + v)
                N += 1
                for k in range(K):
                    g = float(f32(e[k] / s))
                    S0[k] = S0[k] + g
                    for j in range(d):
                        zd = float(zs[k][j])
                        S1[k][j] = S1[k][j] + g * zd
                        S2[k][j] = S2[k][j] + g * (zd * zd)
        n_b.append(N)
        skipped.append(sk)
        stats += S0 + [v for r in S1 for v in r] + [v for r in S2 for v in r]
        # the vector
        if N == 0:
            fv += [0.0] * (2 * K * d)
            continue
        f = []
        for part in (0, 1):
            for k in range(K):
                wk = float(w[k])
                for j in range(d):
                    t = S1[k][j] / (N * math.sqrt(wk)) if part == 0 else (S2[k][j] - S0[k]) / (N * math.sqrt(2.0 * wk))
                    r = math.sqrt(abs(t))
                    f.append(-r if t < 0 else r)
        partial = [0.0] * 256
        for i, v in enumerate(f):
            partial[i % 256] = partial[i % 256] + v * v
        tot = 0.0
        for v in partial:
            tot = tot + v
        nm = math.sqrt(tot)
        fv += [v / nm if nm > 0 else v for v in f]
    return (np.array(fv, np.float64).astype(f32), np.array(stats, np.float64),
            {"pushed": len(desc), "n": np.array(n_b), "skipped": np.array(skipped)})


def same(a, b):
    a, b = np.atleast_1d(a), np.atleast_1d(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def assert_encoded(got, exp):
    assert same(got[0], exp[0]), "vector differs"
    assert same(got[1], exp[1]), "statistics differ"
    assert got[2]["pushed"] == exp[2]["pushed"]
    assert np.array_equal(got[2]["n"], exp[2]["n"]) and np.array_equal(got[2]["skipped"], exp[2]["skipped"])


CASES = [  # K, blocks, desc_dim, n
    (1, [(0, 5, 5)], 5, 7),
    (3, [(0, 4, 2), (4, 6, 1), (1, 3, 3)], 10, 9),
    (5, [(2, 7, 4)], 12, 11),
    (2, [(0, 1, 1), (1, 300, 2)], 301, 4),
]


@pytest.mark.parametrize("K,blocks,desc_dim,n", CASES, ids=["K%d-%dblk" % (c[0], len(c[1])) for c in CASES])
def test_encode_equals_the_loop(K, blocks, desc_dim, n):
    rng = np.random.default_rng(K * 100 + n)
    cb = random_codebook(rng, K, blocks, desc_dim)
    x = rng.normal(0, 1.5, (n, desc_dim)).astype(f32)
    assert_encoded(pp.fisher_encode(x, cb), loop_encode(x, cb))


def test_every_cut_into_pushes_equals_one_push():
    rng = np.random.default_rng(5)
    cb = random_codebook(rng, 4, [(0, 6, 3), (6, 4, 4)], 10)
    x = rng.normal(0, 1.0, (9, 10)).astype(f32)
    x[4, 7] = np.nan
    one = pp.fisher_encode(x, cb)
    s = pp.FisherStream(cb)
    for mask in range(1 << 8):  # a cut after descriptor i where bit i is set
        cuts = [0] + [i + 1 for i in range(8) if mask >> i & 1] + [9]
        for a, b in zip(cuts[:-1], cuts[1:]):
            s.push(x[a:b])
        s.push(x[:0])
        assert_encoded(s.take(), one)


def test_exp_f32_within_its_bound():
    grid = np.arange(0x80000000, 0xC2AE0001, 97, dtype=np.uint64).astype(np.uint32).view(f32)
    grid = np.concatenate([grid, np.array([pp.EXP_CUTOFF, -0.0, 0.0], f32)])
    got = pp.exp_f32(grid).astype(np.float64)
    ref = np.exp(grid.astype(np.float64))
    ulp = np.spacing(ref.astype(f32)).astype(np.float64)
    assert (np.abs(got - ref) / ulp).max() <= 2.0
    assert pp.exp_f32(f32(0.0)) == 1.0 and pp.exp_f32(f32(-0.0)) == 1.0
    below = np.array([np.nextafter(pp.EXP_CUTOFF, f32(-np.inf)), -100.0, -1e30, -np.inf], f32)
    out = pp.exp_f32(below)
    assert np.array_equal(out.view(np.uint32), np.zeros(4, np.uint32))  # +0


@pytest.mark.parametrize("bad", ["nan", "inf", "-inf", "overflow_q", "overflow_z"])
def test_skipped_blocks(bad):
    rng = np.random.default_rng(11)
    cb = random_codebook(rng, 3, [(0, 4, 2), (4, 4, 4)], 8)
    x = rng.normal(0, 1.0, (6, 8)).astype(f32)
    if bad == "overflow_q":  # z finite, q overflows: a large entry in block 1, whose projection is the identity
        cb["proj"][1] = np.eye(4, dtype=f32)
        cb["mean"][1] = np.zeros(4, f32)
        x[2, 4] = 1e25
    elif bad == "overflow_z":
        cb["proj"][1] = np.eye(4, dtype=f32)
        cb["mean"][1] = np.zeros(4, f32)
        cb["isig"][1][:] = 1e10
        x[2, 4] = 3e38
    else:
        x[2, 5] = {"nan": np.nan, "inf": np.inf, "-inf": -np.inf}[bad]
    got = pp.fisher_encode(x, cb)
    assert_encoded(got, loop_encode(x, cb))
    assert list(got[2]["skipped"]) == [0, 1] and list(got[2]["n"]) == [6, 5]
    assert np.isfinite(got[0]).all() and np.isfinite(got[1]).all()
    # a skipped descriptor adds nothing: the block equals the clip without it
    rest = pp.fisher_encode(np.delete(x, 2, 0), cb)
    K = 3
    lo = 2 * K * 2
    assert same(got[0][lo:], rest[0][lo:])


def test_blocks_have_unit_norm_or_are_zero():
    rng = np.random.default_rng(3)
    cb = random_codebook(rng, 6, [(0, 10, 5), (10, 3, 3)], 13)
    x = rng.normal(0, 1.0, (50, 13)).astype(f32)
    x[:, 10] = np.nan  # block 1 skips every descriptor
    fv, _, cnt = pp.fisher_encode(x, cb)
    assert list(cnt["n"]) == [50, 0]
    a, b = fv[:2 * 6 * 5].astype(np.float64), fv[2 * 6 * 5:]
    assert abs(np.sqrt((a * a).sum()) - 1.0) < 1e-6
    assert not b.any()
    fv0, stats0, cnt0 = pp.fisher_encode(x[:0], cb)
    assert not fv0.any() and not stats0.any() and cnt0["pushed"] == 0


def test_fisher_blocks_of_idt():
    assert pp.fisher_blocks(pp.TRAJ_DEFAULTS) == [(0, 30), (30, 96), (126, 108), (234, 96), (330, 96)]
    blocks = [(o, di, di // 2) for o, di in pp.fisher_blocks(pp.TRAJ_DEFAULTS)]
    assert pp.fisher_sizes(256, blocks)["fv"] == 109056


def test_pca_and_its_signs():
    rng = np.random.default_rng(0)
    x = (rng.normal(0, 1, (2000, 4)) * [5.0, 2.0, 1.0, 0.1]).astype(f32)
    (mean, P, ev), = pp.fisher_pca(x, [(0, 4)], [2])
    assert P.shape == (2, 4) and mean.dtype == f32 and P.dtype == f32
    assert np.all(np.diff(ev) <= 0)
    assert np.allclose(np.abs(P), [[1, 0, 0, 0], [0, 1, 0, 0]], atol=0.05)
    assert (P[np.arange(2), np.abs(P).argmax(1)] > 0).all()


def test_fit_recovers_separated_means():
    """Four well-separated Gaussians in 3-D, every one projected through the identity (dim = dim_in): the fitted means
    lie within 0.1 of the true ones (in the PCA frame) and the weights within 0.03 of theirs."""
    rng = np.random.default_rng(1)
    true = np.array([[0, 0, 0], [8, 0, 0], [0, 8, 0], [0, 0, 8]], np.float64)
    wts = np.array([0.4, 0.3, 0.2, 0.1])
    lab = rng.choice(4, 6000, p=wts)
    x = (true[lab] + rng.normal(0, 0.5, (6000, 3))).astype(f32)
    cb = pp.fisher_fit(x, [(0, 3)], [3], K=4, iters=15, seed=7, var_floor=1e-3)
    mean, P = cb["mean"][0].astype(np.float64), cb["proj"][0].astype(np.float64)
    exp = (true - mean) @ P.T
    mu = cb["mu"][0].astype(np.float64)
    order = [int(np.argmin(((mu - e) ** 2).sum(1))) for e in exp]
    assert sorted(order) == [0, 1, 2, 3]
    assert np.abs(mu[order] - exp).max() < 0.1
    assert np.abs(cb["w"][0][order] - wts).max() < 0.03
    pp.fisher_check(cb)


def test_fit_is_deterministic_and_mstep_keeps_empty_gaussians():
    rng = np.random.default_rng(2)
    x = rng.normal(0, 1, (300, 6)).astype(f32)
    a = pp.fisher_fit(x, [(0, 4), (4, 2)], [2, 1], K=5, iters=2, seed=3)
    b = pp.fisher_fit(x, [(0, 4), (4, 2)], [2, 1], K=5, iters=2, seed=3)
    assert same(pp.fisher_pack(a), pp.fisher_pack(b))
    cb, eigs = pp.fisher_init(x, [(0, 4)], [2], 3, 0)
    stats = pp.fisher_encode(x, cb)[1]
    stats[1] = 0.0  # Gaussian 1 saw nothing
    stats[3 + 2:3 + 4] = 0.0
    stats[3 + 6 + 2:3 + 6 + 4] = 0.0
    new = pp.fisher_mstep(cb, stats, eigs, 1e-3)
    for k in ("mu", "isig", "c", "w"):
        assert same(new[k][0][1], cb[k][0][1])


def test_codebook_file_round_trips(tmp_path):
    rng = np.random.default_rng(9)
    cb = random_codebook(rng, 3, [(0, 4, 2), (5, 3, 3)], 9)
    path = str(tmp_path / "cb.fv")
    pp.write_fisher_codebook(path, cb)
    back = pp.read_fisher_codebook(path)
    assert back["K"] == 3 and back["desc_dim"] == 9 and back["blocks"] == cb["blocks"]
    assert same(pp.fisher_pack(back), pp.fisher_pack(cb))
    raw = open(path, "rb").read()
    assert raw[:8] == b"OFDISFV1"
    assert np.array_equal(np.frombuffer(raw, "<i4", 9, 8), [3, 2, 9, 0, 4, 2, 5, 3, 3])
    for bad in (raw[:-4], b"OFDISFV2" + raw[8:], raw[:12]):
        p2 = str(tmp_path / "bad.fv")
        open(p2, "wb").write(bad)
        with pytest.raises(ValueError):
            pp.read_fisher_codebook(p2)
    cb["isig"][1][0, 0] = 0.0
    pp.write_fisher_codebook(path, cb)
    with pytest.raises(ValueError):
        pp.read_fisher_codebook(path)


def test_fit_command_reads_every_nth_descriptor(tmp_path):
    from of_dis_b200 import fisher_fit

    dim = pp.traj_dim(pp.TRAJ_DEFAULTS)
    rng = np.random.default_rng(0)
    x = rng.random((10, dim)).astype(f32)
    path = tmp_path / "desc.txt"
    with open(path, "w") as f:
        f.write("# clip id start mean_x mean_y sd_x sd_y length desc[%d]\n" % dim)
        for i, r in enumerate(x):
            f.write("0 %d 0 1 2 3 4 5 " % i + " ".join("%.9g" % v for v in r) + "\n")
    assert same(fisher_fit.read_samples(str(path), 4), x[::3])
    assert same(fisher_fit.read_samples(str(path), 100), x)
    with open(path, "a") as f:
        f.write("0 1 2 3\n")
    with pytest.raises(ValueError):
        fisher_fit.read_samples(str(path), 100)


def _idt_codebook(K=2, blocks=None):
    rng = np.random.default_rng(0)
    blocks = blocks or [(o, di, di // 2) for o, di in pp.fisher_blocks(pp.TRAJ_DEFAULTS)]
    return random_codebook(rng, K, blocks, pp.traj_dim(pp.TRAJ_DEFAULTS))


@pytest.mark.parametrize("exe,args", [
    ("run_DE_INT", ["--tracks", "t.txt", "--fisher", "cb.fv", "f.txt"]),
    ("run_DE_RGB", ["--tracks", "t.txt", "--fisher", "cb.fv", "f.txt"]),
    ("run_OF_INT", ["--warm-start", "--tracks", "t.txt", "--fisher", "cb.fv", "f.txt"]),
    ("run_OF_RGB", ["--fisher", "cb.fv", "f.txt"]),
    ("run_OF_INT", ["--tracks", "t.txt", "--fisher", "cb.fv"]),
    ("run_OF_INT", ["--tracks", "t.txt", "--fisher", "none.fv", "f.txt"]),
    ("run_OF_INT", ["--tracks", "t.txt", "--fisher", "short.fv", "f.txt"]),
    ("run_OF_INT", ["--tracks", "t.txt", "--fisher", "magic.fv", "f.txt"]),
    ("run_OF_INT", ["--tracks", "t.txt", "--fisher", "zero_w.fv", "f.txt"]),
    ("run_OF_INT", ["--tracks", "t.txt", "--fisher", "blocks.fv", "f.txt"]),
    ("run_OF_RGB", ["--tracks", "t.txt", "--fisher", "dim.fv", "f.txt"]),
    ("run_OF_INT", ["--tracks", "t.txt", "--fisher", "cb.fv", "missing/dir/f.txt"]),
])
def test_batch_command_refuses_fisher(tmp_path, exe, args):
    """The stereo binaries, --warm-start, a missing --tracks, an unreadable, malformed or mismatched codebook and an
    unwritable path are refused before any device work, and no output file is written."""
    import subprocess

    from of_dis_b200 import build

    bindir = build.build_host()
    good = _idt_codebook()
    pp.write_fisher_codebook(str(tmp_path / "cb.fv"), good)
    raw = (tmp_path / "cb.fv").read_bytes()
    (tmp_path / "short.fv").write_bytes(raw[:-4])
    (tmp_path / "magic.fv").write_bytes(b"OFDISFV0" + raw[8:])
    bad = dict(good, w=[a.copy() for a in good["w"]])
    bad["w"][2][1] = 0.0
    pp.write_fisher_codebook(str(tmp_path / "zero_w.fv"), bad)
    pp.write_fisher_codebook(str(tmp_path / "blocks.fv"), _idt_codebook(blocks=[(0, 30, 15), (30, 396, 8)]))
    dim = _idt_codebook(blocks=[(0, 30, 15)])
    dim["desc_dim"] = 30
    pp.write_fisher_codebook(str(tmp_path / "dim.fv"), dim)
    inputs = sorted(q.name for q in tmp_path.iterdir())
    lst = tmp_path / "list.txt"
    lst.write_text("")
    r = subprocess.run([str(bindir) + "/" + exe + "_batch", str(lst)] + args, capture_output=True, text=True,
                       cwd=str(tmp_path))
    expect = 1 if "missing/dir/f.txt" in args else 2
    assert r.returncode == expect, (args, r.stdout, r.stderr)
    assert sorted(q.name for q in tmp_path.iterdir()) == sorted(inputs + ["list.txt"])


def test_batch_command_accepts_fisher(tmp_path):
    import subprocess

    from of_dis_b200 import build

    bindir = build.build_host()
    pp.write_fisher_codebook(str(tmp_path / "cb.fv"), _idt_codebook(K=3))
    (tmp_path / "list.txt").write_text("")
    r = subprocess.run([str(bindir) + "/run_OF_INT_batch", "list.txt", "--tracks", "t.txt", "--fisher", "cb.fv",
                        "f.txt"], capture_output=True, text=True, cwd=str(tmp_path))
    assert r.returncode == 0, (r.stdout, r.stderr)
    assert (tmp_path / "f.txt").read_text() == "# clip n_desc n_0 .. n_4 fv0 .. fv%d\n" % (2 * 3 * 213 - 1)
    assert (tmp_path / "t.txt").read_text() == "# clip frame id x y\n"
