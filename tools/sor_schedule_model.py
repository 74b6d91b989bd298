"""Symbolic model of sor_wave_kernel's data flow (of_dis_b200/csrc/sor_wave_kernel.cuh): every value is
a tag (I, j, sweep); the model replays the producer's loads, the stage ring, the double-buffered board,
the cluster halo ring and the in-place (du,dv) writes super-step by super-step and asserts that every
block reads exactly the operands the lexicographic scan gives it (top/left of this sweep, own/right/
bottom of the previous one) and that no bulk copy reads a location that is written while the copy may
still be in flight.  RT = rows per lane (tile of 4 columns x RT rows per thread and super-step).
run_chain replays the chain mode (one sweep per launch, CTAs in ticket order, any residency).
CPU-only; python tools/sor_schedule_model.py [W4 h HPAD RT K]."""
import sys

PF = 4


def run(W4, h, HPAD, RT, K, verbose=False):
    HB = HPAD * RT
    nb = (h + HB - 1) // HB
    NR = PF + 1 if K == 1 else PF + 2 * K - 1   # sor_stages
    R = (h + RT - 1) // RT
    S = W4 + R + 2 * K - 2
    glob = {(I, j): -1 for I in range(W4) for j in range(h)}  # sweep whose value is stored; -1 = before this solve

    class CTA:
        pass

    ctas = []
    for c in range(nb):
        t = CTA()
        t.c, t.j0, t.r0 = c, c * HB, c * HPAD
        t.hloc = min(HB, h - t.j0)
        t.nl = (t.hloc + RT - 1) // RT
        t.S_loc = W4 + t.nl + 2 * K - 2
        t.dmax = W4 + t.nl - 1
        t.stage = [None] * NR
        t.ist = 0
        t.board = [dict(), dict()]          # parity -> {(k, board row): tag}
        t.halo = [dict(), dict(), dict()]   # slot -> {(dir, k): tag}
        t.thr = {(k, rl): dict(left=[None] * RT, own=[None] * RT, st=0, stp=0, last=None)
                 for k in range(K) for rl in range(t.nl)}
        ctas.append(t)
    cur, prev, hcur, hprev = 0, 1, 0, 2
    checked = 0
    pending = []
    for T in range(-PF, S):
        stores, hstores, gwrites = [], [], []
        for t in ctas:
            tl = T - t.r0
            n = tl + PF
            if 0 <= n < t.S_loc:  # producer: the occupied lane rows of diagonal n (records and du,dv) + the halo block
                ih = min(max(n - HPAD, 0), W4 - 1)
                snap = {}
                if n <= t.dmax:
                    for rl in range(max(0, n - (W4 - 1)), min(t.nl - 1, n) + 1):
                        I = n - rl
                        for s in range(RT):
                            j = t.j0 + rl * RT + s
                            if j < h:
                                snap[("dud", rl, s)] = ((I, j), glob[(I, j)])
                if t.c + 1 < nb:
                    snap["halo"] = ((ih, t.j0 + HB), glob[(ih, t.j0 + HB)])
                t.stage[t.ist] = dict(n=n, rec_d=n, halo_I=ih, snap=snap, issued=T)
                pending.append((t, t.ist, t.r0 + n - 2))  # waited for two super-steps before sweep 0's tile on it
                t.ist = (t.ist + 1) % NR
            for (k, rl), th in t.thr.items():
                n = tl - 2 * k
                I = n - rl
                wlo = rl & ~31
                whi = min(wlo + 31, t.nl - 1)
                active = tl >= 0 and wlo <= n + 1 and whi > n - W4
                in_range = 0 <= I < W4
                if active:
                    st = t.stage[th["st"]]
                    if in_range:
                        assert st is not None and st["n"] == n and st["rec_d"] == I + rl and st["issued"] < T
                        assert ("dud", rl, 0) in st["snap"], "lane row inside the trimmed copy"
                    own = list(th["own"])
                    rf = [None] * RT
                    nxt = [None] * RT
                    if k == 0:
                        if in_range:
                            for s in range(RT):
                                j = t.j0 + rl * RT + s
                                if j >= h:
                                    continue
                                own[s] = st["snap"][("dud", rl, s)]
                                assert own[s] == ((I, j), -1), ("own", own[s])
                            sb = t.stage[(th["st"] + 1) % NR]  # diagonal n+1: right and bottom neighbours
                            jb = t.j0 + rl * RT + RT  # row below the tile
                            if I + 1 < W4 or jb < h:
                                assert sb is not None and sb["n"] == n + 1 and t.r0 + n + 1 - 2 <= T - 1, "load n+1 landed"
                            for s in range(RT):
                                j = t.j0 + rl * RT + s
                                if j < h and I + 1 < W4:
                                    assert sb["snap"][("dud", rl, s)] == ((I + 1, j), -1)
                            if jb < h:
                                if rl + 1 < HPAD:
                                    bot = sb["snap"][("dud", rl + 1, 0)]
                                else:
                                    assert sb["halo_I"] == I
                                    bot = sb["snap"]["halo"]
                                assert bot == ((I, jb), -1), ("bot k0", bot, I, jb)
                    else:
                        for s in range(RT):
                            nxt[s] = t.board[prev].get((k - 1, rl * RT + s + 1))
                        if t.c + 1 < nb and rl == t.nl - 1:
                            botX = t.halo[hprev].get((1, k - 1))
                        else:
                            botX = t.board[prev].get((k - 1, rl * RT + RT + 1))
                        if in_range:
                            for s in range(RT):
                                j = t.j0 + rl * RT + s
                                if j >= h:
                                    continue
                                assert own[s] == (I, j, k - 1), ("own k>0", own[s], (I, j, k - 1), T)
                                if I + 1 < W4:
                                    assert nxt[s] == (I + 1, j, k - 1), ("right", nxt[s], (I + 1, j, k - 1))
                                if j + 1 < h:
                                    b = own[s + 1] if s + 1 < RT else botX
                                    assert b == (I, j + 1, k - 1), ("bot", b, (I, j + 1, k - 1), T, t.c, k, rl, s)
                    topX = t.halo[hprev].get((0, k)) if (t.c > 0 and rl == 0) else t.board[prev].get((k, rl * RT))
                    new = [None] * RT
                    for s in range(RT):
                        j = t.j0 + rl * RT + s
                        if in_range and j < h:
                            if j > 0:
                                top = topX if s == 0 else new[s - 1]
                                assert top == (I, j - 1, k), ("top", top, (I, j - 1, k), T, t.c, k, rl, s)
                            if I > 0:
                                assert th["left"][s] == (I - 1, j, k), ("left", th["left"][s], (I - 1, j, k))
                            checked += 1
                            new[s] = (I, j, k)
                            if k == K - 1:
                                gwrites.append(((I, j), k))
                        else:
                            new[s] = ("junk", T, t.c, k, rl, s)
                        th["left"][s] = new[s]
                        stores.append((t.c, cur, (k, rl * RT + s + 1), new[s]))
                    th["last"] = new
                    if k > 0:
                        th["own"] = nxt
                if nb > 1 and th["last"] is not None:  # unconditional send of the latest tile row
                    if rl == 0 and t.c > 0:
                        hstores.append((t.c - 1, hcur, (1, k), th["last"][0]))
                    elif rl == t.nl - 1 and t.c + 1 < nb:
                        hstores.append((t.c + 1, hcur, (0, k), th["last"][RT - 1]))
                if n >= 0:
                    th["stp"] = th["st"]
                    th["st"] = (th["st"] + 1) % NR
        for ci, par, key, tag in stores:
            ctas[ci].board[par][key] = tag
        for ci, slot, key, tag in hstores:
            ctas[ci].halo[slot][key] = tag
        for key, k in gwrites:
            for t, si, wait_T in pending:
                if wait_T >= T:
                    for what, (blkk, _) in t.stage[si]["snap"].items():
                        assert blkk != key, ("in-place write races a bulk copy", key, T, t.c)
            assert glob[key] == -1
            glob[key] = k
        pending = [(t, si, wt) for (t, si, wt) in pending if wt >= T]
        cur, prev = prev, cur
        hprev, hcur = hcur, (hcur + 1) % 3
    assert checked == W4 * h * K, (checked, W4 * h * K)
    assert all(v == K - 1 for v in glob.values())
    if verbose:
        print("ok: W4=%d h=%d HPAD=%d RT=%d K=%d bands=%d steps=%d, %d block updates checked" % (W4, h, HPAD, RT, K, nb, S, checked))


def run_chain(W4, h, HPAD, RT, nf=2, R=None, pub=4, seed=0, lag=1, verbose=False):
    """Chain mode (one sweep per launch, bands on CTAs that need not be resident together): nf frames of nb
    bands, at most R CTAs resident at once (None = all), CTAs started in a random order, progress published
    every `pub` super-steps.  A super-step of a CTA is two events, interleaved at random with every other
    CTA's: the producer warp's (issue the bulk copy, publish progress, wait for the band above and fetch the
    top halo) and the compute warps' (update and store the blocks); the CTA barrier ends the super-step when
    both have happened.  So a published "tl super-steps done" is visible while super-step tl still runs, as
    in the kernel.  Asserts that every block reads the raster scan's operands, that no bulk copy of
    rec_below (or of the band's own lane rows) overlaps a write of this launch, that some CTA can always
    advance (no deadlock), and that the ticket counter and the progress words are zero again at the end.
    `lag`: super-steps beyond HPAD that the halo fetch for super-step tl+1 waits for (the kernel: tl + 1 +
    HPAD done, lag = 1); lag = 0 is an off-by-one the model must reject."""
    import random
    rnd = random.Random(seed)
    HB = HPAD * RT
    nb = (h + HB - 1) // HB
    NR = PF + 1
    n_cta = nf * nb
    R = n_cta if R is None else R
    glob = {(f, I, j): -1 for f in range(nf) for I in range(W4) for j in range(h)}  # -1: before this launch
    prog = {(f, c): 0 for f in range(nf) for c in range(nb)}
    counter = [0]
    pending = []  # (cta, local super-step that ends the copy's flight, keys)
    checked = [0]

    class CTA:
        pass

    def start(block):
        t = CTA()
        t.block, t.ticket = block, counter[0]
        counter[0] += 1
        if t.ticket == n_cta - 1:
            counter[0] = 0  # the last ticket resets the counter
        t.f, t.c = t.ticket % nf, t.ticket // nf
        t.j0, t.r0 = t.c * HB, t.c * HPAD
        t.nl = (min(HB, h - t.j0) + RT - 1) // RT
        t.S_loc, t.dmax = W4 + t.nl, W4 + t.nl - 1
        t.below, t.above = t.c + 1 < nb, t.c > 0
        t.tl, t.done = -PF, False
        t.prod = t.comp = False  # the producer's / the compute warps' event of super-step tl has happened
        t.stage = {}
        t.halo = {}  # local super-step -> tag of the top-row block it reads
        t.board = {}  # tile row of the band -> tag written in the previous super-step
        t.left = {}
        return t

    def events(t):
        if t.tl == t.S_loc:  # after the loop: wait for the band above's final value
            return ["end"] if not t.above or prog[(t.f, t.c - 1)] == W4 + HPAD else []
        ev = [] if t.comp else ["comp"]
        if not t.prod and not (t.above and 0 <= t.tl + 1 < W4 and prog[(t.f, t.c - 1)] < t.tl + lag + HPAD):
            ev.append("prod")
        return ev

    def write(f, I, j):
        for (u, wtl, keys) in pending:
            assert (f, I, j) not in keys, ("in-place write races a bulk copy", f, I, j, u.c)
        assert glob[(f, I, j)] == -1
        glob[(f, I, j)] = 0

    def step(t, ev):
        tl, f = t.tl, t.f
        if ev == "end":  # after the loop
            if t.below:
                prog[(f, t.c)] = t.S_loc
            if t.above:
                prog[(f, t.c - 1)] = 0
            t.done = True
            return
        if ev == "prod":
            producer(t, tl, f)
            t.prod = True
        else:
            compute(t, tl, f)
            t.comp = True
        if t.prod and t.comp:  # the CTA barrier that ends super-step tl
            pending[:] = [(u, wtl, k) for (u, wtl, k) in pending if not (u is t and wtl <= tl)]
            t.tl += 1
            t.prod = t.comp = False

    def producer(t, tl, f):
        # load tl+PF (own lane rows of the diagonal + the band below's row-0 block), publish, then the top halo
        n = tl + PF
        if 0 <= n < t.S_loc:
            snap, keys = {}, set()
            if n <= t.dmax:
                for rl in range(max(0, n - (W4 - 1)), min(t.nl - 1, n) + 1):
                    for s in range(RT):
                        j = t.j0 + rl * RT + s
                        if j < h:
                            snap[(rl, s)] = ((n - rl, j), glob[(f, n - rl, j)])
                            keys.add((f, n - rl, j))
            if t.below:
                ih = min(max(n - HPAD, 0), W4 - 1)
                snap["halo"] = ((ih, t.j0 + HB), glob[(f, ih, t.j0 + HB)])
                keys.add((f, ih, t.j0 + HB))
            t.stage[n] = snap
            pending.append((t, n - 2, keys))
        if t.below and tl > 0 and tl % pub == 0:
            prog[(f, t.c)] = tl
        if t.above and 0 <= tl + 1 < W4:
            assert prog[(f, t.c - 1)] >= tl + lag + HPAD
            jt = t.j0 - 1
            v = glob[(f, tl + 1, jt)]
            t.halo[tl + 1] = (tl + 1, jt, 0) if v == 0 else ("stale", tl + 1, jt)

    def compute(t, tl, f):
        # sweep 0: lane rl holds block I = tl - rl
        newboard = {}
        if tl >= 0:
            for rl in range(t.nl):
                I = tl - rl
                if not 0 <= I < W4:
                    continue
                st, sb = t.stage[tl], t.stage.get(tl + 1)
                new = []
                for s in range(RT):
                    j = t.j0 + rl * RT + s
                    if j >= h:
                        break
                    assert st[(rl, s)] == ((I, j), -1), ("own", st[(rl, s)])
                    if I + 1 < W4:
                        assert sb[(rl, s)] == ((I + 1, j), -1), ("right", sb[(rl, s)])
                    if j + 1 < h and s == RT - 1:
                        bot = sb[(rl + 1, 0)] if rl + 1 < HPAD else sb["halo"]
                        assert bot == ((I, j + 1), -1), ("bottom", bot, I, j + 1)
                    if j > 0:
                        if s > 0:
                            top = new[s - 1]
                        elif rl == 0:
                            top = t.halo.get(I)
                        else:
                            top = t.board.get(rl * RT - 1)
                        assert top == (I, j - 1, 0), ("top", top, (I, j - 1, 0), t.c, rl, s)
                    if I > 0:
                        assert t.left.get(j) == (I - 1, j, 0), ("left", t.left.get(j))
                    new.append((I, j, 0))
                    t.left[j] = (I, j, 0)
                    newboard[rl * RT + s] = (I, j, 0)
                    write(f, I, j)
                    checked[0] += 1
        t.board = newboard

    order = list(range(n_cta))
    rnd.shuffle(order)  # blockIdx of the CTAs in the order the GPU starts them
    resident, finished = [], 0
    while finished < n_cta:
        runnable = [(t, ev) for t in resident for ev in events(t)]
        startable = len(resident) < R and order
        assert runnable or startable, ("deadlock", [(t.f, t.c, t.tl) for t in resident])
        if startable and (not runnable or rnd.random() < 0.3):
            resident.append(start(order.pop()))
            continue
        t, ev = rnd.choice(runnable)
        step(t, ev)
        if t.done:
            resident.remove(t)
            finished += 1
    assert checked[0] == nf * W4 * h, (checked[0], nf * W4 * h)
    assert all(v == 0 for v in glob.values())
    assert counter[0] == 0 and all(v == 0 for v in prog.values()), "state left for the next launch"
    if verbose:
        print("ok chain: W4=%d h=%d HPAD=%d RT=%d frames=%d bands=%d R=%s pub=%d, %d block updates checked" %
              (W4, h, HPAD, RT, nf, nb, R, pub, checked[0]))


if __name__ == "__main__":
    if len(sys.argv) == 6:
        run(*map(int, sys.argv[1:]), verbose=True)
    else:
        for W4, h, HPAD, RT, K in [(5, 20, 32, 1, 3), (9, 70, 32, 1, 2), (12, 100, 32, 1, 3), (7, 33, 32, 1, 5),
                                   (5, 20, 32, 2, 3), (9, 70, 32, 2, 2), (12, 133, 32, 2, 3), (7, 65, 32, 2, 5),
                                   (3, 64, 32, 2, 1), (16, 56, 32, 2, 3), (6, 257, 32, 4, 3), (4, 130, 32, 4, 2),
                                   (20, 300, 64, 2, 3), (2, 96, 32, 4, 1), (1, 65, 32, 2, 3), (8, 17, 32, 4, 3)]:
            run(W4, h, HPAD, RT, K, verbose=True)
        for W4, h, HPAD, RT in [(5, 100, 32, 1), (9, 130, 32, 2), (3, 257, 32, 4), (12, 96, 32, 1)]:
            for R in (1, 2, None):
                run_chain(W4, h, HPAD, RT, nf=2, R=R, pub=4, seed=R or 0, verbose=True)
