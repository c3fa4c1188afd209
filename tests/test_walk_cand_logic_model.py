"""Lane-level CPU models of the control logic of the walkers in candidate coordinates (openmmtools_b200/csrc/rx_walk2c.cuh):
the words numba's rejection-sampling randint accepts, numbered in stream order, one record per candidate index
{i, j, back-mask, the attempt's uniform, k = candidates among the uniform's two raw words}, a window of 32 candidate
indices, the visited chain for hops {2, 3, 4} resolved with stride-2 add-carry masks in grid phases, forced stops,
staleness, prefix commit and the hand-over to the plain loop at a word position.  Two walkers: the filter walker
k_mix_walk2c (rx_walk2.cuh) and the exact walker k_mix_walk_cand (rx_walk_exact.cuh), which also lets the attempt budget end
inside a window.  Each model must reproduce the sequential reference loop (replicaexchange.py:321-349 with numba's randint,
numba/_random.c) attempt by attempt, including the stream position."""
import sys, math, os, random
import numpy as np
import pytest
sys.path.insert(0, os.path.join(os.path.dirname(__file__), 'golden'))
from energy_models import energies

M32 = 0xffffffff


def popc(x): return bin(x).count('1')


def uniform(words, p):
    return ((words[p] >> 5) * 67108864.0 + (words[p + 1] >> 6)) / 9007199254740992.0


def attempt(K, u, words, mask, perm, p):
    """One attempt of the reference loop from word position p: (si, sj, accepted), the position after it."""
    while True:
        i = words[p] & mask; p += 1
        if i < K: break
    while True:
        j = words[p] & mask; p += 1
        if j < K: break
    si, sj = perm[i], perm[j]
    logp = -(u[i][sj] + u[j][si]) + u[i][si] + u[j][sj]
    if logp >= 0: acc = True
    else:
        acc = uniform(words, p) < math.exp(logp); p += 2
    if acc: perm[i], perm[j] = sj, si
    return (si, sj, acc), p


def reference(K, nswap, u, words, mask):
    perm = list(range(K)); p = 0; log = []
    for _ in range(nswap):
        entry, p = attempt(K, u, words, mask, perm, p)
        log.append(entry)
    return perm, p, log


def chain(Gw, K1w, K2w):
    """w2c_chain, operation for operation."""
    NG = ~Gw & M32
    T = NG & K1w; F = NG & K2w
    XgE = F & 0x55555555; XgO = F & 0xAAAAAAAA
    XpE = (XgE | (XgE << 1)) & M32; XpO = (XgO | (XgO << 1)) & M32
    stE = XgE & ~(XgE << 2) & M32; stO = XgO & ~(XgO << 2) & M32
    sEa = (XpE + (stE & 0x11111111)) & M32; sEb = (XpE + (stE & 0x44444444)) & M32
    sOa = (XpO + (stO & 0x22222222)) & M32; sOb = (XpO + (stO & 0x88888888)) & M32
    VE = 0x55555555 & ~(((sEa ^ XpE) & 0x44444444) | ((sEb ^ XpE) & 0x11111111)) & M32
    VO = 0xAAAAAAAA & ~(((sOa ^ XpO) & 0x88888888) | ((sOb ^ XpO) & 0x22222222)) & M32
    Vc, Xc, gc, Vn, Xn, gn = VE, XpE, 0x55555555, VO, XpO, 0xAAAAAAAA
    st = 1; V = 0
    while True:     # one grid phase per visited T: from position st on the current grid up to its first visited T
        R = ((Xc + st) ^ Xc) & gc & M32
        Vg = (Vc ^ (R if (st & ~Vc & M32) else 0)) & ~((st - 1) & M32) & M32
        Tv = Vg & T; t = Tv & -Tv & M32
        V |= Vg & (((t << 1) - 1) & M32)
        st = (t << 3) & M32
        if st == 0: break
        Vc, Xc, gc, Vn, Xn, gn = Vn, Xn, gn, Vc, Xc, gc
    Cf = V & (0x80000000 | ((T | F) & 0x40000000) | (F & 0x20000000))   # positions whose hop ends beyond position 32
    return V, Cf


def test_chain_masks_reproduce_the_sequential_chain():
    rng = random.Random(3)
    for _ in range(60000):
        pg = rng.choice([0.1, 0.3, 0.5, 0.69, 0.9, 1.0]); pk = rng.choice([0.5, 0.78, 1.0])
        G = K1 = K2 = 0
        for b in range(32):
            if rng.random() < pg: G |= 1 << b
            k = (rng.random() < pk) + (rng.random() < pk)
            if k == 1: K1 |= 1 << b
            if k == 2: K2 |= 1 << b
        V, Cf = chain(G, K1, K2)
        pos = 0; Vs = 0
        while pos < 32:
            Vs |= 1 << pos
            pos += 2 if (G >> pos) & 1 else 2 + ((K1 >> pos) & 1) + 2 * ((K2 >> pos) & 1)
        assert V == Vs
        last = Vs.bit_length() - 1           # the chain's last visited position either is the forced stop or hops to 32 exactly
        hop = 2 if (G >> last) & 1 else 2 + ((K1 >> last) & 1) + 2 * ((K2 >> last) & 1)
        assert Cf == ((1 << last) if last + hop > 32 else 0)


class Pass:
    """One pass over a seeded word stream: the reference's result, the candidate pre-pass (k_cand_count / scan / scatter /
    records) and the parts every walker model shares.  spare: the stream ends that many words after the reference's last
    attempt (None: long enough for the walker to run out of attempts first)."""

    def __init__(self, K, nswap, model, seed, spare=None):
        self.K, self.nswap = K, nswap
        self.u = energies(model, K, 99).tolist()
        self.mask = (1 << (K - 1).bit_length()) - 1
        words = [int(x) for x in np.random.RandomState(seed)._bit_generator.random_raw(12 * nswap + 6000).astype(np.uint64)]
        self.ref = reference(K, nswap, self.u, words, self.mask)
        self.words = words if spare is None else words[:self.ref[1] + spare]
        self.cpos = [p for p, x in enumerate(self.words) if (x & self.mask) < K]
        self.val = [self.words[p] & self.mask for p in self.cpos]
        self.nrec = len(self.cpos) - 3      # records exist for c < ncand - 3

    def rec(self, c):
        val, cpos = self.val, self.cpos
        i, j = val[c], val[c + 1]
        a = cpos[c + 1] + 1
        k = (cpos[c + 2] <= a + 1) + (cpos[c + 3] <= a + 1)
        bm = 0
        for b in range(31):
            cc = c - 1 - b
            if cc >= 0 and (val[cc] in (i, j) or val[cc + 1] in (i, j)): bm |= 1 << (31 - b)
        return i, j, k, a, bm

    def window(self, h, perm):
        """The 32 lanes of the window at candidate h under perm (exact decisions), and the window-order masks the walkers
        resolve: visited positions V, committed visited prefix per stops -> (lanes, V, stops)."""
        u = self.u
        lanes = []
        for w in range(32):
            i, j, k, a, bm = self.rec(h + w)
            si, sj = perm[i], perm[j]
            logp = -(u[i][sj] + u[j][si]) + u[i][si] + u[j][sj]
            ge0 = logp >= 0
            acc = ge0 or uniform(self.words, a) < math.exp(logp)
            lanes.append(dict(i=i, j=j, k=k, si=si, sj=sj, ge0=ge0, acc=acc, bm=bm))
        ballot = lambda f: sum((1 << l) for l in range(32) if f(lanes[l]))
        Gw = ballot(lambda x: x['ge0']); Aw = ballot(lambda x: x['acc'] and x['i'] != x['j'])
        K1w = ballot(lambda x: x['k'] == 1); K2w = ballot(lambda x: x['k'] == 2)
        V, Cf = chain(Gw, K1w, K2w)
        VA = V & Aw
        C = 0
        for w in range(32):
            earlier = (VA << (32 - w)) & M32 if w else 0
            if earlier & lanes[w]['bm']: C |= 1 << w
        Cw = (C | Cf) & V
        assert not (Cw & 1)
        return lanes, V, Cw

    @staticmethod
    def commit(lanes, cm, perm, log):
        for w in range(32):
            if (cm >> w) & 1:
                x = lanes[w]; log.append((x['si'], x['sj'], x['acc']))
        for w in range(32):
            x = lanes[w]
            if (cm >> w) & 1 and x['acc'] and x['i'] != x['j']:
                perm[x['i']] = x['sj']; perm[x['j']] = x['si']

    def finish(self, perm, p, rem, log):
        """The plain loop (k_mix_walk_serial) finishes from word position p; the result must be the reference's."""
        for _ in range(rem):
            entry, p = attempt(self.K, self.u, self.words, self.mask, perm, p)
            log.append(entry)
        perm_ref, head_ref, log_ref = self.ref
        assert log == log_ref
        assert perm == perm_ref and p == head_ref


def run(K, nswap, model, seed):
    """k_mix_walk2c: leaves at least 130 attempts and 560 records of a pass to the plain loop."""
    ps = Pass(K, nswap, model, seed)
    perm = list(range(K)); h = 0; rem = nswap; log = []; rounds = 0
    h_end = ps.nrec - 560 if ps.nrec >= 1200 else 0
    while rem >= 130 and ps.nrec >= 1200 and h + 99 <= h_end:
        rounds += 1
        lanes, V, Cw = ps.window(h, perm)
        low = Cw & -Cw
        below = (low - 1) & M32              # Cw == 0: the whole window commits, the next round starts at position 32
        cm = V & below
        ps.commit(lanes, cm, perm, log)
        h += popc(below); rem -= popc(cm)
    # ---- the plain loop finishes from the word position of candidate h (k_mix_walk_serial)
    ps.finish(perm, ps.cpos[h] if h > 0 else 0, rem, log)
    return rounds


def run_exact(K, nswap, model, seed, spare=None):
    """ex_walk<CAND = true> (k_mix_walk_cand): rounds while h + 32 <= nrec, the budget may end inside a window; the word
    position it hands to the plain loop is the next attempt's first candidate, or the word after the last attempt when the
    budget has ended.  Returns the rounds and the attempts left to the plain loop."""
    ps = Pass(K, nswap, model, seed, spare)
    perm = list(range(K)); h = 0; rem = nswap; log = []; rounds = 0; end = None
    while rem > 0 and h + 32 <= ps.nrec:
        rounds += 1
        lanes, V, stops = ps.window(h, perm)
        low = stops & -stops
        cm = V & ((low - 1) & M32)
        n = popc(cm)
        advance = popc((low - 1) & M32) if stops else 32
        if n > rem:                          # the first visited lane that must not run: the (rem+1)-th set bit of cm
            pos = 0; cnt = 0
            while pos < 32:
                if (cm >> pos) & 1:
                    if cnt == rem: break
                    cnt += 1
                pos += 1
            cm &= (1 << pos) - 1; n = rem; advance = pos
        if n == rem:                         # the budget ends here: the word after the last attempt's j (and uniform)
            last = cm.bit_length() - 1
            end = ps.cpos[h + last + 1] + (1 if lanes[last]['ge0'] else 3)
        ps.commit(lanes, cm, perm, log)
        h += advance; rem -= n
    left = rem
    ps.finish(perm, (ps.cpos[h] if rem else end) if h > 0 else 0, rem, log)
    return rounds, left


@pytest.mark.parametrize('K,model,nswap,seed', [(3, 'flat', 3000, 1), (5, 'normal', 3000, 2), (6, 'zeros', 2000, 3),
                                                (12, 'flat', 4000, 4), (100, 'normal', 6000, 5), (65, 'flat', 5000, 6),
                                                (127, 'ladder', 4000, 7), (129, 'normal', 4000, 8), (200, 'ladder', 5000, 9),
                                                (255, 'flat', 4000, 10)])
def test_model_reproduces_reference(K, model, nswap, seed):
    rounds = run(K, nswap, model, seed)
    assert 0 < rounds < nswap        # the window commits more than one attempt per round (few at tiny K: conflicts)


@pytest.mark.parametrize('K,model,nswap,seed,spare', [(3, 'flat', 3000, 1, None), (5, 'normal', 3000, 2, None),
                                                      (6, 'zeros', 2000, 3, None), (12, 'flat', 4000, 4, None),
                                                      (100, 'normal', 6000, 5, None), (65, 'flat', 5000, 6, None),
                                                      (127, 'ladder', 4000, 7, None), (129, 'normal', 4000, 8, None),
                                                      (1000, 'flat', 3000, 9, None), (300, 'ladder', 4000, 10, 6)])
def test_exact_walker_model_reproduces_reference(K, model, nswap, seed, spare):
    """The budget ends inside a window of the walker, or (spare: the stream ends just behind the reference's last attempt)
    the walker runs out of records and the plain loop finishes the pass."""
    rounds, left = run_exact(K, nswap, model, seed, spare)
    assert 0 < rounds < nswap        # the window commits several attempts per round
    assert (left > 0) == (spare is not None)
