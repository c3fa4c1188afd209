"""Lane-level CPU model of k_mix_walk_any's control logic (openmmtools_b200/csrc/rx_walk_exact.cuh): per-word-position
records (rejection-sampled indices, length, back-mask), the window of 32 word positions, the hop chain by pointer
jumping over the lanes (four doublings), staleness, prefix commit, the budget tail and the hand-over to
the plain loop.  The model must reproduce the sequential reference loop (replicaexchange.py:321-349 with numba's
rejection-sampling randint, numba/_random.c) attempt by attempt."""
import sys, math, os
import numpy as np
import pytest
sys.path.insert(0, os.path.join(os.path.dirname(__file__), 'golden'))
from energy_models import energies

ANY_SCAN = 40


def popc(x): return bin(x).count('1')


def uniform(words, p):
    return ((words[p] >> 5) * 67108864.0 + (words[p + 1] >> 6)) / 9007199254740992.0


def reference(K, nswap, u, words, mask):
    perm = list(range(K)); p = 0; log = []
    for _ in range(nswap):
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
        log.append((si, sj, acc))
        if acc: perm[i], perm[j] = sj, si
    return perm, p, log


def run(K, nswap, model, seed, scan=ANY_SCAN):
    u = energies(model, K, 99).tolist()
    nbits = (K - 1).bit_length()
    mask = (1 << nbits) - 1
    words = [int(x) for x in np.random.RandomState(seed)._bit_generator.random_raw(12 * nswap + 4000).astype(np.uint64)]
    nwords = len(words)
    perm_ref, head_ref, log_ref = reference(K, nswap, u, words, mask)

    # ---- records (k_words_build)
    cache = {}
    def ijl(p):
        if p < 0 or p >= nwords: return (0, 0, 0)
        if p not in cache:
            found = []; out = (0, 0, 0)
            for k in range(scan):
                if p + k >= nwords: break
                r = words[p + k] & mask
                if r < K:
                    found.append(r)
                    if len(found) == 2: out = (found[0], found[1], k + 1); break
            cache[p] = out
        return cache[p]
    def backmask(p):
        i, j, _ = ijl(p); bm = 0
        for b in range(31):
            oi, oj, ol = ijl(p - 1 - b)
            if ol == 0 or oi in (i, j) or oj in (i, j): bm |= 1 << (31 - b)
        return bm

    # ---- walker
    perm = list(range(K)); h = 0; rem = nswap; log = []; rounds = 0; gave_up = False
    while rem > 0 and h + 32 + scan + 2 <= nwords:
        rounds += 1
        lanes = []
        for l in range(32):
            p = h + l
            i, j, ln = ijl(p)
            unknown = ln == 0
            si, sj = perm[i], perm[j]
            logp = -(u[i][sj] + u[j][si]) + u[i][si] + u[j][sj]
            ge0 = logp >= 0
            acc = ge0 or (not unknown and uniform(words, p + ln) < math.exp(logp))
            hop = ln + (0 if ge0 else 2)
            lanes.append(dict(i=i, j=j, ln=ln, unknown=unknown, si=si, sj=sj, ge0=ge0, acc=acc, hop=hop, bm=backmask(p)))
        ballot = lambda f: sum((1 << l) for l in range(32) if f(lanes[l]))
        A = ballot(lambda x: x['acc'] and x['i'] != x['j'] and not x['unknown'])
        N = [64 if lanes[l]['unknown'] else l + lanes[l]['hop'] for l in range(32)]
        R = [1 << l for l in range(32)]
        for k in range(4):
            Rn = [R[N[l] & 31] for l in range(32)]; Nn = [N[N[l] & 31] for l in range(32)]
            for l in range(32):
                if N[l] < 32: R[l] |= Rn[l]; N[l] = Nn[l]
        V = R[0]; c = N[0]
        VA = V & A
        C = 0
        for l in range(32):
            earlier = (VA << (32 - l)) & 0xffffffff if l else 0
            if (earlier & lanes[l]['bm']) != 0 or lanes[l]['unknown']: C |= 1 << l
        C &= V
        low = C & -C
        cm = V & ((low - 1) & 0xffffffff)
        n = popc(cm)
        advance = popc((low - 1) & 0xffffffff) if C else c
        if C & 1: gave_up = True; break
        if n > rem:
            pos = 0; cnt = 0
            while pos < 32:
                if (cm >> pos) & 1:
                    if cnt == rem: break
                    cnt += 1
                pos += 1
            cm &= (1 << pos) - 1; n = rem; advance = pos
        for l in range(32):
            if (cm >> l) & 1:
                x = lanes[l]
                log.append((x['si'], x['sj'], x['acc']))
        for l in range(32):
            x = lanes[l]
            if (cm >> l) & 1 and x['acc'] and x['i'] != x['j']:
                perm[x['i']] = x['sj']; perm[x['j']] = x['si']
        h += advance; rem -= n
    # ---- the plain loop finishes (k_mix_walk_serial)
    p = h
    while rem > 0:
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
        log.append((si, sj, acc))
        if acc: perm[i], perm[j] = sj, si
        rem -= 1
    assert log == log_ref
    assert perm == perm_ref and p == head_ref
    return rounds, gave_up


@pytest.mark.parametrize('K,model,nswap,seed', [(3, 'flat', 3000, 1), (5, 'normal', 3000, 2), (6, 'zeros', 2000, 3),
                                                (12, 'flat', 4000, 4), (100, 'normal', 6000, 5), (65, 'flat', 5000, 6),
                                                (127, 'ladder', 4000, 7), (129, 'normal', 4000, 8), (1000, 'flat', 3000, 9)])
def test_model_reproduces_reference(K, model, nswap, seed):
    rounds, gave_up = run(K, nswap, model, seed)
    assert not gave_up
    assert rounds < nswap   # the window really commits several attempts per round


def test_unknown_positions_hand_over_to_the_plain_loop():
    """With a scan limit of 3 words many positions are 'unknown' (K = 65 rejects half of the words): rounds end before them
    and the walker gives up when one opens a window -- the result must still be the reference's."""
    rounds, gave_up = run(65, 3000, 'flat', 11, scan=3)
    assert gave_up
