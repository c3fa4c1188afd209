"""A CPU model of the speculative walker's ROUND LOGIC (openmmtools_b200/csrc/rx_walk_exact.cuh, k_mix_walk_pow2), checked against
the golden vectors of the real reference loop.  It restates, with Python integers, exactly the bit arithmetic of the
kernel -- slot records with the back-mask in bit order 31-b, the add-carry resolution of the visited chain, staleness
from `shl(VA, 32 - lane) & backmask`, the committed prefix and the advance -- so that a change of that logic can be
tried and regression-tested without a GPU.  Decisions are exact f64 (the device's f32 filter only ever defers to them)."""
import math
import os
import sys
import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'golden'))
from energy_models import energies

G = np.load(os.path.join(HERE, 'golden', 'mixing_golden.npz'))
M32 = 0xFFFFFFFF


def mt_words(seed, n):
    """numba's generator after np.random.seed(seed): init_genrand(seed), raw 32-bit outputs."""
    return np.random.RandomState(seed)._bit_generator.random_raw(n).astype(np.uint64)


def build_slots(words, K):
    mask = K - 1
    n = len(words) // 2
    i = (words[0:2 * n:2] & mask).astype(np.int64); j = (words[1:2 * n:2] & mask).astype(np.int64)
    a = (words[0:2 * n:2] >> 5).astype(np.float64); b = (words[1:2 * n:2] >> 6).astype(np.float64)
    U = (a * 67108864.0 + b) / 9007199254740992.0
    with np.errstate(divide='ignore'):
        logU = np.where(U == 0.0, -745.5, np.log(U))
    back = np.zeros(n, np.int64)
    for bidx in range(31):                      # bit 31-b: slot s-1-b shares a replica index with slot s
        d = bidx + 1
        hit = np.zeros(n, bool)
        hit[d:] = (i[d:] == i[:-d]) | (i[d:] == j[:-d]) | (j[d:] == i[:-d]) | (j[d:] == j[:-d])
        back |= hit.astype(np.int64) << (31 - bidx)
    return i, j, logU, back


def walk(u, K, words, nswap, perm):
    """Rounds of 32 slots until nswap attempts are done; returns (perm, n_accepted, n_proposed)."""
    i_all, j_all, logU, back = build_slots(words, K)
    nacc = np.zeros((K, K), np.int64); nprop = np.zeros((K, K), np.int64)
    h, rem = 0, nswap
    ul = u
    while rem > 0:
        ge0 = [False] * 32; acc = [False] * 32; si_l = [0] * 32; sj_l = [0] * 32
        for lane in range(32):
            s = h + lane
            i, j = int(i_all[s]), int(j_all[s])
            si, sj = perm[i], perm[j]
            si_l[lane], sj_l[lane] = si, sj
            logp = -(ul[i, sj] + ul[j, si]) + ul[i, si] + ul[j, sj]       # replicaexchange.py:333-335, same order
            if logp >= 0.0:
                ge0[lane] = acc[lane] = True
            else:
                d = logp - logU[s + 1]                                      # the uniform lives in the NEXT slot
                if d > 1e-9:
                    acc[lane] = True
                elif d >= -1e-9:                                            # guard band: what the reference does
                    a = int(words[2 * (s + 1)]) >> 5; b = int(words[2 * (s + 1) + 1]) >> 6
                    acc[lane] = (a * 67108864.0 + b) / 9007199254740992.0 < math.exp(logp)
        Gm = sum(1 << l for l in range(32) if ge0[l])
        Am = sum(1 << l for l in range(32) if acc[l] and int(i_all[h + l]) != int(j_all[h + l]))
        X = ~Gm & M32
        starts = X & ~((X << 1) & M32) & M32
        SE, SO = starts & 0x55555555, starts & 0xAAAAAAAA
        sumE, sumO = X + SE, X + SO                                          # 33-bit sums: the carry out matters below
        skip = ((((sumE & M32) ^ X) & ~SE & M32) & 0xAAAAAAAA) | ((((sumO & M32) ^ X) & ~SO & M32) & 0x55555555)
        V = ~skip & M32
        VA = V & Am
        C = 0
        for lane in range(32):
            earlier = (VA << (32 - lane)) & M32 if lane else 0               # shl.b32 by 32 gives 0
            if earlier & int(back[h + lane]):
                C |= 1 << lane
        C &= V
        low = C & (-C & M32)
        cm = V & ((low - 1) & M32)
        n = bin(cm).count('1')
        advance = bin((low - 1) & M32).count('1') if C else 32 + (1 if (sumO >> 32) else 0)
        if n > rem:
            pos = cnt = 0
            while pos < 32:
                if (cm >> pos) & 1:
                    if cnt == rem:
                        break
                    cnt += 1
                pos += 1
            cm &= (1 << pos) - 1; n = rem; advance = pos
        for lane in range(32):
            if (cm >> lane) & 1:
                i, j = int(i_all[h + lane]), int(j_all[h + lane])
                si, sj = si_l[lane], sj_l[lane]
                nprop[si, sj] += 1; nprop[sj, si] += 1
                if acc[lane]:
                    nacc[si, sj] += 1; nacc[sj, si] += 1
                    if i != j:
                        perm[i], perm[j] = sj, si
        h += advance; rem -= n
    return perm, nacc, nprop


CASES = ['all_K2_s0_flat', 'all_K2_s1234_normal', 'all_K16_s0_zeros', 'all_K16_s1_normal', 'all_K16_s1234_ladder',
         'all_K16_s1234_flat', 'all_K64_s0_flat', 'all_K64_s1234_ladder']


@pytest.mark.parametrize('tag', [t for t in CASES if t in set(map(str, G['all_cases']))])
def test_round_logic_model_reproduces_the_reference_loop(tag):
    _, Ks, ss, model = tag.split('_')
    K, seed = int(Ks[1:]), int(ss[1:])
    u = np.asarray(energies(model, K, K * 1000 + (seed % 1000)), np.float64)
    nswap = K ** 3
    words = mt_words(seed, 4 * nswap + 4096)
    perm = list(range(K))
    perm, nacc, nprop = walk(u, K, words, nswap, perm)
    assert np.array_equal(np.array(perm), G[f'{tag}_perm1']), tag
    if f'{tag}_nacc1' in G.files:
        assert np.array_equal(nacc, G[f'{tag}_nacc1']) and np.array_equal(nprop, G[f'{tag}_nprop1'])
    assert nprop.sum() == 2 * nswap
