"""CPU study (no GPU): how many rounds would the speculative walker need under different policies?

The exact swap-all chain of replicaexchange.py:321-349 is run sequentially on the MT19937 word stream (numba semantics, K a
power of two), recording for every 2-word slot whether an attempt starts there, its replicas and whether it changed the
permutation.  Rounds are then counted for:
  P0       the shipped walker: a round ends at the first visited slot that shares a replica with an earlier accepted,
           state-changing swap of the same round (window of W slots);
  P1       first-order forwarding: such a slot may stay in the round when exactly ONE earlier swap of the round touched it
           and that swap was itself evaluated normally (its new state could be forwarded by a shuffle);
  P2, P3   one-level forwarding without iteration.  The partner of slot p = (i, j), i != j, is the most recent of the 31
           slots before it that shares a replica with it (state independent).  Every slot is evaluated under the round's
           starting states (branch 0) and under the states its partner's swap would leave (branch 1); it takes branch 1
           if its partner lies in the window, changes the permutation under the starting states and is guessed visited:
           P2 guesses visited unless slot q-1 (in the window, evaluated under the starting states) draws a uniform, P3
           takes q's bit of the visited chain of the branch-0 decisions.  A visited slot is stale if a visited changing
           swap other than its partner shares a replica with it, if its guess was wrong, or if its partner is a visited
           slot that took branch 1; the round ends at the first stale slot or at a slot-31 attempt that draws a uniform.
           (Measured on an H100 with P3 in k_mix_walk2: the headline's rounds fell 1.44x, but a round took 275 instead of
           128 SASS instructions and 2.3x as long, so the walker was 1.52x slower; DESIGN.md section 9.)
  levels   the dependency depth of the true DAG (attempt waits for the last accepted swap that touched its replicas, and
           for its predecessor in the stream): the floor for any scheme without value prediction.
Usage: python tools/simulate_walker_policies.py [K] [nswap] [model]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden'))
import numpy as np
from energy_models import energies

K = int(sys.argv[1]) if len(sys.argv) > 1 else 256
nswap = int(sys.argv[2]) if len(sys.argv) > 2 else 300000
model = sys.argv[3] if len(sys.argv) > 3 else 'flat'
u = energies(model, K, 99)
words = np.random.RandomState(1234)._bit_generator.random_raw(4 * nswap + 64).astype(np.uint64)
mask = K - 1
perm = list(range(K))
ul = u.tolist()
slots = []   # (is_start, i, j, changed)
p = 0
import math
for t in range(nswap):
    i = int(words[p]) & mask; j = int(words[p + 1]) & mask
    si, sj = perm[i], perm[j]
    logp = -(ul[i][sj] + ul[j][si]) + ul[i][si] + ul[j][sj]
    p += 2
    if logp >= 0.0:
        acc = True; drew = False
    else:
        a, b = int(words[p]) >> 5, int(words[p + 1]) >> 6
        r = (a * 67108864.0 + b) / 9007199254740992.0
        acc = r < math.exp(logp); drew = True
        p += 2
    changed = acc and i != j
    if changed:
        perm[i], perm[j] = sj, si
    slots.append((True, i, j, changed))
    if drew:
        slots.append((False, -1, -1, False))
n_slots = len(slots)
print('K=%d model=%s attempts=%d slots=%d (%.2f slots/attempt)' % (K, model, nswap, n_slots, n_slots / nswap))


def rounds(W, forward):
    h = 0; n_rounds = 0; att = 0
    while h < n_slots:
        touched = {}          # replica -> number of accepted swaps of this round that touched it (and whether forwarded)
        s = h
        end = min(h + W, n_slots)
        while s < end:
            st, i, j, ch = slots[s]
            if st:
                ci, cj = touched.get(i), touched.get(j)
                stale = ci is not None or cj is not None
                fwd_lane = False
                if stale:
                    if not forward:
                        break
                    deps = [c for c in (ci, cj) if c is not None]
                    # forwardable: every touching swap was a normally evaluated one, and each replica was touched once
                    if any(c[0] > 1 or c[1] for c in deps) or s == h:
                        break
                    fwd_lane = True
                if ch:
                    for r in (i, j):
                        c = touched.get(r)
                        touched[r] = (1 if c is None else c[0] + 1, fwd_lane or (c is not None and c[1]))
                att += 1
            s += 1
        if s == h:   # the first lane itself can never be stale (fresh round): safety
            s = h + 1
        h = s
        n_rounds += 1
    return n_rounds


for W in (32, 64):
    r0 = rounds(W, False); r1 = rounds(W, True)
    print('window %2d slots: P0 %7d rounds (%.2f attempts/round)   P1 %7d rounds (%.2f attempts/round, x%.2f fewer)' % (
        W, r0, nswap / r0, r1, nswap / r1, r0 / r1))


def rounds_forward(guess, limit):
    """P2 (guess = 'prev') and P3 (guess = 'v0') over a 32-slot window: (rounds, attempts), the first `limit` attempts."""
    IJ = [(int(words[2 * s]) & mask, int(words[2 * s + 1]) & mask) for s in range(len(words) // 2 - 2)]

    def decide(s, si, sj):   # (log_p >= 0, accepted) of an attempt at slot s with replica states si, sj
        i, j = IJ[s]
        lp = -(ul[i][sj] + ul[j][si]) + ul[i][si] + ul[j][sj]
        if lp >= 0.0:
            return True, True
        a, b = int(words[2 * s + 2]) >> 5, int(words[2 * s + 3]) >> 6
        return False, (a * 67108864.0 + b) / 9007199254740992.0 < math.exp(lp)

    def partner(s):          # (d, r, b) or None
        i, j = IJ[s]
        if i == j:
            return None
        for d in range(1, min(32, s + 1)):
            oi, oj = IJ[s - d]
            if oi in (i, j) or oj in (i, j):
                if i != j and {oi, oj} == {i, j}:
                    return d, i, j
                r = i if i in (oi, oj) else j
                return d, r, (oj if oi == r else oi)
        return None

    perm = list(range(K)); h = 0; n_rounds = 0; att = 0
    while att < limit:
        n_rounds += 1
        start = perm[:]
        b0 = [decide(h + w, start[IJ[h + w][0]], start[IJ[h + w][1]]) for w in range(32)]
        v0 = set(); w = 0
        while w < 32:
            v0.add(w); w += 1 if b0[w][0] else 2
        fw = [False] * 32; alt = [None] * 32; part = [None] * 32
        for w in range(1, 32):
            pq = partner(h + w)
            if pq is None or pq[0] > w:
                continue
            d, r, b = pq; q = w - d; part[w] = q
            i, j = IJ[h + w]
            st = {i: start[i], j: start[j]}
            if {i, j} == {r, b} and r != b:
                st = {i: start[j], j: start[i]}
            else:
                st[r] = start[b]
            alt[w] = decide(h + w, st[i], st[j])
            qchg = b0[q][1] and r != b
            if guess == 'v0':
                seen = q in v0
            elif guess == 'prev':
                seen = not (q - 1 >= 0 and not b0[q - 1][0])
            else:   # P0: never forward
                seen = False
            fw[w] = qchg and seen
        committed = {}   # window position -> (changed, took branch 1)
        w = 0
        while w < 32 and att < limit:
            i, j = IJ[h + w]
            q = part[w]
            stale = any(c[0] and e != q and set(IJ[h + e]) & {i, j} for e, c in committed.items())
            if q is not None:
                q_va = q in committed and committed[q][0]
                stale = stale or fw[w] != q_va or (q in committed and committed[q][1])
            if stale:
                break
            ge, acc = alt[w] if fw[w] else b0[w]
            assert (ge, acc) == decide(h + w, perm[i], perm[j])   # the rules commit only decisions under the right states
            if w == 31 and not ge:
                break
            committed[w] = (acc and i != j, fw[w])
            if acc:
                perm[i], perm[j] = perm[j], perm[i]
            att += 1
            w += 1 if ge else 2
        h += max(w, 1)
    return n_rounds, att


n_fwd = min(nswap, 60000)
rp0 = rounds_forward('none', n_fwd)
for name, g in (('P2', 'prev'), ('P3', 'v0')):
    rf = rounds_forward(g, n_fwd)
    print('window 32 slots, first %d attempts: P0 %d rounds (%.2f attempts/round)   %s %d rounds (x%.2f fewer)' % (
        n_fwd, rp0[0], rp0[1] / rp0[0], name, rf[0], rp0[0] / rf[0]))
# dependency levels
last = [0] * K
F = 0
for st, i, j, ch in slots:
    if not st:
        continue
    l = max(last[i], last[j]) + 1
    F = max(F, l)
    if ch:
        last[i] = F; last[j] = F
print('true dependency depth: %d levels (%.2f attempts/level)' % (F, nswap / F))
