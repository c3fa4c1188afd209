"""The commit of k_mix_walk2 / k_mix_walk2c (openmmtools_b200/csrc/rx_walk2.cuh) decides per lane from the round's stop mask
(window order) and the lane's prefix mask lem = (2 << w) - 1: the lane's record leaves the window iff (stops & lem) == 0,
its attempt is committed iff it also lies on the visited chain.  This must be the committed prefix of the round,
below = (stops & -stops) - 1 (stops == 0: the whole window), for every stop mask and window position, including the
encodings of the one exact attempt (stops = 2 or 4 for slots, 4 or 4 << k for candidate indices)."""
import random

M32 = 0xffffffff


def lem(w):
    return ((2 << w) - 1) & M32   # 32-bit: w = 31 gives all ones


def below(stops):
    return ((stops & (-stops & M32)) - 1) & M32


def check(stops, vis):
    b = below(stops)
    for w in range(32):
        promoted = (stops & lem(w)) == 0
        assert promoted == bool((b >> w) & 1), (hex(stops), w)
        mine = promoted and bool((vis >> w) & 1)
        assert mine == bool(((vis & b) >> w) & 1)


def test_prefix_mask_matches_committed_prefix():
    rng = random.Random(3)
    masks = [0, 1, M32, 0x80000000, 0x40000000, 2, 4, 8, 16, 4 << 1, 4 << 2]
    masks += [1 << k for k in range(32)] + [rng.getrandbits(32) for _ in range(3000)]
    masks += [rng.getrandbits(32) & ~((1 << rng.randrange(32)) - 1) for _ in range(3000)]
    for stops in masks:
        check(stops, rng.getrandbits(32))
        check(stops, M32)


def test_exact_attempt_encodings():
    # slots: 1 or 2 positions leave; candidates: 2 or 2 + k (k = 0, 1, 2)
    for stops, n in [(2, 1), (4, 2), (4, 2), (4 << 1, 3), (4 << 2, 4)]:
        assert bin(below(stops)).count('1') == n
        assert [w for w in range(32) if (stops & lem(w)) == 0] == list(range(n))
    # nothing committed: stops = 1 (position 0 stops), no lane leaves
    assert all((1 & lem(w)) != 0 for w in range(32)) and below(1) == 0
