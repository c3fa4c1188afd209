"""Two alchemical regions in double precision, built from the one-region CPU oracle by inclusion-exclusion.

With region ids 0 (environment), 1 and 2, the energy of the reference's two-region system (alchemy.py:1539-2038, no
alchemical_regions_interactions) is E_EE + E_E1(l1) + E_11 + E_E2(l2) + E_22: no term covers the pairs across the two
regions.  A one-region system whose other-region atoms have epsilon = 0 has exactly the terms of its own region and of
the environment (an epsilon of 0 zeroes every pair it is in, plain or soft-core), so

    E(l1, l2) = E_1(l1) + E_2(l2) - E_0,

where E_r is the one-region oracle with region r alchemical and the other region's epsilons zeroed, and E_0 the oracle
with the epsilons of both regions zeroed.  Forces add the same way."""
import numpy as np
from helpers import oracle_system


class RegionsReference:
    def __init__(self, s, region, annihilate_1=False, annihilate_2=False, alpha=0.5, a=1.0, b=1.0, c=6.0, box=None,
                 use_switch=True):
        ids = np.asarray(region)
        self.N = len(ids)

        def one(alch_id, zero_ids, annihilate):
            t = dict(s)
            t['eps'] = np.where(np.isin(ids, zero_ids), 0.0, s['eps'])
            t['alch'] = (ids == alch_id).astype(np.uint8)
            if box is not None:
                t['box'] = np.asarray(box, np.float64)
            return oracle_system(t, annihilate=annihilate, alpha=alpha, a=a, b=b, c=c, use_switch=use_switch)

        self.s1 = one(1, [2], annihilate_1)
        self.s2 = one(2, [1], annihilate_2)
        self.s0 = one(1, [1, 2], False)

    def energy(self, x, l1, l2, forces=False):
        r1, r2, r0 = (s.energy(x, lam, forces=forces) for s, lam in ((self.s1, l1), (self.s2, l2), (self.s0, 1.0)))
        U = r1[0] + r2[0] - r0[0]
        return (U, r1[2] + r2[2] - r0[2]) if forces else U

    def energy_matrix(self, xs, l1, l2, betas, offsets=None):
        l1, l2, betas = (np.asarray(v, np.float64) for v in (l1, l2, betas))
        u = (self.s1.energy_matrix(xs, l1, betas) + self.s2.energy_matrix(xs, l2, betas) -
             self.s0.energy_matrix(xs, np.ones_like(l1), betas))
        if offsets is not None:
            u = u + betas * np.asarray(offsets, np.float64)
        return u
