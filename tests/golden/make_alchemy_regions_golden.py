#!/usr/bin/env python
"""Golden data for two alchemical regions, from the REAL reference code (build container only).

Runs the reference's ``AbsoluteAlchemicalFactory._alchemically_modify_NonbondedForce`` unmodified, with the loaders and
recording stand-ins of ``make_alchemy_golden.py``, on a list of two ``AlchemicalRegion``s, and records:

  * the force inventory: per force its type, global parameters, interaction groups (as full sorted atom lists) and, for
    the NonbondedForce, the epsilons it keeps (the regions' atoms are zeroed, alchemy.py:1903-1909);
  * every force in full (particle parameters, groups, globals, flags, as make_adapter_golden.py dumps them), which the
    adapter test rebuilds into stand-ins;
  * the total energy of a periodic configuration on a (lambda_1, lambda_2) grid that includes 0 and 1 on both axes,
    evaluated with numpy (NonbondedForce: Lorentz-Berthelot LJ; CustomNonbondedForce: the Lepton expression over the
    interaction groups), switching function off.

Configurations: regions 'A' + 'B' with B annihilating; None + 'B'; 'A' + 'B' with a non-default soft core.
Output: tests/golden/alchemy_regions_golden.npz
"""
import json, os, sys
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_alchemy_golden import (load_factory, reference_force, nonbonded_energy, custom_nonbonded_energy, lj_setup,
                                 NonbondedForce, CustomNonbondedForce, u)
from make_adapter_golden import dump

N = 40
REGION_1, REGION_2 = [0, 1, 2, 3], [4, 5, 6]
GRID = [0.0, 0.4, 1.0]
CONFIGS = [  # names, annihilate_sterics of each region, softcore (alpha, a, b, c)
    (('A', 'B'), (False, True), (0.5, 1, 1, 6)),
    ((None, 'B'), (True, False), (0.5, 1, 1, 6)),
    (('A', 'B'), (False, False), (0.3, 2, 1.5, 12)),
]


def inventory(forces_by_lambda):
    out = []
    for key, forces in forces_by_lambda.items():
        for f in forces:
            d = {'key': repr(key), 'type': type(f).__name__, 'globals': dict(f.globals)}
            if isinstance(f, CustomNonbondedForce):
                d.update(expression=f.expression, groups=[[list(map(int, a)), list(map(int, b))] for a, b in f.groups],
                         n_particles=len(f.particles), lrc=bool(f.lrc))
            elif isinstance(f, NonbondedForce):
                d.update(eps=[float(u.to_md(p[2])) for p in f.particles])
            else:
                d.update(n_bonds=len(f.bonds))
            out.append(d)
    return out


if __name__ == '__main__':
    Factory, Region = load_factory()
    s = lj_setup(N=N, n_alch=0, reduced_density=0.4, seed=78)
    x, L = s['x'], s['L']
    out = {'x': x, 'L': L, 'sigma': s['sigma'], 'eps': s['eps'], 'rc': s['rc'], 'grid': np.array(GRID),
           'region_1': np.array(REGION_1), 'region_2': np.array(REGION_2)}
    for c, (names, ann, (alpha, a, b, cc)) in enumerate(CONFIGS):
        regions = [Region(alchemical_atoms=list(atoms), name=nm, annihilate_sterics=an, softcore_alpha=alpha, softcore_a=a,
                          softcore_b=b, softcore_c=cc) for atoms, nm, an in zip((REGION_1, REGION_2), names, ann)]
        forces_by_lambda = Factory()._alchemically_modify_NonbondedForce(reference_force(s), regions, frozenset())
        out['config%d_forces' % c] = np.array(json.dumps(inventory(forces_by_lambda)))
        out['config%d_full' % c] = np.array(json.dumps([dump(f) for v in forces_by_lambda.values() for f in v]))
        out['config%d_meta' % c] = np.array(json.dumps({'names': names, 'annihilate': ann, 'softcore': [alpha, a, b, cc]}))
        sfx = ['' if nm is None else '_' + nm for nm in names]
        U = np.zeros((len(GRID), len(GRID)))
        for i, l1 in enumerate(GRID):
            for j, l2 in enumerate(GRID):
                lam = {'lambda_sterics' + sfx[0]: l1, 'lambda_electrostatics' + sfx[0]: l1,
                       'lambda_sterics' + sfx[1]: l2, 'lambda_electrostatics' + sfx[1]: l2}
                e = 0.0
                for forces in forces_by_lambda.values():
                    for f in forces:
                        if isinstance(f, NonbondedForce):
                            e += nonbonded_energy(f, x, L)
                        elif isinstance(f, CustomNonbondedForce):
                            e += custom_nonbonded_energy(f, x, L, lam)
                        else:
                            assert len(f.bonds) == 0
                U[i, j] = e
        out['config%d_U' % c] = U
        print(c, names, ann, U.ravel())
        for d in inventory(forces_by_lambda):
            print('   ', d['type'], d['globals'], [[len(g[0]), len(g[1])] for g in d.get('groups', [])])
    dst = os.path.join(HERE, 'alchemy_regions_golden.npz')
    np.savez_compressed(dst, **out)
    print('wrote', dst, os.path.getsize(dst))
