"""Two alchemical regions against the REAL reference factory (tests/golden/make_alchemy_regions_golden.py): the
reference's ``_alchemically_modify_NonbondedForce`` (alchemy.py:1539-2038) ran unmodified on two regions, and its
forces were recorded and evaluated with numpy on a (lambda_1, lambda_2) grid.  Pins: the two-region energy function of
the oracle (regions_ref.py) to 1e-10, the force inventory (no force covers the pairs across the regions, the regions'
epsilons are zeroed in the NonbondedForce, each region's lambda_sterics<suffix>), and the adapter's reading of those
forces against the package's own factory."""
import json
import os
import sys
import numpy as np
import pytest
from openmmtools_b200 import unit as u, alchemy, states, _backend
from openmmtools_b200.contrib import openmm_adapter as adapter
from helpers import lj_setup
from regions_ref import RegionsReference

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'golden'))
from make_alchemy_regions_golden import CONFIGS, GRID, N, REGION_1, REGION_2

G = np.load(os.path.join(HERE, 'golden', 'alchemy_regions_golden.npz'))


def setup():
    s = lj_setup(N=N, n_alch=0, reduced_density=0.4, seed=78)
    assert np.array_equal(s['x'], G['x']) and s['L'] == float(G['L'])
    ids = np.zeros(N, np.uint8)
    ids[REGION_1] = 1
    ids[REGION_2] = 2
    return s, ids


@pytest.mark.parametrize('c', range(len(CONFIGS)))
def test_oracle_energy_equals_the_reference_two_region_forces(c):
    names, ann, (alpha, a, b, cc) = CONFIGS[c]
    s, ids = setup()
    ref = RegionsReference(s, ids, *ann, alpha=alpha, a=a, b=b, c=cc, box=(s['L'],) * 3, use_switch=False)
    U = G['config%d_U' % c]
    for i, l1 in enumerate(GRID):
        for j, l2 in enumerate(GRID):
            e = ref.energy(s['x'], l1, l2)
            assert abs(e - U[i, j]) < 1e-10 * max(1.0, abs(U[i, j])), (c, l1, l2, e, U[i, j])


@pytest.mark.parametrize('c', range(len(CONFIGS)))
def test_reference_force_inventory(c):
    names, ann, soft = CONFIGS[c]
    inv = json.loads(str(G['config%d_forces' % c]))
    r1, r2 = set(REGION_1), set(REGION_2)
    env = set(range(N)) - r1 - r2
    pairs = []
    for f in inv:
        if f['type'] != 'CustomNonbondedForce':
            continue
        for a, b in f['groups']:
            a, b = set(a), set(b)
            # no interaction group puts an atom of one region against an atom of the other
            assert not ((a & r1 and b & r2) or (a & r2 and b & r1)), f['groups']
            pairs.append((frozenset(a), frozenset(b), f))
    sterics = [p for p in pairs if 'lambda_electrostatics' not in ''.join(p[2]['globals'])]
    for region, name, annihilate in zip((r1, r2), names, ann):
        lam = 'lambda_sterics' + ('' if name is None else '_' + name)
        ex = [f for a, b, f in sterics if {a, b} == {frozenset(env), frozenset(region)}]
        rr = [f for a, b, f in sterics if a == b == frozenset(region)]
        assert len(ex) == 1 and len(rr) == 1
        assert lam in ex[0]['globals']                             # environment x region: that region's lambda
        assert (lam in rr[0]['globals']) == annihilate             # region x region: only when annihilating
        for f in ex + rr:
            assert tuple(f['globals'][k] for k in ('softcore_alpha', 'softcore_a', 'softcore_b', 'softcore_c')) == tuple(soft)
    nb = [f for f in inv if f['type'] == 'NonbondedForce']
    assert len(nb) == 1
    eps = np.array(nb[0]['eps'])
    assert np.all(eps[REGION_1 + REGION_2] == 0.0) and np.all(eps[sorted(env)] > 0.0)


class StandInSystem:
    def __init__(self, s):
        self.s = s

    def getParticleMass(self, i):
        return self.s['mass'][i] * u.dalton

    def getDefaultPeriodicBoxVectors(self):
        L = self.s['L']
        return [np.array(v) * u.nanometer for v in ([L, 0, 0], [0, L, 0], [0, 0, L])]


class _Stub:
    """A force rebuilt from the fixture, with the OpenMM getters the adapter uses."""
    CutoffPeriodic = 2

    def __init__(self, d):
        self.d = d
        self.globals = d['globals']
        self.expression = d.get('expression')
        self.particles = d.get('particles', [])
        self.groups = [(a, b) for a, b in d.get('groups', [])]
        self.lrc = d.get('lrc')
        self.bonds = [None] * d.get('n_bonds', 0)

    def getNumParticles(self): return len(self.particles)
    def getParticleParameters(self, i): return list(self.particles[i])
    def getNumExceptions(self): return self.d['exceptions']
    def getNonbondedMethod(self): return self.d['method']
    def getCutoffDistance(self): return self.d['cutoff']
    def getUseSwitchingFunction(self): return self.d['use_switch']
    def getSwitchingDistance(self): return self.d['switch_distance']
    def getUseDispersionCorrection(self): return self.d['dispersion']


@pytest.mark.parametrize('c', range(len(CONFIGS)))
def test_adapter_reads_the_reference_two_region_forces_like_our_factory(c):
    names, ann, (alpha, a, b, cc) = CONFIGS[c]
    s, ids = setup()
    forces = [type(d['type'], (_Stub,), {})(d) for d in json.loads(str(G['config%d_full' % c]))]
    rec = adapter.system_from_openmm(StandInSystem(s), forces)
    # the package's factory on the same fluid and regions
    plain = adapter.system_from_openmm(StandInSystem(s), [f for f in forces if type(f).__name__ == 'NonbondedForce'])
    plain.epsilon = np.asarray(s['eps'], np.float64)
    regions = [alchemy.AlchemicalRegion(alchemical_atoms=atoms, name=nm, annihilate_sterics=an, softcore_alpha=alpha,
                                        softcore_a=a, softcore_b=b, softcore_c=cc)
               for atoms, nm, an in zip((REGION_1, REGION_2), names, ann)]
    own = alchemy.AbsoluteAlchemicalFactory().create_alchemical_system(plain, regions)
    assert rec.alchemical_regions == own.alchemical_regions
    assert np.array_equal(rec.alchemical_region_ids(), ids)
    assert rec.global_parameters == own.global_parameters
    assert (rec.softcore_alpha, rec.softcore_a, rec.softcore_b, rec.softcore_c) == (alpha, a, b, cc)
    assert np.allclose(rec.sigma, s['sigma']) and np.allclose(rec.epsilon, s['eps'])
    assert rec.alchemical_dispersion_correction == own.alchemical_dispersion_correction
    # the same engine tables from both records
    l1, l2 = [1.0, 0.6, 0.0], [0.0, 0.3, 1.0]
    ts_rec = adapter.thermodynamic_states_from_openmm(rec, [300.0] * 3, l1, l2)
    comp = [alchemy.AlchemicalState.from_system(own, parameters_name_suffix=n) for n in names]
    k1, k2 = ['lambda_sterics' + ('' if n is None else '_' + n) for n in names]
    ts_own = states.create_thermodynamic_state_protocol(own, {k1: l1, k2: l2}, constants={'temperature': 300.0 * u.kelvin},
                                                        composable_states=comp)
    _, t_rec = _backend.engine_tables(ts_rec)
    _, t_own = _backend.engine_tables(ts_own)
    for k in ('temperature', 'lambda_sterics', 'lambda_sterics_2'):
        assert np.array_equal(t_rec[k], t_own[k]), k
    assert np.allclose(t_rec['energy_offset'], t_own['energy_offset'], rtol=1e-12, atol=0)
