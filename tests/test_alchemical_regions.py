"""Two alchemical regions on the host: the factory's checks and records, suffixed AlchemicalStates, the engine tables
and the dispersion corrections (no GPU)."""
import copy
import pickle
import numpy as np
import pytest
from openmmtools_b200 import alchemy, states, testsystems, unit, _backend
from openmmtools_b200.alchemy import AlchemicalRegion, AlchemicalState, AbsoluteAlchemicalFactory


def fluid(N=64, dispersion=True):
    f = testsystems.LennardJonesFluid(nparticles=N, dispersion_correction=dispersion)
    return f.system


def two_regions(system, names=('A', 'B'), ann=(False, True), atoms=(range(0, 3), range(3, 5)), **kw):
    regions = [AlchemicalRegion(alchemical_atoms=atoms[0], name=names[0], annihilate_sterics=ann[0], **kw),
               AlchemicalRegion(alchemical_atoms=atoms[1], name=names[1], annihilate_sterics=ann[1], **kw)]
    return AbsoluteAlchemicalFactory().create_alchemical_system(system, regions)


def test_factory_records_regions_and_suffixed_parameters():
    s = two_regions(fluid())
    assert s.alchemical_regions == (('A', (0, 1, 2), False), ('B', (3, 4), True))
    assert s.alchemical_atoms == (0, 1, 2, 3, 4)
    assert list(s.alchemical_region_ids()[:6]) == [1, 1, 1, 2, 2, 0]
    for n in ('lambda_sterics_A', 'lambda_electrostatics_A', 'lambda_sterics_B', 'lambda_electrostatics_B'):
        assert s.global_parameters[n] == 1.0
    assert 'lambda_sterics' not in s.global_parameters
    s2 = two_regions(fluid(), names=(None, 'B'))
    assert s2.lambda_sterics_names() == ('lambda_sterics', 'lambda_sterics_B')
    # a single region keeps the one-region record (and the standard hash of before)
    one = AbsoluteAlchemicalFactory().create_alchemical_system(fluid(), AlchemicalRegion(alchemical_atoms=range(3)))
    assert one.alchemical_regions is None
    assert one.standard_hash() != two_regions(fluid()).standard_hash()


def test_factory_refusals():
    f = AbsoluteAlchemicalFactory()
    r = lambda atoms, **kw: AlchemicalRegion(alchemical_atoms=atoms, **kw)
    with pytest.raises(ValueError):
        f.create_alchemical_system(fluid(), [r([0, 1], name='A'), r([1, 2], name='B')])
    with pytest.raises(ValueError):
        f.create_alchemical_system(fluid(), [r([0, 1], name='A'), r([2, 3], name='A')])
    with pytest.raises(ValueError):
        f.create_alchemical_system(fluid(), [r([0, 1]), r([2, 3])])
    with pytest.raises(NotImplementedError):
        f.create_alchemical_system(fluid(), [r([0], name='A'), r([1], name='B')],
                                   alchemical_regions_interactions=frozenset([(0, 1)]))
    with pytest.raises(NotImplementedError):
        f.create_alchemical_system(fluid(), [r([0], name='A'), r([1], name='B'), r([2], name='C')])
    with pytest.raises(NotImplementedError):
        f.create_alchemical_system(fluid(), [r([0], name='A'), r([1], name='B', softcore_alpha=0.3)])


def test_suffixed_alchemical_state():
    s = two_regions(fluid())
    a = AlchemicalState.from_system(s, parameters_name_suffix='A')
    b = AlchemicalState.from_system(s, parameters_name_suffix='B')
    assert a.lambda_sterics_A == 1.0 and b.lambda_sterics_B == 1.0
    a.lambda_sterics_A = 0.25
    assert a.lambda_sterics_A == 0.25
    with pytest.raises(ValueError):
        a.lambda_sterics_A = 1.5
    with pytest.raises(AttributeError):
        a.lambda_sterics
    with pytest.raises(AttributeError):
        a.lambda_sterics = 0.5
    with pytest.raises(AttributeError):
        a.lambda_sterics_B
    c = AlchemicalState(parameters_name_suffix='A', lambda_sterics=0.5)
    assert c.lambda_sterics_A == 0.5 and c._parameters['lambda_electrostatics_A'] is None
    # serialised under the unsuffixed names plus the suffix (states.py:3879-3898)
    st = a.__getstate__()
    assert st['_parameters_name_suffix'] == 'A' and st['_parameters']['lambda_sterics'] == 0.25
    for back in (pickle.loads(pickle.dumps(a)), copy.deepcopy(a)):
        assert back == a and back.lambda_sterics_A == 0.25
    a.set_alchemical_parameters(0.0)
    assert a.lambda_sterics_A == 0.0 and a.lambda_electrostatics_A == 0.0
    # an unsuffixed state is unchanged
    u = AlchemicalState(lambda_sterics=0.3)
    assert u.lambda_sterics == 0.3 and u.__getstate__()['_parameters_name_suffix'] is None


def protocol(system, l1, l2, names=('A', 'B')):
    comp = [AlchemicalState.from_system(system, parameters_name_suffix=n) for n in names]
    k1, k2 = ['lambda_sterics' + ('' if n is None else '_' + n) for n in names]
    return states.create_thermodynamic_state_protocol(system, {k1: list(l1), k2: list(l2)},
                                                      constants={'temperature': 300.0 * unit.kelvin},
                                                      composable_states=comp)


def test_protocol_and_engine_tables():
    s = two_regions(fluid())
    l1, l2 = [1.0, 0.5, 0.0], [0.0, 0.5, 1.0]
    ts = protocol(s, l1, l2)
    assert [t.lambda_sterics_A for t in ts] == l1 and [t.lambda_sterics_B for t in ts] == l2
    p = ts[1]._engine_parameters()
    assert p['lambda_sterics_A'] == 0.5 and p['lambda_sterics_B'] == 0.5
    sys0, tab = _backend.engine_tables(ts)
    assert np.array_equal(tab['lambda_sterics'], l1) and np.array_equal(tab['lambda_sterics_2'], l2)
    for l in range(3):
        want = _backend.lj_dispersion_correction(s) + _backend.alchemical_dispersion_correction(s, l1[l], l2[l])
        assert tab['energy_offset'][l] == want
    # the whole compound state survives a round trip
    back = pickle.loads(pickle.dumps(ts[1]))
    assert back.lambda_sterics_A == 0.5 and back.lambda_sterics_B == 0.5
    # a region named None takes the unsuffixed parameter
    s2 = two_regions(fluid(), names=(None, 'B'))
    ts2 = protocol(s2, l1, l2, names=(None, 'B'))
    _, tab2 = _backend.engine_tables(ts2)
    assert np.array_equal(tab2['lambda_sterics'], l1) and np.array_equal(tab2['lambda_sterics_2'], l2)
    # NPT: the dispersion coefficients use both lambdas
    ts3 = [states.CompoundThermodynamicState(states.ThermodynamicState(s, 300.0 * unit.kelvin, 1.0 * unit.bar), t._composable_states)
           for t in ts]
    p3, c3 = _backend.pressure_tables(ts3)
    V = abs(np.linalg.det(s.box_vectors))
    assert np.allclose(c3, (tab['energy_offset']) * V, rtol=1e-14)


def with_eps_zero(system, atoms):
    t = system.copy()
    t.epsilon = np.array(t.epsilon, np.float64)
    t.epsilon[list(atoms)] = 0.0
    return t


@pytest.mark.parametrize('ann', [(False, False), (False, True), (True, True)])
def test_dispersion_correction_is_the_sum_of_the_regions(ann):
    """Two regions = region A alone with B's epsilons zeroed + region B alone with A's epsilons zeroed: every
    environment x r and r x r class pair exactly once, no A x B pair (alchemy.py:1684-1685, 1774-1777)."""
    N = 64
    ref = fluid(N)
    t = ref.copy()
    t.epsilon = np.where(np.arange(N) % 3 == 0, 0.9, 1.3) * np.asarray(ref.epsilon)   # two epsilon classes
    t.sigma = np.where(np.arange(N) % 2 == 0, 0.30, 0.36)
    A, B = [0, 1, 2, 7], [3, 4, 9]
    s = two_regions(t, ann=ann, atoms=(A, B))
    fa = AbsoluteAlchemicalFactory()
    one_a = fa.create_alchemical_system(with_eps_zero(t, B), AlchemicalRegion(alchemical_atoms=A, annihilate_sterics=ann[0]))
    one_b = fa.create_alchemical_system(with_eps_zero(t, A), AlchemicalRegion(alchemical_atoms=B, annihilate_sterics=ann[1]))
    for l1, l2 in [(1.0, 1.0), (0.3, 0.8), (0.0, 0.45), (1.0, 0.0)]:
        got = _backend.alchemical_dispersion_correction(s, l1, l2)
        want = _backend.alchemical_dispersion_correction(one_a, l1) + _backend.alchemical_dispersion_correction(one_b, l2)
        assert abs(got - want) <= 1e-12 * abs(want), (l1, l2, got, want)
    # the NonbondedForce correction counts the atoms of both regions with epsilon 0 (alchemy.py:1903-1909)
    assert _backend.lj_dispersion_correction(s) == _backend.lj_dispersion_correction(
        fa.create_alchemical_system(t, AlchemicalRegion(alchemical_atoms=A + B)))


def test_region_with_zero_epsilon_is_invisible_and_names_swap():
    """Region B with epsilon 0 everywhere: the corrections are those of region A alone; swapping the regions' names
    and lambdas changes nothing."""
    N = 64
    t = fluid(N)
    A, B = [0, 5, 6], [10, 11]
    z = with_eps_zero(t, B)
    s = two_regions(z, atoms=(A, B))
    one = AbsoluteAlchemicalFactory().create_alchemical_system(z, AlchemicalRegion(alchemical_atoms=A))
    assert abs(_backend.lj_dispersion_correction(s) - _backend.lj_dispersion_correction(one)) <= 1e-12 * abs(
        _backend.lj_dispersion_correction(one))
    swapped = two_regions(t, names=('B', 'A'), ann=(True, False), atoms=(B, A))
    s = two_regions(t, atoms=(A, B))
    for l1, l2 in [(0.2, 0.9), (1.0, 0.0)]:
        assert abs(_backend.alchemical_dispersion_correction(s, l1, l2) -
                   _backend.alchemical_dispersion_correction(swapped, l2, l1)) <= 1e-12 * abs(
            _backend.alchemical_dispersion_correction(s, l1, l2))
        zs = two_regions(z, atoms=(A, B))
        assert abs(_backend.alchemical_dispersion_correction(zs, l1, l2) -
                   _backend.alchemical_dispersion_correction(one, l1)) <= 1e-12 * abs(
            _backend.alchemical_dispersion_correction(one, l1))
