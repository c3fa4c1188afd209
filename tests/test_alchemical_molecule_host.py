"""Alchemical small molecules on the host: the factory's bookkeeping and refusals, and the float64 oracle
(oracle/alchemical_molecule.py) against the unmodified molecule oracles at the end states and against finite differences."""
import numpy as np
import pytest
from openmmtools_b200 import alchemy, testsystems, unit, states
from openmmtools_b200.alchemy import AbsoluteAlchemicalFactory, AlchemicalRegion, AlchemicalState


def _x(t):
    return np.ascontiguousarray(t.positions.value_in_unit(unit.nanometer), np.float64)


SYSTEMS = {
    'toluene-vacuum': (testsystems.TolueneVacuum, range(15)),
    'toluene-obc1': (testsystems.TolueneImplicit, range(15)),
    'toluene-obc2': (testsystems.TolueneImplicitOBC2, range(15)),
    'aladip-vacuum': (testsystems.AlanineDipeptideVacuum, range(22)),
    'aladip-obc1': (testsystems.AlanineDipeptideImplicit, range(22)),
    'toluene-obc1-partial': (testsystems.TolueneImplicit, range(7, 15)),
    'toluene-obc2-partial': (testsystems.TolueneImplicitOBC2, [0, 3, 9, 10]),
    'aladip-vacuum-partial': (testsystems.AlanineDipeptideVacuum, range(6, 12)),
}


def _make(name, **region):
    cls, atoms = SYSTEMS[name]
    t = cls()
    return t, AbsoluteAlchemicalFactory().create_alchemical_system(t.system, AlchemicalRegion(alchemical_atoms=atoms, **region))


def _unmodified(system):
    from oracle import oracle, implicit
    return oracle.Molecule(system) if system.gb_radius is None else implicit.Molecule(system)


def _with_obc2_literals(system):
    """The unmodified OBC2 system with the alchemical expression's constants: 138.935485 for 138.935456 (through the solute
    dielectric, which the oracle multiplies by 138.935456) and 28.3919551 for 4 pi sa_energy."""
    s = system.copy()
    g = list(s.gb_parameters)
    k = (1.0 / g[4] - 1.0 / g[5]) * 138.935485 / 138.935456
    g[4] = 1.0 / (k + 1.0 / g[5])
    g[6] = 28.3919551 / (4.0 * np.pi)
    s.gb_parameters = tuple(g)
    return s


@pytest.mark.parametrize('name', sorted(SYSTEMS))
def test_oracle_at_lambda_one_is_the_unmodified_molecule(name):
    from oracle.alchemical_molecule import AlchemicalMolecule
    t, asys = _make(name)
    ref = t.system if not asys.alchemical_obc2 else _with_obc2_literals(t.system)
    x = _x(t)
    e0 = _unmodified(ref).energy(x)
    e1 = AlchemicalMolecule(asys).energy(x, 1.0, 1.0)
    assert abs(e1 - e0) <= 1e-12 * abs(e0), (e1, e0)


@pytest.mark.parametrize('name', ['toluene-obc1', 'toluene-obc2', 'aladip-obc1', 'toluene-obc1-partial', 'toluene-obc2-partial'])
def test_gb_at_lambda_electrostatics_zero_drops_the_alchemical_charges_screening_and_ace(name):
    """w = 0: an unmodified model with the alchemical charges and screening factors zeroed and their ACE terms dropped."""
    from oracle.alchemical_molecule import AlchemicalMolecule
    from oracle import implicit
    t, asys = _make(name)
    mask = asys.alchemical_mask().astype(bool)
    ref = (_with_obc2_literals if asys.alchemical_obc2 else lambda s: s.copy())(t.system)
    ref.charge = np.where(mask, 0.0, ref.charge)
    ref.gb_scale = np.where(mask, 0.0, ref.gb_scale)
    x = _x(t)
    m = implicit.Molecule(ref)
    B, engulfed = m.born_radii(x)
    assert engulfed == 0
    alpha, beta, gamma, offset, e_in, e_out, sa, probe = ref.gb_parameters
    rho = np.asarray(ref.gb_radius)
    ace = 4.0 * np.pi * sa * (rho + probe) ** 2 * (rho / B) ** 6
    expect = m.gb_energy(x) - ace[mask].sum()
    got = AlchemicalMolecule(asys).gb_energy(x, 0.0)
    assert abs(got - expect) <= 1e-12 * max(abs(expect), 1.0), (got, expect)


@pytest.mark.parametrize('name', ['toluene-vacuum', 'aladip-vacuum', 'aladip-vacuum-partial'])
def test_annihilated_sterics_vanish_at_lambda_sterics_zero(name):
    from oracle.alchemical_molecule import AlchemicalMolecule
    from oracle import oracle
    t, asys = _make(name, annihilate_sterics=True)
    mask = asys.alchemical_mask().astype(bool)
    ref = t.system.copy()
    ref.epsilon = np.where(mask, 0.0, ref.epsilon)
    exc = np.array(ref.exceptions)
    exc[mask[exc[:, 0].astype(int)] | mask[exc[:, 1].astype(int)], 4] = 0.0
    ref.exceptions = exc
    x = _x(t)
    e0 = oracle.Molecule(ref).energy(x)
    e1 = AlchemicalMolecule(asys).energy(x, 0.0, 1.0)
    assert abs(e1 - e0) <= 1e-12 * abs(e0), (e1, e0)


@pytest.mark.parametrize('name', ['toluene-vacuum', 'toluene-obc1', 'toluene-obc2-partial', 'aladip-obc1'])
@pytest.mark.parametrize('annihilate', [False, True])
def test_oracle_forces_are_the_gradient_of_its_energy(name, annihilate):
    from oracle.alchemical_molecule import AlchemicalMolecule
    t, asys = _make(name, annihilate_sterics=annihilate)
    m = AlchemicalMolecule(asys)
    x = _x(t)
    rng = np.random.default_rng(5)
    x = x + rng.normal(0, 0.003, x.shape)
    lam = (0.4, 0.7)
    _, F = m.energy(x, *lam, forces=True)
    h = 1e-6
    for a in range(0, x.shape[0], 3):
        for c in range(3):
            xp, xm = x.copy(), x.copy()
            xp[a, c] += h; xm[a, c] -= h
            fd = -(m.energy(xp, *lam) - m.energy(xm, *lam)) / (2 * h)
            assert abs(F[a, c] - fd) <= 1e-5 * max(1.0, np.abs(F).max()), (a, c, F[a, c], fd)


def _engulfed():
    from alchemical_cases import make
    from oracle.alchemical_molecule import AlchemicalMolecule
    from oracle import implicit
    s, x, asys = make('engulfed-methane-obc2')
    x = x + np.random.default_rng(9).normal(0, 0.003, x.shape)
    B, engulfed = implicit.Molecule(s).born_radii(x)
    assert engulfed == 4 and np.all(B > 0)        # every (H, C) pair: sr_C - r > rt_H
    return s, x, asys, AlchemicalMolecule(asys)


@pytest.mark.parametrize('le', [0.0, 0.5, 1.0])
def test_oracle_forces_are_the_gradient_of_its_energy_at_engulfed_pairs(le):
    """The alchemical OBC2 expression's engulfment term C = 2 (1/rt_i - 1/L) step(sr_j - r - rt_i) and its force."""
    _, x, _, m = _engulfed()
    _, F = m.energy(x, 0.7, le, forces=True)
    h = 1e-6
    for a in range(x.shape[0]):
        for c in range(3):
            xp, xm = x.copy(), x.copy()
            xp[a, c] += h; xm[a, c] -= h
            fd = -(m.energy(xp, 0.7, le) - m.energy(xm, 0.7, le)) / (2 * h)
            assert abs(F[a, c] - fd) <= 1e-6 * max(1.0, np.abs(F).max()), (a, c, F[a, c], fd)


def test_engulfment_term_is_continuous_at_its_boundary_and_vanishes_without_engulfed_pairs():
    """Moving one hydrogen along its bond through r = sr_C - rt_H, where C = 0 (L = rt_H): no jump in energy, forces the
    gradient on both sides.  Stretched so that no pair is engulfed, the molecule at lambda 1 is the unmodified OBC2 model; at
    its own geometry it is not (the term is on)."""
    from oracle import implicit
    s, x, asys, m = _engulfed()
    rt, sr = s.gb_radius[1] - s.gb_parameters[3], s.gb_scale[0] * (s.gb_radius[0] - s.gb_parameters[3])
    edge = sr - rt
    u = (x[1] - x[0]) / np.linalg.norm(x[1] - x[0])
    at = lambda r: np.concatenate([x[:1], [x[0] + r * u], x[2:]])
    for le in (0.0, 0.5, 1.0):
        Fmax = np.abs(m.energy(at(edge), 0.7, le, forces=True)[1]).max()
        d = 1e-7
        assert abs(m.energy(at(edge + d), 0.7, le) - m.energy(at(edge - d), 0.7, le)) <= 2 * d * Fmax * 1.01
        for r in (edge - 2e-3, edge + 2e-3):
            _, F = m.energy(at(r), 0.7, le, forces=True)
            h = 1e-6
            fd = -(m.energy(at(r + h), 0.7, le) - m.energy(at(r - h), 0.7, le)) / (2 * h)
            assert abs(F[1] @ u - fd) <= 1e-6 * max(1.0, Fmax), (le, r, F[1] @ u, fd)
    ref = _with_obc2_literals(s)
    xs = x[0] + 1.8 * (x - x[0])           # hydrogens 0.196 nm out: past the boundary
    assert implicit.Molecule(ref).born_radii(xs)[1] == 0
    e0, e1 = implicit.Molecule(ref).energy(xs), m.energy(xs, 1.0, 1.0)
    assert abs(e1 - e0) <= 1e-12 * abs(e0), (e1, e0)
    assert abs(m.energy(x, 1.0, 1.0) - implicit.Molecule(ref).energy(x)) > 1.0


def test_alchemical_cases_of_the_device_tests_build_and_reach_what_they_are_for():
    """tests/alchemical_cases.py: each case has the region, the pair table and the flags its device tests rely on."""
    import alchemical_cases as A
    from oracle.alchemical_molecule import AlchemicalMolecule
    got = {}
    for name, swapped in A.variants():
        s, x, asys = A.make(name, swapped)
        got[name, swapped] = (asys, AlchemicalMolecule(asys))
    a, m = got['decane-obc2-top', False]
    assert a.n_particles == 32 and 31 in a.alchemical_atoms and a.alchemical_obc2
    a, m = got['decane-all-annihilated', False]
    n = a.n_particles
    n_plain = n * (n - 1) // 2 - len(a.exclusions) - len(a.exceptions)
    assert len(m.pairs) == n_plain + len(a.exceptions) and all(p[5] and p[6] for p in m.pairs)   # no plain pair
    assert len(got['methane-obc1-carbon', False][1].pairs) == 0
    assert got['ion-obc1', False][0].n_particles == 1
    for c in ('torsion-probe-sc-c4', 'torsion-probe-sc-c12'):
        a = got[c, False][0]
        assert a.softcore_c != 6 and a.softcore_a == 2 and a.softcore_b == 2 and a.softcore_alpha == 0.3
        assert len(got[c, False][1].pairs) == 2
    # the swapped flags change which lambdas the alchemical/alchemical pairs follow
    for c in A.SWAPPED:
        assert [p[5:] for p in got[c, False][1].pairs] != [p[5:] for p in got[c, True][1].pairs], c


def test_factory_records_the_region_and_the_lambdas():
    t, asys = _make('toluene-obc2-partial', annihilate_sterics=True, annihilate_electrostatics=False)
    assert asys.alchemical_atoms == (0, 3, 9, 10)
    assert asys.annihilate_sterics and not asys.annihilate_electrostatics
    assert asys.alchemical_obc2 and not t.system.is_alchemical
    assert asys.global_parameters['lambda_sterics'] == 1.0 and asys.global_parameters['lambda_electrostatics'] == 1.0
    assert asys.standard_hash() != t.system.standard_hash()
    # a copy of the reference keeps its hash (other molecules' hashes are unchanged)
    assert t.system.copy().standard_hash() == testsystems.TolueneImplicitOBC2().system.standard_hash()
    _, obc1 = _make('toluene-obc1')
    assert not obc1.alchemical_obc2
    a = AlchemicalState.from_system(asys)
    a.lambda_electrostatics, a.lambda_sterics = 0.25, 0.5
    protocol = {'lambda_electrostatics': [1.0, 0.5, 0.0], 'lambda_sterics': [1.0, 1.0, 0.25]}
    tss = states.create_thermodynamic_state_protocol(asys, protocol, constants={'temperature': 300 * unit.kelvin},
                                                     composable_states=a)
    from openmmtools_b200 import _backend
    _, tab = _backend.engine_tables(tss)
    assert list(tab['lambda_electrostatics']) == [1.0, 0.5, 0.0]
    assert list(tab['lambda_sterics']) == [1.0, 1.0, 0.25]
    # a protocol varying temperature and the lambdas together
    tss2 = states.create_thermodynamic_state_protocol(
        asys, {'temperature': [300 * unit.kelvin, 310 * unit.kelvin], 'lambda_electrostatics': [1.0, 0.0]},
        composable_states=AlchemicalState.from_system(asys))
    _, tab2 = _backend.engine_tables(tss2)
    assert list(tab2['lambda_electrostatics']) == [1.0, 0.0] and tab2['temperature'][1] == 310.0


def test_non_alchemical_tables_carry_no_electrostatic_lambda():
    from openmmtools_b200 import _backend
    t = testsystems.TolueneImplicit()
    tss = [states.ThermodynamicState(t.system, T * unit.kelvin) for T in (300, 320)]
    _, tab = _backend.engine_tables(tss)
    assert 'lambda_electrostatics' not in tab


@pytest.mark.parametrize('kw, exc', [
    (dict(alchemical_bonds=True), NotImplementedError),
    (dict(alchemical_angles=[0]), NotImplementedError),
    (dict(alchemical_torsions=True), NotImplementedError),
    (dict(softcore_beta=0.5), NotImplementedError),
    (dict(softcore_d=2), NotImplementedError),
    (dict(softcore_e=2), NotImplementedError),
    (dict(softcore_f=1), NotImplementedError),
])
def test_factory_refuses_what_molecules_do_not_provide(kw, exc):
    t = testsystems.TolueneImplicit()
    with pytest.raises(exc):
        AbsoluteAlchemicalFactory().create_alchemical_system(t.system, AlchemicalRegion(alchemical_atoms=range(3), **kw))


def test_factory_refuses_two_regions_consistent_exceptions_and_foreign_obc2_constants():
    t = testsystems.TolueneImplicitOBC2()
    two = [AlchemicalRegion(alchemical_atoms=range(3), name='A'), AlchemicalRegion(alchemical_atoms=range(3, 6), name='B')]
    with pytest.raises(NotImplementedError):
        AbsoluteAlchemicalFactory().create_alchemical_system(t.system, two)
    with pytest.raises(NotImplementedError):
        AbsoluteAlchemicalFactory(consistent_exceptions=True).create_alchemical_system(
            t.system, AlchemicalRegion(alchemical_atoms=range(3)))
    for field, value in ((3, 0.01), (6, 2.0), (7, 0.15)):   # offset, surface-area energy, probe radius
        s = t.system.copy()
        g = list(s.gb_parameters); g[field] = value; s.gb_parameters = tuple(g)
        with pytest.raises(NotImplementedError):
            AbsoluteAlchemicalFactory().create_alchemical_system(s, AlchemicalRegion(alchemical_atoms=range(3)))
    # OBC1 carries no literals of its own: other constants are its own
    s = testsystems.TolueneImplicit().system
    g = list(s.gb_parameters); g[6] = 2.0; s.gb_parameters = tuple(g)
    AbsoluteAlchemicalFactory().create_alchemical_system(s, AlchemicalRegion(alchemical_atoms=range(3)))
    with pytest.raises(ValueError):
        AbsoluteAlchemicalFactory().create_alchemical_system(t.system, AlchemicalRegion(alchemical_atoms=[15]))
    asys = AbsoluteAlchemicalFactory().create_alchemical_system(t.system, AlchemicalRegion(alchemical_atoms=[0]))
    with pytest.raises(ValueError):
        AbsoluteAlchemicalFactory().create_alchemical_system(asys, AlchemicalRegion(alchemical_atoms=[0]))
