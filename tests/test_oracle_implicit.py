"""OBC implicit solvent in the CPU oracle (oracle/rx_oracle_gb.c): AMBER radii and screening factors, the model against a
numpy restatement, forces against finite differences, analytic limits, and AMBER 9 sander's single-point energies of the
T4-lysozyme L99A ligand (igb=2, which is OBC1)."""
import os
import numpy as np
import pytest
import helpers as H
import implicit_helpers as IH
from openmmtools_b200 import amber, testsystems
from oracle import oracle, implicit

KCAL = 4.184


def test_alanine_dipeptide_radii_are_mbondi2():
    d = amber.read_prmtop(os.path.join(IH.GOLDEN, 'alanine-dipeptide.prmtop'))
    s = testsystems.AlanineDipeptideImplicit().system
    assert np.array_equal(s.gb_radius, d['radii']) and np.array_equal(s.gb_scale, d['screen'])
    assert d['radius_set'] == 'H(N)-modified Bondi radii (mbondi2)'
    heavy = {}
    for b in d['bonds']:
        heavy.setdefault(b[0], []).append(b[1]); heavy.setdefault(b[1], []).append(b[0])
    for i, name in enumerate(d['names']):
        if name.startswith('H'):
            on_n = any(d['names'][j].startswith('N') for j in heavy[i])
            assert s.gb_radius[i] == pytest.approx(0.13 if on_n else 0.12, abs=1e-15), (i, name)
    assert s.gb_parameters == (0.8, 0.0, 2.909125, 0.009, 1.0, 78.5, 2.25936, 0.14)


def test_toluene_radii_are_mbondi():
    d = amber.read_prmtop(os.path.join(IH.GOLDEN, 'toluene-solvent.prmtop'))
    s = testsystems.TolueneImplicit().system
    assert np.array_equal(s.gb_radius, d['radii']) and np.array_equal(s.gb_scale, d['screen'])
    assert d['radius_set'] == 'modified Bondi radii (mbondi)'
    h = np.array([n.startswith('H') for n in d['names']])
    assert np.allclose(s.gb_radius[h], 0.13, atol=1e-15) and np.allclose(s.gb_radius[~h], 0.17, atol=1e-15)
    x = amber.read_inpcrd(os.path.join(IH.GOLDEN, 'toluene-solvent.inpcrd'))
    assert np.array_equal(testsystems.TolueneImplicit().positions._value, x)
    assert testsystems.TolueneImplicitOBC2().system.gb_parameters[:3] == (1.0, 0.8, 4.85)
    assert testsystems.TolueneImplicitOBC1().system.gb_parameters[:3] == (0.8, 0.0, 2.909125)
    assert testsystems.TolueneVacuum().system.gb_radius is None


def _cases():
    out = {}
    for name in ('alanine-dipeptide', 'toluene'):
        out[name] = lambda name=name: IH.implicit_system(name)
    out['t4-ligand'] = lambda: IH.ligand()
    for name, build in (('decane', lambda: H.alkane(10)), ('waters-ion', lambda: H.waters(10, ions=1, shuffle=3)),
                        ('mixture', lambda: H.mixture()), ('diatomic', lambda: H.diatomic()), ('ion', lambda: H.ion())):
        out[name] = lambda build=build: (lambda s, x: (IH.obc(s), x))(*build())
    return out


CASES = _cases()


@pytest.mark.parametrize('ace', [True, False])
@pytest.mark.parametrize('model', ['OBC1', 'OBC2'])
@pytest.mark.parametrize('name', list(CASES))
def test_oracle_matches_a_numpy_restatement(name, model, ace):
    s, x = CASES[name]()
    s = IH.with_model(s, model, ace)
    rng = np.random.default_rng(1)
    for xk in (x, x + rng.normal(0, 0.003, x.shape)):
        ref = IH.numpy_gb_energy(s, xk)
        m = implicit.Molecule(s)
        assert abs(m.gb_energy(xk) - ref) <= 1e-12 * max(1.0, abs(ref)), (m.gb_energy(xk), ref)
        # (the total is the vacuum force field plus the GB energy)
        vac = s.copy(); vac.gb_radius = None
        assert abs(m.energy(xk) - (oracle.Molecule(vac).energy(xk) + ref)) <= 1e-12 * max(1.0, abs(m.energy(xk)))


@pytest.mark.parametrize('model', ['OBC1', 'OBC2'])
@pytest.mark.parametrize('name', ['alanine-dipeptide', 'toluene', 't4-ligand', 'waters-ion', 'mixture'])
def test_oracle_forces_are_the_gradient_of_its_energy(name, model):
    s, x = CASES[name]()
    m = implicit.Molecule(IH.with_model(s, model))
    x = x + np.random.default_rng(2).normal(0, 0.002, x.shape)
    for energy in (m.gb_energy, m.energy):
        _, f = energy(x, forces=True)
        h = 1e-6
        fd = np.zeros_like(x)
        for i in range(len(x)):
            for c in range(3):
                xp, xm = x.copy(), x.copy()
                xp[i, c] += h; xm[i, c] -= h
                fd[i, c] = -(energy(xp) - energy(xm)) / (2 * h)
        assert np.abs(f - fd).max() <= 1e-5 * np.abs(f).max(), np.abs(f - fd).max() / np.abs(f).max()


def test_one_ion_is_its_self_energy_plus_ace():
    s, x = H.ion()
    s = IH.obc(s)
    rho = s.gb_radius[0]
    rt = rho - 0.009
    P = -138.935456 * (1.0 - 1.0 / 78.5)
    ace = 4 * np.pi * 2.25936 * (rho + 0.14) ** 2 * (rho / rt) ** 6
    assert abs(implicit.Molecule(s).gb_energy(x) - (0.5 * P / rt + ace)) <= 1e-12 * abs(0.5 * P / rt)


def test_two_distant_ions_screen_coulomb_by_the_solvent_dielectric():
    s, x = H.ion(2)
    s.charge = np.array([1.0, -1.0])
    s = IH.obc(s, ace=False)
    x = np.array([[0.0, 0.0, 0.0], [10.0, 0.0, 0.0]])
    m = implicit.Molecule(s)
    B, _ = m.born_radii(x)
    P = -138.935456 * (1.0 - 1.0 / 78.5)
    expected = -138.935456 / (78.5 * 10.0) + 0.5 * P * (1.0 / B[0] + 1.0 / B[1])
    assert abs(m.energy(x) - expected) <= 1e-6 * abs(expected)


@pytest.mark.parametrize('name', ['alanine-dipeptide', 'toluene', 't4-ligand'])
def test_no_shipped_molecule_has_an_engulfed_pair(name):
    s, x = CASES[name]()
    if name == 't4-ligand':
        xs = [x, IH.ligand(coordinates='ligand-minimized.crd')[1]]
    else:
        xs = [x]
    for xk in xs:
        B, engulfed = implicit.Molecule(s).born_radii(xk)
        assert engulfed == 0 and np.all(B > 0)


def _component(s, keep):
    """The system with only one energy component left (exclusions kept: exceptions are zeroed, not removed)."""
    c = s.copy()
    c.gb_radius = None
    zero = lambda w: np.zeros((0, w))
    if keep != 'bond': c.bonds = zero(4)
    if keep != 'angle': c.angles = zero(5)
    if keep != 'dihedral': c.torsions = zero(7)
    if keep != 'eel': c.charge = np.zeros_like(c.charge)
    if keep != 'vdw': c.epsilon = np.zeros_like(c.epsilon)
    c.exceptions = c.exceptions.copy()
    if keep != '14eel': c.exceptions[:, 2] = 0.0
    if keep != '14vdw': c.exceptions[:, 4] = 0.0
    return c


@pytest.mark.parametrize('coordinates,sander_out', [('ligand.crd', 'ligand-min.sander.out'),
                                                     ('ligand-minimized.crd', 'ligand-testenergy.sander.out')])
def test_ligand_components_match_sander(coordinates, sander_out):
    s, x = IH.ligand(coordinates=coordinates)
    e = IH.sander_energies(os.path.join(IH.GOLDEN, 't4-' + sander_out))
    scale = IH.SANDER_ELEC_SCALE
    ref = {'angle': e['ANGLE'], 'dihedral': e['DIHED'], '14vdw': e.get('1-4 VDW', e.get('1-4 NB')),
           '14eel': e['1-4 EEL'] * scale, 'vdw': e['VDWAALS'], 'eel': e.get('EEL', e.get('EELEC')) * scale}
    if coordinates == 'ligand.crd':   # (ntf=2 in the other run: its BOND leaves out the bonds to hydrogen)
        ref['bond'] = e['BOND']
    for k, v in ref.items():
        mine = oracle.Molecule(_component(s, k)).energy(x) / KCAL
        assert abs(mine - v) <= 1e-4, (k, mine, v)
    egb = implicit.Molecule(s).gb_energy(x) / KCAL
    assert abs(egb - e['EGB'] * scale) <= 1e-4, (egb, e['EGB'] * scale)


def test_vacuum_hash_is_unchanged_and_implicit_hash_differs():
    vac = testsystems.AlanineDipeptideVacuum().system
    imp = testsystems.AlanineDipeptideImplicit().system
    # the hash of the vacuum system as the parent commit computed it (no GB fields)
    import hashlib
    h = hashlib.sha1()
    h.update(vac.kind.encode()); h.update(vac.masses.tobytes())
    for a in (vac.sigma, vac.epsilon, vac.charge, vac.bonds, vac.angles, vac.torsions, vac.exclusions, vac.exceptions,
              vac.constraints):
        h.update(np.asarray(a, dtype=np.float64).tobytes())
    h.update(repr(vac.remove_cm_motion).encode())
    assert vac.standard_hash() == h.hexdigest()
    assert imp.standard_hash() != vac.standard_hash()
    assert testsystems.TolueneImplicitOBC2().system.standard_hash() != testsystems.TolueneImplicitOBC1().system.standard_hash()


@pytest.mark.parametrize('cls', ['TolueneImplicitHCT', 'TolueneImplicitGBn', 'TolueneImplicitGBn2'])
def test_other_gb_models_are_refused(cls):
    with pytest.raises(NotImplementedError):
        getattr(testsystems, cls)()


@pytest.mark.parametrize('kwargs', [dict(implicitSolventKappa=1.0), dict(implicitSolventSaltConc=0.15),
                                    dict(nonbondedCutoff=1.0), dict(nonbondedMethod='CutoffNonPeriodic'),
                                    dict(hydrogenMass=4.0)])
def test_salt_cutoffs_and_repartitioning_are_refused(kwargs):
    with pytest.raises(NotImplementedError):
        testsystems.TolueneImplicit(**kwargs)


def test_constructor_signatures_match_the_reference():
    """Argument names and defaults of the reference's classes (tests/golden/implicit_signatures_golden.json); the reference's
    app.HBonds default is the string 'HBonds' here."""
    import inspect, json
    gold = json.load(open(os.path.join(IH.GOLDEN, 'implicit_signatures_golden.json')))
    for name, g in gold.items():
        p = inspect.signature(getattr(testsystems, name).__init__).parameters
        mine = [[k, None if v.default is inspect.Parameter.empty else repr(v.default)] for k, v in p.items()
                if k != 'self' and v.kind != inspect.Parameter.VAR_KEYWORD]
        ref = [[k, {'app.HBonds': "'HBonds'"}.get(d, d)] for k, d in g['args']]
        assert mine == ref, (name, mine, ref)
        assert any(v.kind == inspect.Parameter.VAR_KEYWORD for v in p.values()) == (g['kwarg'] is not None), name
