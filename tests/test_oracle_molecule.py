"""The small-molecule path on the CPU: the AMBER reader and the fixture of testsystems.AlanineDipeptideVacuum
(testsystems.py:3352-3388), the oracle's force field (forces = -grad U by finite differences) and its constrained Langevin
steps (integrators.py:1404-1460).  Parity with OpenMM itself is unpinned (not installable here); the energy at the input
geometry is pinned to this implementation's own value so that a regression shows."""
import copy
import json
import os
import sys
import numpy as np
import pytest
from openmmtools_b200 import testsystems, unit, amber
from oracle import oracle

HERE = os.path.dirname(os.path.abspath(__file__))
KB = 8.31446261815324e-3


def aladip():
    a = testsystems.AlanineDipeptideVacuum()
    return a, np.ascontiguousarray(a.positions.value_in_unit(unit.nanometer), np.float64)


def test_fixture_equals_a_fresh_parse_of_the_reference_files():
    # tests/golden/alanine-dipeptide.{prmtop,crd}: openmmtools' data files, unchanged
    sys.path.insert(0, os.path.join(HERE, 'golden'))
    import make_aladip_fixture as m
    fresh = json.loads(json.dumps(m.build()))
    stored = json.load(open(os.path.join(HERE, '..', 'openmmtools_b200', 'data', 'alanine_dipeptide_vacuum.json')))
    assert fresh == stored


def test_topology_counts_and_units():
    a, x = aladip()
    s = a.system
    assert s.n_particles == 22 and a.atom_names[:4] == ['HH31', 'CH3', 'HH32', 'HH33']
    assert abs(s.charge.sum()) < 1e-8 and abs(s.masses.sum() - 144.176) < 1e-9
    assert len(s.constraints) == 12 and len(s.bonds) == 9 and len(s.angles) == 36 and len(s.torsions) == 32
    assert len(s.exclusions) == 57 and len(s.exceptions) == 41 and s.getNumConstraints() == 12
    # every constrained bond involves a hydrogen and has its AMBER length; the input geometry satisfies it to 1e-7 nm
    for i, j, d in s.constraints:
        assert min(s.masses[int(i)], s.masses[int(j)]) < 1.1
        assert abs(np.linalg.norm(x[int(i)] - x[int(j)]) - d) < 2e-7
    # ff96 numbers: CT sigma 3.39967 A, epsilon 0.1094 kcal/mol; C-N bond 490 kcal/mol/A^2 at 1.335 A
    assert abs(s.sigma[1] - 0.339967) < 1e-6 and abs(s.epsilon[1] - 0.1094 * 4.184) < 1e-6
    cn = [b for b in s.bonds if {int(b[0]), int(b[1])} == {4, 6}][0]
    assert abs(cn[2] - 2 * 490.0 * 418.4) < 1e-6 and abs(cn[3] - 0.1335) < 1e-12
    # 1-4 pairs: Coulomb / 1.2, Lennard-Jones epsilon / 2
    i, j, qq, sg, ep = s.exceptions[0]
    i, j = int(i), int(j)
    assert abs(qq - s.charge[i] * s.charge[j] / 1.2) < 1e-15
    assert abs(ep - np.sqrt(s.epsilon[i] * s.epsilon[j]) / 2.0) < 1e-9 and abs(sg - 0.5 * (s.sigma[i] + s.sigma[j])) < 1e-9
    none = testsystems.AlanineDipeptideVacuum(constraints=None).system
    assert len(none.constraints) == 0 and len(none.bonds) == 21


def test_oracle_forces_are_the_gradient_of_the_energy():
    a, x = aladip()
    x = x + np.random.default_rng(0).normal(0, 0.005, x.shape)
    for constraints in ('HBonds', None):
        m = oracle.Molecule(testsystems.AlanineDipeptideVacuum(constraints=constraints).system)
        U, f = m.energy(x, forces=True)
        g = np.zeros_like(x); h = 1e-6
        for i in range(22):
            for c in range(3):
                xp = x.copy(); xp[i, c] += h; xm = x.copy(); xm[i, c] -= h
                g[i, c] = -(m.energy(xp) - m.energy(xm)) / (2 * h)
        assert np.abs(g - f).max() < 1e-5 * np.abs(f).max()
        assert np.abs(f.sum(0)).max() < 1e-8      # no net force


def test_energy_at_the_input_geometry_is_pinned():
    a, x = aladip()
    U = oracle.Molecule(a.system).energy(x)
    assert abs(U - (-88.08858703851178)) < 1e-9      # kJ/mol (this implementation's own value: -21.0537 kcal/mol)
    # each term alone (kcal/mol): bonds without H, angles, torsions, nonbonded incl. 1-4
    s0 = a.system
    parts = {}
    for name in ('bonds', 'angles', 'torsions'):
        s = copy.deepcopy(s0)
        for other in ('bonds', 'angles', 'torsions'):
            if other != name: setattr(s, other, np.zeros((0, getattr(s, other).shape[1])))
        s.charge = np.zeros(22); s.epsilon = np.zeros(22); s.exceptions = np.zeros((0, 5))
        parts[name] = oracle.Molecule(s).energy(x) / 4.184
    assert 0.0 <= parts['bonds'] < 0.1 and 0.2 < parts['angles'] < 0.6 and 1.0 < parts['torsions'] < 12.0


def test_constrained_langevin_keeps_the_constraints_and_the_temperature():
    a, x = aladip()
    m = oracle.Molecule(a.system)
    kT = KB * 300.0
    rng = np.random.default_rng(1)
    v = np.ascontiguousarray(rng.normal(size=x.shape) * np.sqrt(kT / m.mass)[:, None])
    n = 4000
    kes = []
    for block in range(8):
        m.langevin(x, v, rng.normal(size=(n // 8, 22, 3)), kT, 0.002, 5.0, n // 8, 'VRORV', tol=1e-10)
        kes.append(m.kinetic(v))
    c = a.system.constraints
    i, j = c[:, 0].astype(int), c[:, 1].astype(int)
    assert np.abs(np.linalg.norm(x[i] - x[j], axis=1) - c[:, 2]).max() < 1e-10
    assert np.abs(((x[i] - x[j]) * (v[i] - v[j])).sum(1)).max() < 1e-9
    # 66 - 12 constraints - 3 (centre of mass) degrees of freedom
    assert abs(np.mean(kes) / (0.5 * kT * 51) - 1.0) < 0.5
    assert np.isfinite(m.energy(x))


# ---- molecules beyond alanine dipeptide (tests/helpers.py builders) ----------------------------------------------------
import helpers as H

BUILDERS = {
    'decane': lambda: H.alkane(10),
    'decane-3terms-shuffled': lambda: H.alkane(10, terms_per_torsion=3, shuffle=5),
    'methane': lambda: H.alkane(1),
    'propane-AllBonds': lambda: H.alkane(3, constraints='AllBonds'),
    'propane-AllBonds-shuffled': lambda: H.alkane(3, constraints='AllBonds', shuffle=2),
    'propane-flexible': lambda: H.alkane(3, constraints=None),
    'waters': lambda: H.waters(10),
    'waters-ion-shuffled': lambda: H.waters(10, ions=1, shuffle=3),
    'torsion-probe': lambda: H.torsion_probe(5, 0.3, -1.2),
    'mixture': lambda: H.mixture(),
    'mixture-shuffled': lambda: H.mixture(shuffle=7),
    'ion': lambda: H.ion(),
    'diatomic': lambda: H.diatomic(),
    'fragment-33': lambda: H.alkane(11, hydrogens=[2] * 11),
}


def dihedral(xi, xj, xk, xl):
    """IUPAC dihedral from the bond vectors b1 = j - i, b2 = k - j, b3 = l - k (Blondel & Karplus's atan2 form)."""
    b1, b2, b3 = xj - xi, xk - xj, xl - xk
    return np.arctan2(np.linalg.norm(b2) * np.dot(b1, np.cross(b2, b3)), np.dot(np.cross(b1, b2), np.cross(b2, b3)))


def numpy_energy(s, x):
    """The force field restated term by term (bonds, angles, periodic torsions, Coulomb + LJ with exclusions, exceptions);
    returns the energy and the sum of the magnitudes of its terms."""
    terms = []
    for i, j, K, r0 in s.bonds:
        terms.append(0.5 * K * (np.linalg.norm(x[int(i)] - x[int(j)]) - r0) ** 2)
    for i, j, k, K, t0 in s.angles:
        u, v = x[int(i)] - x[int(j)], x[int(k)] - x[int(j)]
        t = np.arccos(np.clip(np.dot(u, v) / np.linalg.norm(u) / np.linalg.norm(v), -1.0, 1.0))
        terms.append(0.5 * K * (t - t0) ** 2)
    for i, j, k, l, n, phase, kk in s.torsions:
        phi = dihedral(*(x[int(q)] for q in (i, j, k, l)))
        terms.append(kk * (1.0 + np.cos(n * phi - phase)))
    n = s.n_particles
    skip = {frozenset((int(i), int(j))) for i, j in s.exclusions} | {frozenset((int(e[0]), int(e[1]))) for e in s.exceptions}
    for i in range(n):
        for j in range(i + 1, n):
            if frozenset((i, j)) in skip:
                continue
            r = np.linalg.norm(x[i] - x[j])
            sg, ep = 0.5 * (s.sigma[i] + s.sigma[j]), np.sqrt(s.epsilon[i] * s.epsilon[j])
            terms.append(138.935456 * s.charge[i] * s.charge[j] / r + 4 * ep * ((sg / r) ** 12 - (sg / r) ** 6))
    for i, j, qq, sg, ep in s.exceptions:
        r = np.linalg.norm(x[int(i)] - x[int(j)])
        terms.append(138.935456 * qq / r + 4 * ep * ((sg / r) ** 12 - (sg / r) ** 6))
    return float(np.sum(terms)), float(np.sum(np.abs(terms)))


@pytest.mark.parametrize('name', sorted(BUILDERS))
def test_builders_hold_their_constraints_and_their_documented_shapes(name):
    s, x = BUILDERS[name]()
    c = s.constraints
    if len(c):
        i, j = c[:, 0].astype(int), c[:, 1].astype(int)
        assert np.abs(np.linalg.norm(x[i] - x[j], axis=1) - c[:, 2]).max() < 1e-12
    shapes = sorted(len(q) for q in H.constraint_clusters(c, s.n_particles))
    expect = {'decane': [2] * 8 + [3] * 2, 'methane': [4], 'propane-AllBonds': [10], 'waters': [3] * 10, 'mixture': [1, 2, 3, 4],
              'diatomic': [1], 'ion': [], 'torsion-probe': []}
    for k, v in expect.items():
        if name.startswith(k):
            assert shapes == v, shapes
    n_atoms = {'decane': 32, 'waters-ion': 31, 'waters': 30, 'ion': 1, 'diatomic': 2, 'fragment-33': 33, 'mixture': 14,
               'methane': 5, 'propane': 11, 'torsion-probe': 5}
    assert s.n_particles == next(v for k, v in n_atoms.items() if name.startswith(k))
    if 'shuffled' in name:
        heavy = s.masses > 1.1
        assert not np.any(heavy[:np.argmax(heavy)]) and np.all(heavy[np.argmax(heavy):])     # hydrogens first
        assert np.all(c[:, 0] > c[:, 1])
        root = {}
        for q in H.constraint_clusters(c, s.n_particles):
            for row in q:
                root[tuple(row)] = id(q)
        owner = [root[tuple(r)] for r in c]
        assert all(a != b for a, b in zip(owner[:len(set(owner))], owner[1:len(set(owner))]))   # clusters alternate
    if name.startswith('decane-3terms'):
        per = s.torsions[:, 4]
        assert set(per) == {1.0, 2.0, 3.0} and np.any(s.torsions[:, 6] < 0) and np.any(np.abs(s.torsions[:, 5] - 0.3) < 1e-15)
    if s.n_particles > 1:
        assert s.masses.max() / s.masses.min() > 11.9


@pytest.mark.parametrize('name', sorted(BUILDERS))
def test_numpy_restatement_of_the_force_field_agrees_with_the_oracle(name):
    s, x = BUILDERS[name]()
    m = oracle.Molecule(s)
    for q in range(3):
        xq = x + np.random.default_rng(q).normal(0, 0.003, x.shape) if q else x
        U, scale = numpy_energy(s, xq)
        assert abs(m.energy(xq) - U) <= 1e-12 * max(1.0, scale), (m.energy(xq), U)


@pytest.mark.parametrize('n', [1, 2, 3, 4, 5, 6])
@pytest.mark.parametrize('k', [1.3, -0.7])
def test_the_sign_of_the_dihedral_is_pinned_by_construction(n, k):
    """j = 0, k = 0.15 z, i = 0.1 x, l = (0.1 cos phi, 0.1 sin phi, 0.15): the IUPAC dihedral is +phi.  With the asymmetric
    phase 0.3, k (1 + cos(n phi - 0.3)) differs between +phi and -phi for every n, so a flipped sign shows."""
    for deg in (70.0, -70.0):
        phi = np.deg2rad(deg)
        s, x = H.torsion_probe(n, 0.3, k, phi=phi)
        assert abs(dihedral(x[0], x[1], x[2], x[3]) - phi) < 1e-13
        s.bonds = np.zeros((0, 4)); s.angles = np.zeros((0, 5)); s.exceptions = np.zeros((0, 5))
        s.charge = np.zeros(5); s.epsilon = np.zeros(5)
        proper = s.torsions[(s.torsions[:, :4] == [0, 1, 2, 3]).all(1)]
        assert len(proper) == 1
        s.torsions = proper
        U = oracle.Molecule(s).energy(x)
        assert abs(U - k * (1.0 + np.cos(n * phi - 0.3))) < 1e-13
        assert abs(U - k * (1.0 + np.cos(-n * phi - 0.3))) > 1e-3 * abs(k)


@pytest.mark.parametrize('name', sorted(BUILDERS))
def test_oracle_forces_are_the_gradient_on_every_builder(name):
    s, x = BUILDERS[name]()
    x = x + np.random.default_rng(4).normal(0, 0.002, x.shape)
    m = oracle.Molecule(s)
    U, f = m.energy(x, forces=True)
    g = np.zeros_like(x); h = 1e-6
    for i in range(len(x)):
        for c in range(3):
            xp = x.copy(); xp[i, c] += h; xm = x.copy(); xm[i, c] -= h
            g[i, c] = -(m.energy(xp) - m.energy(xm)) / (2 * h)
    assert np.abs(g - f).max() <= 1e-5 * max(1.0, np.abs(f).max())
    assert np.abs(f.sum(0)).max() < 1e-8 * max(1.0, np.abs(f).max())


@pytest.mark.parametrize('name', [b for b in sorted(BUILDERS) if b not in ('ion', 'torsion-probe', 'propane-flexible')])
def test_oracle_shake_and_rattle_hold_every_cluster_shape(name):
    s, x = BUILDERS[name]()
    m = oracle.Molecule(s)
    kT = KB * 300.0
    rng = np.random.default_rng(6)
    v = np.ascontiguousarray(rng.normal(size=x.shape) * np.sqrt(kT / m.mass)[:, None])
    x = x.copy()
    m.langevin(x, v, rng.normal(size=(100, len(x), 3)), kT, 0.002, 5.0, 100, 'VRORV', tol=1e-10)
    c = s.constraints
    i, j = c[:, 0].astype(int), c[:, 1].astype(int)
    assert np.abs(np.linalg.norm(x[i] - x[j], axis=1) - c[:, 2]).max() < 1e-10
    assert np.abs(((x[i] - x[j]) * (v[i] - v[j])).sum(1)).max() < 1e-10
    assert np.isfinite(m.energy(x))
