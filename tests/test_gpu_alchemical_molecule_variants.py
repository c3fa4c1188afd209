"""Alchemical molecules beyond toluene and alanine dipeptide on the GPU (the ALCH instantiations of k_energy_mol,
k_propagate_mol, k_propagate_mol_hmc, k_mc_move_mol and k_minimize_mol) against the float64 oracle
(oracle/alchemical_molecule.py): energy rows over a ladder built to stress k_energy_mol's row cache, Langevin steps on the
device's noise (tests/mol_langevin_oracle.py), HMC trials, Monte Carlo moves, FIRE, forces at the lambda end points and at a
soft-core overlap, engulfed OBC2 pairs, and the shared-memory limit -- on the cases of tests/alchemical_cases.py, every state
table differing in lambda_sterics and lambda_electrostatics, and the replicas on a permutation of the states.  The tests
record the largest deviations they see with record_property (pytest --junitxml=... -o junit_family=legacy writes them)."""
import numpy as np
import pytest
import alchemical_cases as A
import hmc_oracle as ho
import mc_oracle as mo
import mol_langevin_oracle as mlo
from helpers import KB, device_noise, gpu_engine
from test_gpu_hmc import check_replica, SEED, IT
from test_gpu_hmc_variants import assert_exercised, molecule_start
from test_gpu_mc_moves import run_moves, replay, check
from test_gpu_molecule import projected_rms, constraint_error
from openmmtools_b200 import _lib

pytestmark = pytest.mark.gpu

PERM3 = np.array([2, 0, 1])
# three states that differ in both lambdas and in temperature
STATES3 = [(1.0, 0.7, 300.0), (0.6, 0.2, 350.0), (0.3, 0.0, 400.0)]


def _ids(cases):
    return ['%s%s' % (n, '-swapped' if s else '') for n, s in cases]


def engine(asys, states, K, constraint_tolerance=1e-10, offsets=None):
    """A molecule engine with the alchemical system's soft-core parameters and the states (lambda_s, lambda_e, T)."""
    e = gpu_engine(_lib.RX_SYSTEM_MOLECULE, K, len(states), asys.n_particles, softcore_alpha=asys.softcore_alpha,
                   softcore_a=asys.softcore_a, softcore_b=asys.softcore_b, softcore_c=asys.softcore_c)
    e.set_molecule(asys, constraint_tolerance=constraint_tolerance)
    ls, le, T = (np.array([s[q] for s in states], float) for q in range(3))
    e.set_states(T, lambda_sterics=ls, lambda_electrostatics=le, energy_offset=offsets)
    return e


def oracle(asys):
    from oracle.alchemical_molecule import AlchemicalMolecule
    return AlchemicalMolecule(asys)


def forces_at(m, state):
    ls, le = state[0], state[1]
    return lambda x: m.energy(np.ascontiguousarray(x), ls, le, forces=True)


def unconstrained(asys):
    a = asys.copy()
    a.constraints = np.zeros((0, 3))
    a.remove_cm_motion = False
    return a


# -- energy rows --------------------------------------------------------------------------------------------------------
def cache_ladder():
    """48 states for k_energy_mol's row cache (the OBC energy kept while lambda_e repeats, the alchemical pairs while (la, ob,
    lambda_e) repeat): runs of equal lambda_e with changing lambda_s and the reverse, A-B-A returns, temperature-only
    changes, duplicates, and lambdas of exactly 0 and 1."""
    L = [(1.0, 1.0, 300.0), (0.8, 1.0, 300.0), (0.5, 1.0, 300.0), (0.0, 1.0, 300.0),        # lambda_e fixed
         (0.0, 0.6, 300.0), (0.0, 0.3, 300.0), (0.0, 0.0, 300.0),                           # lambda_s fixed
         (0.5, 0.5, 300.0), (0.2, 0.9, 300.0), (0.5, 0.5, 300.0),                           # A-B-A
         (0.5, 0.5, 320.0), (0.5, 0.5, 350.0), (0.5, 0.5, 350.0),                           # temperature only, duplicate
         (1.0, 0.0, 300.0), (0.0, 1.0, 330.0), (1.0, 1.0, 310.0), (0.0, 0.0, 300.0),       # end points
         (0.7, 0.5, 300.0), (0.7, 0.25, 300.0), (0.7, 0.5, 300.0), (0.3, 0.5, 300.0),       # lambda_e returns, lambda_s moves
         (0.3, 0.5, 300.0), (0.3, 0.5, 300.0)]
    rng = np.random.default_rng(12)
    grid = [0.0, 0.25, 0.5, 0.75, 1.0]
    while len(L) < 48:
        ls, le = rng.choice(grid), rng.choice(grid)
        for _ in range(int(rng.integers(1, 4))):     # runs of a repeated pair at other temperatures
            L.append((float(ls), float(le), float(rng.choice([300.0, 340.0, 400.0]))))
    return L[:48]


def oracle_rows(m, xs, states, offsets=None):
    memo = {}
    off = np.zeros(len(states)) if offsets is None else offsets
    u = np.zeros((len(xs), len(states)))
    for k, x in enumerate(xs):
        for l, (ls, le, T) in enumerate(states):
            if (k, ls, le) not in memo:
                memo[k, ls, le] = m.energy(x, ls, le)
            u[k, l] = (memo[k, ls, le] + off[l]) / (KB * T)
    return u


@pytest.mark.parametrize('name,swapped', A.variants(), ids=_ids(A.variants()))
def test_energy_rows_over_a_cache_ladder_match_the_oracle(record_property, name, swapped):
    _, x, asys = A.make(name, swapped)
    m = oracle(asys)
    ladder = cache_ladder()
    rng = np.random.default_rng(3)
    K = 3
    xs = np.stack([x + rng.normal(0, 0.004, x.shape) for _ in range(K)])
    e = engine(asys, ladder, K)
    try:
        e.set_replica_states(PERM3)
        e.set_positions(xs)
        u = e.compute_energies()
        ref = oracle_rows(m, xs, ladder)
        record_property('rel_dev_rows', float(np.abs(u - ref).max() / np.abs(ref).max()))
        np.testing.assert_allclose(u, ref, rtol=1e-10, atol=0)
        # 100 unsampled states (more than a warp's lanes), with offsets; the resident matrix untouched
        more = [(float(a), float(b), float(c)) for a, b, c in zip(rng.choice([0.0, 0.1, 0.5, 0.9, 1.0], 100),
                                                                  rng.choice([0.0, 0.4, 1.0], 100), rng.uniform(280.0, 500.0, 100))]
        off = rng.normal(0, 30.0, 100)
        ls, le, T = (np.array([s[q] for s in more]) for q in range(3))
        ua = e.compute_energies_at(T, lambda_sterics=ls, lambda_electrostatics=le, energy_offset=off)
        ref = oracle_rows(m, xs, more, off)
        record_property('rel_dev_at', float(np.abs(ua - ref).max() / np.abs(ref).max()))
        np.testing.assert_allclose(ua, ref, rtol=1e-10, atol=0)
        assert e.get_energies().tobytes() == u.tobytes()
    finally:
        e.close()


# -- Langevin steps on the device's noise --------------------------------------------------------------------------------
def star_path(asys):
    """Whether k_propagate_mol takes the MolStar path: every constraint cluster has at most three constraints."""
    c = np.asarray(asys.constraints if asys.constraints is not None else np.zeros((0, 3)))
    if not len(c):
        return True
    comp = list(range(asys.n_particles))

    def find(a):
        while comp[a] != a:
            a = comp[a]
        return a
    for i, j, _ in c:
        comp[find(int(i))] = find(int(j))
    sizes = np.bincount([find(int(i)) for i, _, _ in c])
    return sizes.max() <= 3


LANGEVIN = [(n, s, sp, False) for n, s in A.variants() for sp in ('V R O R V', 'O V R V O', 'V R R O R R V')] + \
           [(n, s, 'V R O R V', True) for n, s in A.variants() if star_path(A.make(n, s)[2])]


@pytest.mark.parametrize('name,swapped,splitting,no_star', LANGEVIN,
                         ids=['%s%s-%s%s' % (n, '-swapped' if s else '', sp.replace(' ', ''), '-general' if g else '')
                              for n, s, sp, g in LANGEVIN])
def test_langevin_steps_match_the_oracle_on_the_device_noise(monkeypatch, record_property, name, swapped, splitting, no_star):
    """K = 3 replicas on PERM3 against tests/mol_langevin_oracle.py with the oracle's forces at each replica's own state,
    at the bounds of test_gpu_molecule's constrained steps; the reported potential is the replica's energy-row entry."""
    if no_star:
        monkeypatch.setenv('RX_MOL_NO_STAR', '1')
    _, x, asys = A.make(name, swapped)
    m = oracle(asys)
    n, K = asys.n_particles, 3
    rng = np.random.default_rng(8)
    mass = np.asarray(asys.masses, float)
    v0 = np.stack([rng.normal(size=x.shape) * np.sqrt(KB * STATES3[PERM3[k]][2] / mass)[:, None] for k in range(K)])
    n_steps, dt, gamma, seed, it = 10, 0.001, 5.0, 4242, 17
    e = engine(asys, STATES3, K)
    try:
        e.set_integrator(dt, gamma, n_steps, splitting)
        e.set_positions(np.stack([x] * K)); e.set_velocities(v0)
        e.set_replica_states(PERM3)
        e.propagate(seed, it)
        xg, vg = e.get_positions(), e.get_velocities()
        pg, kg = e.get_replica_energies()
        u = e.compute_energies()
    finally:
        e.close()
    nO = splitting.replace(' ', '').count('O')
    cons = asys.constraints if asys.constraints is not None and len(asys.constraints) else None
    dev = np.zeros(4)
    for k in range(K):
        st = STATES3[PERM3[k]]
        xo, vo, U = mlo.run(x, v0[k], mass, KB * st[2], forces_at(m, st), device_noise(seed, it, k, n, n_steps * nO), dt, gamma,
                            n_steps, splitting, cons=cons, remove_cm=bool(asys.remove_cm_motion))
        dev = np.maximum(dev, [np.abs(xg[k] - xo).max(), np.abs(vg[k] - vo).max(), abs(pg[k] - U),
                               abs(u[k, PERM3[k]] * KB * st[2] - pg[k]) / max(abs(pg[k]), 1.0)])
        record_property('dev_x_v_pot_row', dev.tolist())
        assert np.abs(xg[k] - xo).max() < 3e-7, (k, np.abs(xg[k] - xo).max())
        assert np.abs(vg[k] - vo).max() < 1e-4, (k, np.abs(vg[k] - vo).max())
        assert abs(pg[k] - U) < 2e-3 and abs(kg[k] - 0.5 * np.sum(mass[:, None] * vo * vo)) < 2e-3, (k, pg[k] - U)
        if cons is not None:
            assert constraint_error(asys, xg[k]) < 1e-9
        assert abs(u[k, PERM3[k]] * KB * st[2] - pg[k]) <= 1e-14 * max(abs(pg[k]), 1.0), (k, u[k, PERM3[k]] * KB * st[2], pg[k])


# -- HMC ------------------------------------------------------------------------------------------------------------------
# (n_steps, dt ps) per case at the states of STATES2, chosen on the host with hmc_oracle and the device's draws for an
# acceptance of 0.3-0.8 over the 2 x 2 x n_steps trials of a test (0.46, 0.57, 0.69, 0.38, 0.63 and 0.47).  (The rigid
# waters, chaotic at the steps that bring their acceptance into the band -- test_gpu_hmc_variants.CHAOTIC --, are left to
# the Monte Carlo test.)
STATES2 = [(0.8, 0.4, 300.0), (0.3, 0.0, 450.0)]
HMC_CASES = {
    'decane-obc2-top': (7, 0.004), 'decane-all-annihilated': (7, 0.004), 'propane-allbonds-obc1-half': (8, 0.0035),
    'mixture-obc2-half': (8, 0.005), 'torsion-probe-sc-c4': (8, 0.0035), 'engulfed-methane-obc2': (8, 0.006),
}
HMC = [(n, False) for n in HMC_CASES] + [(n, True) for n in HMC_CASES if star_path(A.make(n)[2])]


@pytest.mark.parametrize('name,no_star', HMC, ids=['%s%s' % (n, '-general' if g else '') for n, g in HMC])
def test_hmc_trials_match_the_oracle_at_each_replica_state(monkeypatch, name, no_star):
    if no_star:
        monkeypatch.setenv('RX_MOL_NO_STAR', '1')
    _, x, asys = A.make(name)
    m = oracle(asys)
    from oracle import oracle as om
    mm = om.Molecule(asys)     # (masses and constraints)
    n_steps, dt = HMC_CASES[name]
    K, perm = 2, np.array([1, 0])
    e = engine(asys, STATES2, K)
    try:
        e.set_hmc_integrator(dt, n_steps)
        x0 = molecule_start(asys, x, mm, K)
        e.set_positions(x0); e.set_velocities(np.zeros_like(x0))
        e.set_replica_states(perm)
        its = (IT, IT + 1)
        for it in its:
            e.propagate(SEED, it)
        xg, vg = e.get_positions(), e.get_velocities()
        cons = mm.cons if len(mm.cons) else None
        per = [check_replica(e, k, x0[k], mm.mass, KB * STATES2[perm[k]][2], forces_at(m, STATES2[perm[k]]), dt, n_steps, xg, vg,
                             tol_x=2e-5, tol_v=1e-2, cons=cons, iterations=its) for k in range(K)]
    finally:
        e.close()
    assert_exercised(per, n_steps)
    if cons is not None:
        assert constraint_error(asys, xg) < 1e-10


# -- Monte Carlo moves ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', ['waters-ion-obc2-ion', 'waters-ion-obc2-water'])
def test_mc_moves_of_the_ligand_among_waters_match_the_oracle(record_property, name):
    """Displacements and rotations of the alchemical ion, then of the alchemical water, at four lambda states: decisions and
    statistics exact, positions to 2e-6 nm, both an acceptance and a rejection."""
    _, x, asys = A.make(name)
    m = oracle(asys)
    sub = np.array(asys.alchemical_atoms)
    states = [(1.0, 1.0, 300.0), (1.0, 0.5, 320.0), (0.6, 0.0, 300.0), (0.2, 0.0, 350.0)]
    K = 8
    rng = np.random.default_rng(4)
    xs = np.stack([x + rng.normal(0, 0.01, x.shape) for _ in range(K)])
    moves = [[(mo.DISPLACEMENT, 0.04, sub), (mo.ROTATION, 0.0, sub), (mo.DISPLACEMENT, 0.15, sub)]] * len(states)
    e = engine(asys, states, K)
    perm = np.arange(K)[::-1] % len(states)
    try:
        e.set_replica_states(perm)
        xd, stats = run_moves(e, xs, moves)
    finally:
        e.close()
    betas = 1.0 / (KB * np.array([s[2] for s in states]))
    xo, dec = replay(xs, moves, perm, lambda l, k, y: m.energy(y, states[l][0], states[l][1]), betas, store=np.float64)
    record_property('dev_x', float(np.abs(xd - xo).max()))
    check(xd, xo, dec, stats, moves, perm)
    d = [y for row in dec for y in row]
    assert 0 < sum(d) < len(d), dec


# -- FIRE -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', ['propane-allbonds-obc1-half', 'decane-obc2-top'])
def test_minimizer_reports_the_projected_rms_at_each_replica_state(record_property, name):
    """k_minimize_mol with the replicas on the reversed permutation: the RMS force each replica reports is the tangent
    projection's RMS of the oracle's force at ITS state, and its energy there went down."""
    _, x, asys = A.make(name)
    m = oracle(asys)
    K = 3
    perm = np.array([2, 1, 0])
    rng = np.random.default_rng(6)
    x0 = np.stack([x + rng.normal(0, 0.003, x.shape) for _ in range(K)])
    if asys.constraints is not None and len(asys.constraints):
        x0 = np.stack([ho.shake(asys.constraints, asys.masses, xk, xk, 1e-12) for xk in x0])
    e = engine(asys, STATES3, K)
    try:
        e.set_replica_states(perm)
        e.set_positions(x0)
        rms, its = e.minimize(1.0, 3000)
        xm = e.get_positions()
    finally:
        e.close()
    for k in range(K):
        ls, le, _ = STATES3[perm[k]]
        U, F = m.energy(xm[k], ls, le, forces=True)
        ref = projected_rms(asys, xm[k], F)
        record_property('rel_dev_rms_%d' % k, float(abs(rms[k] / ref - 1)))
        assert abs(rms[k] - ref) <= 1e-6 * ref, (k, rms[k], ref)
        assert U < m.energy(x0[k], ls, le) - 1.0 and its[k] > 0


# -- forces at the lambda end points and at a soft-core overlap --------------------------------------------------------------
def v_step(asys, x, states, perm):
    """One V step of dt = 1e-4 from rest of unconstrained copies: dt F / m."""
    a = unconstrained(asys)
    K = len(perm)
    e = engine(a, states, K)
    try:
        e.set_replica_states(perm)
        e.set_positions(np.stack([x] * K) if x.ndim == 2 else x)
        e.set_velocities(np.zeros((K,) + x.shape[-2:]))
        e.set_integrator(1e-4, 0.0, 1, 'V O R')   # (O: a no-op without friction)
        e.propagate(1, 0)
        return e.get_velocities()
    finally:
        e.close()


def check_v_step(asys, x, states, perm, bound=1e-4):
    m = oracle(asys)
    v = v_step(asys, x, states, perm)
    worst = 0.0
    for k in range(len(perm)):
        ls, le, _ = states[perm[k]]
        _, F = m.energy(x if x.ndim == 2 else x[k], ls, le, forces=True)
        ref = 1e-4 * F / np.asarray(asys.masses)[:, None]
        scale = max(np.abs(ref).max(), 1e-300)
        worst = max(worst, np.abs(v[k] - ref).max() / scale)
        assert np.abs(v[k] - ref).max() <= bound * scale, (k, np.abs(v[k] - ref).max() / scale)
    return worst


ENDS = [(0.0, 0.0, 300.0), (0.0, 1.0, 300.0), (1.0, 0.0, 300.0), (1.0, 1.0, 300.0)]
END_CASES = [(n, s) for n, s in A.variants() if n in ('decane-obc2-top', 'decane-all-annihilated', 'propane-allbonds-obc1-half',
                                                      'mixture-obc2-half', 'torsion-probe-sc-c4', 'torsion-probe-sc-c12',
                                                      'waters-ion-obc2-water')]


@pytest.mark.parametrize('name,swapped', END_CASES, ids=_ids(END_CASES))
def test_forces_at_the_lambda_end_points_match_the_oracle(record_property, name, swapped):
    _, x, asys = A.make(name, swapped)
    x = x + np.random.default_rng(5).normal(0, 0.003, x.shape)
    record_property('dev_force', check_v_step(asys, x, ENDS, np.array([3, 0, 2, 1])))


@pytest.mark.parametrize('swapped', [False, True])
def test_forces_at_a_soft_core_overlap_match_the_oracle(record_property, swapped):
    """The alchemical ion 0.03 nm from a water oxygen, and (fully alchemical decane, both lambdas annihilated) two hydrogens of
    different carbons 0.03 nm apart, at lambda_s = 0 and 0.1 with lambda_e = 0: the soft-core sterics stay finite and the
    forces match."""
    states = [(0.0, 0.0, 300.0), (0.1, 0.0, 300.0)]
    _, x, asys = A.make('waters-ion-obc2-ion', swapped)
    ion = asys.alchemical_atoms[0]
    o = int(np.argmax(np.asarray(asys.masses) == 15.9994))
    x = x.copy()
    x[ion] = x[o] + np.array([0.03, 0.0, 0.0])
    record_property('dev_force_ion', check_v_step(asys, x, states, np.array([1, 0])))
    _, x, asys = A.make('decane-all-annihilated', swapped)
    m = oracle(asys)
    far = [p for p in m.pairs if asys.masses[p[0]] < 2 and asys.masses[p[1]] < 2 and np.linalg.norm(x[p[0]] - x[p[1]]) > 0.4]
    i, j = far[0][0], far[0][1]
    x = x.copy()
    x[j] = x[i] + np.array([0.0, 0.03, 0.0])
    record_property('dev_force_decane', check_v_step(asys, x, states, np.array([1, 0])))


# -- engulfed OBC2 pairs ----------------------------------------------------------------------------------------------------
def test_engulfed_pairs_energies_and_forces_match_the_oracle(record_property):
    """Methane with four engulfed (H, C) pairs (alchemical_cases.engulfed_methane), at lambda_e 0, 0.5 and 1: energy rows to
    1e-10 and one-step forces to 1e-4 of the largest."""
    from oracle import implicit
    s, x, asys = A.make('engulfed-methane-obc2')
    m = oracle(asys)
    rng = np.random.default_rng(13)
    K = 3
    xs = np.stack([x + rng.normal(0, 0.003, x.shape) for _ in range(K)])
    for xk in xs:
        assert implicit.Molecule(s).born_radii(xk)[1] == 4
    states = [(0.7, 0.0, 300.0), (0.7, 0.5, 330.0), (1.0, 1.0, 300.0)]
    e = engine(asys, states, K)
    try:
        e.set_replica_states(PERM3)
        e.set_positions(xs)
        u, ref = e.compute_energies(), oracle_rows(m, xs, states)
        record_property('rel_dev_rows', float(np.abs(u - ref).max() / np.abs(ref).max()))
        np.testing.assert_allclose(u, ref, rtol=1e-10, atol=0)
    finally:
        e.close()
    record_property('dev_force', check_v_step(asys, xs, states, PERM3))


# -- shared memory --------------------------------------------------------------------------------------------------------
def test_fully_alchemical_decane_in_obc2_runs_and_matches_the_oracle(record_property):
    """The largest tables a molecule can have: 32 atoms, every pair in the alchemical table, OBC2.  They fit in an H100
    block's opt-in shared memory, so set_molecule accepts them and every kernel runs them (a refusal would have to come
    from set_molecule / set_implicit_solvent as EngineError, never from a launch)."""
    from openmmtools_b200.alchemy import AbsoluteAlchemicalFactory, AlchemicalRegion
    from implicit_helpers import obc
    from test_gpu_molecule import MOLECULES
    s, x = MOLECULES['decane']()
    asys = AbsoluteAlchemicalFactory().create_alchemical_system(
        obc(s, 'OBC2'), AlchemicalRegion(alchemical_atoms=range(32), annihilate_sterics=True, annihilate_electrostatics=True))
    m = oracle(asys)
    K = 3
    rng = np.random.default_rng(3)
    xs = np.stack([x + rng.normal(0, 0.003, x.shape) for _ in range(K)])
    e = engine(asys, STATES3, K)
    try:
        e.set_replica_states(PERM3)
        e.set_positions(xs)
        u, ref = e.compute_energies(), oracle_rows(m, xs, STATES3)
        record_property('rel_dev_rows', float(np.abs(u - ref).max() / np.abs(ref).max()))
        np.testing.assert_allclose(u, ref, rtol=1e-10, atol=0)
        e.set_integrator(0.001, 5.0, 5, 'V R O R V')
        e.set_velocities(np.zeros_like(xs))
        e.propagate(3, 1)
        e.minimize(1.0, 50)
        e.set_hmc_integrator(0.002, 2)
        e.propagate(3, 2)
        e.set_mc_moves([[(mo.DISPLACEMENT, 0.01, list(range(32)))]] * 3)
        e.propagate(3, 3)
        assert np.all(np.isfinite(e.compute_energies()))
    finally:
        e.close()
    record_property('dev_force', check_v_step(asys, xs, STATES3, PERM3))
