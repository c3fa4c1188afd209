"""RX_SYSTEM_MOLECULE on the GPU against the oracle (oracle/rx_oracle_mol.c): energies, constrained Langevin steps with the
same noise, constraint satisfaction over a long launch, and config 4 of BASELINE.json -- ParallelTemperingSampler on
testsystems.AlanineDipeptideVacuum (paralleltempering.py:109-237, testsystems.py:3352-3388) -- at reduced size."""
import numpy as np
import pytest
import helpers as H
from helpers import gpu_engine, KB, device_noise, device_reassign_noise, device_randomize_noise
from openmmtools_b200 import testsystems, unit, _lib

pytestmark = pytest.mark.gpu


def aladip(constraints='HBonds'):
    a = testsystems.AlanineDipeptideVacuum(constraints=constraints)
    return a, np.ascontiguousarray(a.positions.value_in_unit(unit.nanometer), np.float64)


def _aladip_system(constraints):
    a, x = aladip(constraints)
    return a.system, x


# (system, positions) of every molecule the tests run; tests/helpers.py builds all but alanine dipeptide.  "shuffled":
# hydrogens numbered first, constraint endpoints i > j, the constraints of different clusters alternating in the list.
MOLECULES = {
    'alanine-dipeptide': lambda: _aladip_system('HBonds'),
    'alanine-dipeptide-flexible': lambda: _aladip_system(None),
    'decane': lambda: H.alkane(10),                                                      # 32 atoms, > 48 KB of tables
    'decane-3terms-shuffled': lambda: H.alkane(10, terms_per_torsion=3, shuffle=5),
    'methane': lambda: H.alkane(1),                                                      # one cluster of 4: Newton M-SHAKE
    'propane-AllBonds': lambda: H.alkane(3, constraints='AllBonds'),                     # one cluster of 10: sweeps
    'propane-AllBonds-shuffled': lambda: H.alkane(3, constraints='AllBonds', shuffle=2),
    'waters': lambda: H.waters(10),                                                      # ten 3-constraint cycles
    'waters-ion-shuffled': lambda: H.waters(10, ions=1, shuffle=3),                      # n = 31
    'torsion-probe': lambda: H.torsion_probe(5, 0.3, -1.2),                              # n = 5, phase 0.3, k < 0, improper
    'mixture': lambda: H.mixture(),                                                      # clusters of 1, 2, 3 and 4
    'mixture-shuffled': lambda: H.mixture(shuffle=7),
    'ion': lambda: H.ion(),                                                              # n = 1
    'diatomic': lambda: H.diatomic(),                                                    # n = 2
}


def constraint_error(s, x):
    c = s.constraints
    if c is None or not len(c):
        return 0.0
    i, j = c[:, 0].astype(int), c[:, 1].astype(int)
    return np.abs(np.linalg.norm(x[..., i, :] - x[..., j, :], axis=-1) - c[:, 2]).max()


def make_engine(system, temps, constraint_tolerance=1e-10):
    K = len(temps)
    e = gpu_engine(_lib.RX_SYSTEM_MOLECULE, K, K, system.n_particles)
    e.set_molecule(system, constraint_tolerance=constraint_tolerance)
    e.set_states(np.asarray(temps, float), np.ones(K))
    return e


def test_energy_rows_match_the_oracle():
    for name in ('alanine-dipeptide', 'alanine-dipeptide-flexible'):
        check_energy_rows(name)


@pytest.mark.parametrize('name', [k for k in MOLECULES if not k.startswith('alanine')])
def test_energy_rows_of_every_molecule_match_the_oracle(name):
    check_energy_rows(name)


def check_energy_rows(name):
    """k_energy_mol (f64) against the oracle; also at 100 other temperatures with offsets (more states than the warp's
    32 lanes: the l += 32 loop)."""
    from oracle import oracle
    system, x = MOLECULES[name]()
    temps = np.array([300.0, 350.0, 420.0, 600.0])
    rng = np.random.default_rng(3)
    xs = np.stack([x + rng.normal(0, 0.004, x.shape) for _ in temps])
    e = make_engine(system, temps)
    e.set_positions(xs)
    u = e.compute_energies()
    T100 = np.linspace(280.0, 900.0, 100)
    off = np.random.default_rng(4).normal(0, 50.0, 100)
    u100 = e.compute_energies_at(T100, energy_offset=off)
    e.close()
    m = oracle.Molecule(system)
    U = np.array([m.energy(xk) for xk in xs])
    ref = U[:, None] / (KB * temps)[None, :]
    assert np.abs(u - ref).max() <= 1e-10 * max(1.0, np.abs(ref).max())
    ref100 = (U[:, None] + off[None, :]) / (KB * T100)[None, :]
    assert np.abs(u100 - ref100).max() <= 1e-10 * max(1.0, np.abs(ref100).max())


@pytest.mark.parametrize('splitting,n_steps', [('V R O R V', 1), ('V R O R V', 25), ('O V R V O', 10), ('R V O', 7)])
@pytest.mark.parametrize('constraints', ['HBonds', None])
def test_constrained_steps_match_the_oracle_with_the_same_noise(splitting, n_steps, constraints):
    from oracle import oracle
    a, x = aladip(constraints)
    temps = np.array([300.0, 450.0, 600.0])
    K = len(temps)
    rng = np.random.default_rng(8)
    m = oracle.Molecule(a.system)
    v0 = np.stack([rng.normal(size=x.shape) * np.sqrt(KB * T / m.mass)[:, None] for T in temps])
    e = make_engine(a.system, temps)
    dt, gamma = 0.001, 5.0
    e.set_integrator(dt, gamma, n_steps, splitting)
    e.set_positions(np.stack([x] * K)); e.set_velocities(v0)
    e.set_replica_states(np.array([2, 0, 1]))
    seed, it = 4242, 17
    e.propagate(seed, it)
    xg, vg = e.get_positions(), e.get_velocities()
    pg, kg = e.get_replica_energies()
    e.close()
    nO = splitting.replace(' ', '').count('O')
    perm = [2, 0, 1]
    for k in range(K):
        xo, vo = x.copy(), np.ascontiguousarray(v0[k])
        # (the kernel first projects the incoming velocities onto the constraints: zero steps of the oracle do the same)
        noise = device_noise(seed, it, k, 22, n_steps * nO)
        kT = KB * temps[perm[k]]
        U = oracle_run(m, xo, vo, noise, kT, dt, gamma, n_steps, splitting)
        # (the kernel evaluates forces in f32 -- as k_propagate does -- on f64 positions; energies and constraints in f64)
        assert np.abs(xg[k] - xo).max() < 3e-7, (k, np.abs(xg[k] - xo).max())
        # (flexible bonds to hydrogen amplify rounding differences faster than the constrained system)
        assert np.abs(vg[k] - vo).max() < 1e-4, (k, np.abs(vg[k] - vo).max())
        # (energies: a 1e-9 nm difference on an unconstrained 284512 kJ/mol/nm^2 bond is 1e-5 kJ/mol)
        assert abs(pg[k] - U) < 2e-3 and abs(kg[k] - m.kinetic(vo)) < 2e-3


def oracle_run(m, x, v, noise, kT, dt, gamma, n_steps, splitting):
    """The oracle with the kernel's entry convention: incoming velocities are first made to obey the constraints."""
    import ctypes as C
    from oracle import oracle
    if len(m.cons):
        oracle.lib().orc_mol_rattle(C.byref(m.s), x.ctypes.data_as(C.c_void_p), v.ctypes.data_as(C.c_void_p), C.c_double(1e-10))
    return m.langevin(x, v, noise, kT, dt, gamma, n_steps, splitting, tol=1e-10)


@pytest.mark.parametrize('splitting', ['V R O R V', 'O V R V O', 'V R R O R R V'])
@pytest.mark.parametrize('name', ['decane', 'propane-AllBonds-shuffled', 'mixture-shuffled', 'waters', 'decane-3terms-shuffled'])
def test_constrained_steps_of_every_cluster_shape_match_the_oracle(name, splitting):
    """The new molecules through k_propagate_mol<true> (decane, waters) and <false> (AllBonds: sweeps; the mixture: clusters
    of 1-4 at once) with the device's noise, at the bounds of the alanine dipeptide case."""
    from oracle import oracle
    system, x = MOLECULES[name]()
    n = system.n_particles
    temps = np.array([300.0, 450.0, 600.0])
    K = len(temps)
    rng = np.random.default_rng(8)
    m = oracle.Molecule(system)
    v0 = np.stack([rng.normal(size=x.shape) * np.sqrt(KB * T / m.mass)[:, None] for T in temps])
    n_steps, dt, gamma = 10, 0.001, 5.0
    e = make_engine(system, temps)
    e.set_integrator(dt, gamma, n_steps, splitting)
    e.set_positions(np.stack([x] * K)); e.set_velocities(v0)
    e.set_replica_states(np.array([2, 0, 1]))
    seed, it = 4242, 17
    e.propagate(seed, it)
    xg, vg = e.get_positions(), e.get_velocities()
    pg, kg = e.get_replica_energies()
    e.close()
    nO = splitting.replace(' ', '').count('O')
    perm = [2, 0, 1]
    for k in range(K):
        xo, vo = x.copy(), np.ascontiguousarray(v0[k])
        U = oracle_run(m, xo, vo, device_noise(seed, it, k, n, n_steps * nO), KB * temps[perm[k]], dt, gamma, n_steps, splitting)
        assert np.abs(xg[k] - xo).max() < 3e-7, (k, np.abs(xg[k] - xo).max())
        assert np.abs(vg[k] - vo).max() < 1e-4, (k, np.abs(vg[k] - vo).max())
        assert abs(pg[k] - U) < 2e-3 and abs(kg[k] - m.kinetic(vo)) < 2e-3
        assert constraint_error(system, xg[k]) < 1e-9


def test_long_launch_keeps_constraints_and_is_reproducible():
    check_long_launch('alanine-dipeptide')


@pytest.mark.parametrize('name', ['methane', 'propane-AllBonds-shuffled', 'waters', 'mixture-shuffled', 'decane-3terms-shuffled',
                                  'diatomic', 'ion'])
def test_long_launch_keeps_every_cluster_shape_and_is_reproducible(name):
    check_long_launch(name)


def check_long_launch(name):
    system, x = MOLECULES[name]()
    temps = np.linspace(300.0, 600.0, 8)
    K = len(temps)
    out = []
    for rep in range(2):
        e = make_engine(system, temps)
        e.set_integrator(0.002, 5.0, 500, 'V R O R V')
        e.set_positions(np.stack([x] * K)); e.randomize_velocities(11)
        e.propagate(5, 1); e.propagate(5, 2)
        out.append((e.get_positions(), e.get_velocities(), e.get_replica_energies()))
        e.close()
    (xa, va, (pa, ka)), (xb, vb, (pb, kb)) = out
    assert np.array_equal(xa, xb) and np.array_equal(va, vb) and np.array_equal(pa, pb)     # bit-reproducible
    assert constraint_error(system, xa) < 1e-9
    assert np.all(np.isfinite(pa)) and np.all(ka > 0)
    # the replica energies the launch reports are the energy kernel's (u = beta U: equal up to the rounding of beta)
    e = make_engine(system, temps)
    e.set_positions(xa)
    u = e.compute_energies()
    e.close()
    assert np.abs(u[np.arange(K), np.arange(K)] * KB * temps - pa).max() <= 1e-14 * np.abs(pa).max()
    if system.n_particles >= 14:
        # hotter replicas have more kinetic energy on average (alanine dipeptide: 51 degrees of freedom each)
        assert ka[-3:].mean() > ka[:3].mean()


def test_register_resident_cluster_path_agrees_with_the_general_one(monkeypatch):
    check_star_against_general(monkeypatch, 'alanine-dipeptide')


@pytest.mark.parametrize('name', ['decane-3terms-shuffled', 'waters'])
def test_register_resident_cluster_path_agrees_with_the_general_one_on_decane_and_waters(monkeypatch, name):
    check_star_against_general(monkeypatch, name)


def check_star_against_general(monkeypatch, name):
    """k_propagate_mol<true> (clusters of <= 3 constraints on register copies, cached RATTLE inverse, chord SHAKE) against
    k_propagate_mol<false> (Newton M-SHAKE / one solve per RATTLE, any cluster size; forced with RX_MOL_NO_STAR): the same
    constrained trajectory to the constraint tolerance.  The two solvers stop at different points inside the tolerance, and
    40 stochastic steps amplify that difference: with 1e-10 the trajectories part by ~1e-8 nm, depending on the compiler's
    rounding, so both are run at 1e-12, where what is left is the difference of the algorithms."""
    system, x = MOLECULES[name]()
    temps = np.linspace(300.0, 600.0, 6)
    K = len(temps)
    out = []
    for general in (False, True):
        if general:
            monkeypatch.setenv('RX_MOL_NO_STAR', '1')
        e = make_engine(system, temps, constraint_tolerance=1e-12)
        e.set_integrator(0.002, 5.0, 40, 'V R O R V')
        e.set_positions(np.stack([x] * K)); e.randomize_velocities(5)
        e.propagate(9, 3)
        out.append((e.get_positions(), e.get_velocities()))
        e.close()
    (xs, vs), (xg, vg) = out
    assert np.abs(xs - xg).max() < 1e-8 and np.abs(vs - vg).max() < 1e-5, (np.abs(xs - xg).max(), np.abs(vs - vg).max())
    for xx in (xs, xg):
        assert constraint_error(system, xx) < 1e-10


def test_parallel_tempering_on_alanine_dipeptide():
    """BASELINE config 4 at reduced size: 12 temperatures 300-600 K, 5 iterations of 100 steps."""
    from oracle import oracle
    from openmmtools_b200 import states, mcmc, multistate
    a, x = aladip()
    ts = states.ThermodynamicState(a.system, 300.0 * unit.kelvin)
    move = mcmc.LangevinSplittingDynamicsMove(timestep=2.0 * unit.femtosecond, collision_rate=5.0 / unit.picosecond, n_steps=100)
    s = multistate.ParallelTemperingSampler(mcmc_moves=move, number_of_iterations=5, seed=9)
    s.create(ts, [states.SamplerState(a.positions)], storage=None, min_temperature=300.0 * unit.kelvin,
             max_temperature=600.0 * unit.kelvin, n_temperatures=12)
    s.run()
    assert s.iteration == 5
    u = np.array(s._energy_thermodynamic_states)
    m = oracle.Molecule(a.system)
    T = np.array([st.temperature.value_in_unit(unit.kelvin) for st in s._thermodynamic_states])
    assert abs(T[0] - 300.0) < 1e-9 and abs(T[-1] - 600.0) < 1e-9
    for k, st in enumerate(s.sampler_states):
        xk = np.ascontiguousarray(st.positions.value_in_unit(unit.nanometer), np.float64)
        U = m.energy(xk)
        assert np.abs(u[k] - U / (KB * T)).max() < 1e-8 * max(1.0, abs(U))
    assert sorted(s._replica_thermodynamic_states.tolist()) == list(range(12))


def test_minimize_descends_on_the_constraint_manifold():
    """sampler.minimize() (multistatesampler.py:611-647) on the molecule: the energy goes down, the projected force falls
    below the tolerance, the constrained bonds keep their lengths."""
    from oracle import oracle
    from openmmtools_b200 import states, mcmc, multistate
    a, x = aladip()
    m = oracle.Molecule(a.system)
    ts = states.ThermodynamicState(a.system, 300.0 * unit.kelvin)
    s = multistate.ParallelTemperingSampler(mcmc_moves=mcmc.LangevinSplittingDynamicsMove(n_steps=10), number_of_iterations=1, seed=2)
    s.create(ts, [states.SamplerState(a.positions)], storage=None, min_temperature=300.0 * unit.kelvin,
             max_temperature=400.0 * unit.kelvin, n_temperatures=4)
    s.run()                                    # thermal configurations
    before = [m.energy(np.ascontiguousarray(st.positions.value_in_unit(unit.nanometer), np.float64)) for st in s.sampler_states]
    s.minimize(tolerance=5.0 * unit.kilojoules_per_mole / unit.nanometers, max_iterations=5000)
    c = a.system.constraints
    i, j = c[:, 0].astype(int), c[:, 1].astype(int)
    for k, st in enumerate(s.sampler_states):
        xk = np.ascontiguousarray(st.positions.value_in_unit(unit.nanometer), np.float64)
        assert m.energy(xk) < before[k] - 1.0
        assert np.abs(np.linalg.norm(xk[i] - xk[j], axis=1) - c[:, 2]).max() < 1e-8
    assert np.all(s._last_minimization['rms_force'] <= 5.0)
    assert np.all(s._last_minimization['iterations'] > 0)


def test_nan_restart_on_a_molecule_retries_only_the_failed_replica():
    """The restart policy (mcmc.py:706-759) with the molecule's f64 state: the replica that went NaN restarts from the
    device-side snapshot, the others keep their result."""
    from openmmtools_b200 import states, mcmc, multistate
    from openmmtools_b200.multistate.utils import SimulationNaNError
    a, x = aladip()
    def sampler():
        ts = states.ThermodynamicState(a.system, 300.0 * unit.kelvin)
        s = multistate.ParallelTemperingSampler(mcmc_moves=mcmc.LangevinSplittingDynamicsMove(n_steps=50), number_of_iterations=100,
                                                seed=12, replica_mixing_scheme=None)
        s.create(ts, [states.SamplerState(a.positions)], storage=None, min_temperature=300.0 * unit.kelvin,
                 max_temperature=500.0 * unit.kelvin, n_temperatures=6)
        return s
    clean, sick = sampler(), sampler()
    clean.run(3)
    sick.run(2)
    v = sick._engine.get_velocities()
    v[2] = np.nan       # (f64 state: absurd but finite velocities would not overflow)
    sick._engine.set_velocities(v[2:3], first=2)
    with pytest.raises(SimulationNaNError):
        sick.run(1)
    xs, xc = sick._engine.get_positions(), clean._engine.get_positions()
    for k in range(6):
        if k != 2:
            assert np.array_equal(xs[k], xc[k]), k


def test_rigid_waters_are_clusters_of_the_register_resident_path():
    """Ten rigid TIP3P waters in vacuum (30 atoms; three constraints over three atoms per molecule: a cycle, SETTLE's case in
    OpenMM; no centre-of-mass motion removal) through k_propagate_mol<true> and, forced, through the general path -- against
    the oracle with the same noise."""
    import os
    from oracle import oracle
    s, x = MOLECULES['waters']()
    n = s.n_particles
    temps = np.array([300.0, 420.0])
    K = len(temps)
    m = oracle.Molecule(s)
    rng = np.random.default_rng(2)
    v0 = np.stack([rng.normal(size=x.shape) * np.sqrt(KB * T / m.mass)[:, None] for T in temps])
    seed, it, n_steps, dt, gamma = 99, 3, 40, 0.002, 5.0
    ref = []
    for k in range(K):
        xo, vo = x.copy(), v0[k].copy()          # (a copy: the oracle integrates in place, and v0 goes to the device below)
        U = oracle_run(m, xo, vo, device_noise(seed, it, k, n, n_steps), KB * temps[k], dt, gamma, n_steps, 'V R O R V')
        ref.append((xo, vo, U))
    for general in (False, True):
        if general:
            os.environ['RX_MOL_NO_STAR'] = '1'
        try:
            e = gpu_engine(_lib.RX_SYSTEM_MOLECULE, K, K, n)
            e.set_molecule(s, constraint_tolerance=1e-10)
            e.set_states(temps, np.ones(K))
            e.set_integrator(dt, gamma, n_steps, 'V R O R V')
            e.set_positions(np.stack([x] * K)); e.set_velocities(v0)
            e.propagate(seed, it)
            xg, vg = e.get_positions(), e.get_velocities()
            pg, _ = e.get_replica_energies()
            e.close()
        finally:
            os.environ.pop('RX_MOL_NO_STAR', None)
        for k in range(K):
            assert constraint_error(s, xg[k]) < 1e-10
            assert np.abs(xg[k] - ref[k][0]).max() < 3e-7 and np.abs(vg[k] - ref[k][1]).max() < 1e-4, (general, k)
            assert abs(pg[k] - ref[k][2]) < 2e-3


def projected_rms(system, x, f):
    """RMS of the Euclidean tangent projection P = F - J^T (J J^T)^-1 J F of the force (J: gradients of the constraints)."""
    c = system.constraints
    n = len(x)
    if c is None or not len(c):
        return np.sqrt((f * f).sum() / (3 * n))
    J = np.zeros((len(c), 3 * n))
    for r, (i, j, _) in enumerate(c):
        d = x[int(i)] - x[int(j)]
        J[r, 3 * int(i):3 * int(i) + 3] = d
        J[r, 3 * int(j):3 * int(j) + 3] = -d
    F = f.reshape(-1)
    P = F - J.T @ np.linalg.solve(J @ J.T, J @ F)
    return np.sqrt(P @ P / (3 * n))


@pytest.mark.parametrize('name', ['mixture-shuffled', 'propane-AllBonds', 'alanine-dipeptide'])
def test_minimizer_reports_the_projected_rms_force(name):
    """k_minimize_mol from thermal configurations: the RMS force it reports is the RMS of the tangent projection of the
    oracle's force at the returned positions, both are below the tolerance, the constraints hold, the energy went down.
    (The AllBonds propane is one cluster of 10 constraints: more than the Newton solve's 4.)"""
    from oracle import oracle
    system, x = MOLECULES[name]()
    m = oracle.Molecule(system)
    temps = np.array([300.0, 400.0, 500.0])
    K = len(temps)
    e = make_engine(system, temps)
    e.set_integrator(0.001, 5.0, 200, 'V R O R V')
    e.set_positions(np.stack([x] * K)); e.randomize_velocities(3)
    e.propagate(21, 1)
    x0 = e.get_positions()
    tol = 5.0
    rms, its = e.minimize(tol, max_iterations=20000)
    xm = e.get_positions()
    e.close()
    for k in range(K):
        U, f = m.energy(xm[k], forces=True)
        ref = projected_rms(system, xm[k], f)
        assert abs(rms[k] - ref) <= 1e-12 * ref, (k, rms[k], ref)      # (8.5e-14 measured on an H100)
        assert rms[k] <= tol and ref <= tol, (k, rms[k], ref, its[k])
        assert U < m.energy(x0[k]) - 1.0
        assert constraint_error(system, xm[k]) < 1e-8


def test_randomized_and_reassigned_velocities_are_per_atom():
    """k_randomize_velocities_mol and the reassign branch of k_propagate_mol: v_i = sqrt(kT_state / m_i) xi_i with the
    device's Philox streams, atom by atom (four masses, 1.008-35.45 amu), each replica at the temperature of its state."""
    from oracle import oracle
    system, x = MOLECULES['mixture-shuffled']()
    n = system.n_particles
    temps = np.array([300.0, 350.0, 500.0, 700.0])
    perm = np.array([3, 1, 0, 2])
    K = len(temps)
    e = make_engine(system, temps)
    e.set_replica_states(perm)
    e.set_positions(np.stack([x] * K))
    e.randomize_velocities(77, stream=3)
    v = e.get_velocities()
    for k in range(K):
        sg = np.sqrt(KB * temps[perm[k]] / system.masses)[:, None]
        assert np.abs(v[k] - sg * device_randomize_noise(77, k, n, 3)).max() <= 1e-5 * sg.min()
    # reassign on the unconstrained molecule with zero steps: the outgoing velocities are the reassigned ones
    flex, xf = H.alkane(3, constraints=None)
    flex.remove_cm_motion = False
    nf = flex.n_particles
    e2 = make_engine(flex, temps)
    e2.set_replica_states(perm)
    e2.set_integrator(0.001, 5.0, 0, 'V R O R V')
    e2.set_positions(np.stack([xf] * K)); e2.set_velocities(np.zeros((K, nf, 3)))
    e2.propagate(1234, 56, reassign_velocities=True)
    v2, x2 = e2.get_velocities(), e2.get_positions()
    e2.close()
    assert np.array_equal(x2, np.stack([xf] * K))
    for k in range(K):
        sg = np.sqrt(KB * temps[perm[k]] / flex.masses)[:, None]
        assert np.abs(v2[k] - sg * device_reassign_noise(1234, 56, k, nf)).max() <= 1e-5 * sg.min()
    # reassign on the constrained mixture: the oracle from the reassigned velocities (made to obey the constraints)
    m = oracle.Molecule(system)
    seed, it, n_steps, dt, gamma = 4321, 9, 8, 0.001, 5.0
    e.set_integrator(dt, gamma, n_steps, 'V R O R V')
    e.set_positions(np.stack([x] * K)); e.set_velocities(np.zeros((K, n, 3)))
    e.propagate(seed, it, reassign_velocities=True)
    xg, vg = e.get_positions(), e.get_velocities()
    e.close()
    for k in range(K):
        xo = x.copy()
        vo = np.ascontiguousarray(np.sqrt(KB * temps[perm[k]] / system.masses)[:, None] * device_reassign_noise(seed, it, k, n))
        oracle_run(m, xo, vo, device_noise(seed, it, k, n, n_steps), KB * temps[perm[k]], dt, gamma, n_steps, 'V R O R V')
        assert np.abs(xg[k] - xo).max() < 3e-7 and np.abs(vg[k] - vo).max() < 1e-4, (k, np.abs(xg[k] - xo).max(), np.abs(vg[k] - vo).max())


@pytest.mark.parametrize('name', ['mixture-shuffled', 'decane'])
def test_exclusions_equal_exceptions_that_carry_nothing(name):
    """Replacing every 1-2 / 1-3 exclusion by an exception with zero charge product, epsilon = 0 and sigma = 1 nm gives the
    same positions, velocities and energies bit for bit (the zero terms add exact zeros to their slots)."""
    system, x = MOLECULES[name]()
    alt = system.copy()
    ex = np.asarray(system.exclusions, float)
    alt.exceptions = np.concatenate([system.exceptions, np.c_[ex, np.zeros(len(ex)), np.ones(len(ex)), np.zeros(len(ex))]])
    alt.exclusions = np.zeros((0, 2), np.int64)
    temps = np.array([300.0, 500.0])
    K = len(temps)
    out = []
    for s in (system, alt):
        e = make_engine(s, temps)
        e.set_integrator(0.002, 5.0, 50, 'V R O R V')
        e.set_positions(np.stack([x] * K)); e.randomize_velocities(8)
        e.propagate(3, 4)
        out.append((e.get_positions(), e.get_velocities(), *e.get_replica_energies(), e.compute_energies()))
        e.close()
    for a, b in zip(*out):
        assert np.array_equal(a, b)


def test_molecules_above_32_atoms_are_refused():
    from openmmtools_b200 import states, _backend
    from openmmtools_b200._engine import EngineError
    system, x = H.alkane(11, hydrogens=[2] * 11)
    assert system.n_particles == 33
    with pytest.raises(EngineError) as err:
        gpu_engine(_lib.RX_SYSTEM_MOLECULE, 1, 1, 33)
    assert err.value.code == _lib.RX_ERR_UNSUPPORTED
    with pytest.raises(NotImplementedError):
        _backend.build_engine([states.ThermodynamicState(system, 300.0 * unit.kelvin)], 1)


def test_tables_beyond_shared_memory_are_refused_at_set_molecule():
    """1500 torsion terms on 32 atoms need more shared memory than a block can have: set_molecule refuses them (instead of a
    launch failing later); the 32-atom molecules of the other tests need more than the 48 KB available without opt-in and
    run."""
    from openmmtools_b200._engine import EngineError
    system, x = MOLECULES['decane']()
    big = system.copy()
    big.torsions = np.resize(system.torsions, (1500, 7))
    e = gpu_engine(_lib.RX_SYSTEM_MOLECULE, 2, 2, 32)
    with pytest.raises(EngineError) as err:
        e.set_molecule(big)
    assert err.value.code == _lib.RX_ERR_UNSUPPORTED
    e.set_molecule(system)
    e.set_states(np.array([300.0, 400.0]), np.ones(2))
    e.set_integrator(0.001, 5.0, 2, 'V R O R V')
    e.set_positions(np.stack([x] * 2)); e.randomize_velocities(1)
    e.propagate(1, 1)
    assert np.all(np.isfinite(e.compute_energies()))
    e.close()
