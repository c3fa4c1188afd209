"""RX_SYSTEM_MOLECULE in OBC implicit solvent (rx_set_implicit_solvent) on the GPU against the oracle
(oracle/rx_oracle_gb.c): energies, the T4 ligand's GB energy against AMBER sander, constrained Langevin steps with the
same noise, long launches, the minimiser, and the ParallelTemperingSampler docstring example on AlanineDipeptideImplicit."""
import os
import numpy as np
import pytest
import helpers as H
import implicit_helpers as IH
from helpers import KB, device_noise
from test_gpu_molecule import make_engine, oracle_run, constraint_error, projected_rms
from openmmtools_b200 import testsystems, unit, _lib, _engine

pytestmark = pytest.mark.gpu

SYSTEMS = {
    'alanine-dipeptide': lambda: IH.implicit_system('alanine-dipeptide'),
    'alanine-dipeptide-flexible': lambda: IH.implicit_system('alanine-dipeptide', None),
    'toluene': lambda: IH.implicit_system('toluene'),
    'toluene-flexible': lambda: IH.implicit_system('toluene', None),
    't4-ligand': lambda: IH.ligand(),
    'decane': lambda: (lambda s, x: (IH.obc(s), x))(*H.alkane(10)),                              # 32 atoms
    'waters-ion': lambda: (lambda s, x: (IH.obc(s), x))(*H.waters(10, ions=1, shuffle=3)),      # 31 atoms
    'ion': lambda: (lambda s, x: (IH.obc(s), x))(*H.ion()),                                     # n = 1
    'diatomic': lambda: (lambda s, x: (IH.obc(s), x))(*H.diatomic()),                           # n = 2
}


@pytest.mark.parametrize('model', ['OBC1', 'OBC2'])
@pytest.mark.parametrize('name', list(SYSTEMS))
def test_energy_rows_match_the_oracle(name, model):
    from oracle import implicit
    system, x = SYSTEMS[name]()
    system = IH.with_model(system, model)
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
    m = implicit.Molecule(system)
    U = np.array([m.energy(xk) for xk in xs])
    ref = U[:, None] / (KB * temps)[None, :]
    assert np.abs(u - ref).max() <= 1e-10 * max(1.0, np.abs(ref).max())
    ref100 = (U[:, None] + off[None, :]) / (KB * T100)[None, :]
    assert np.abs(u100 - ref100).max() <= 1e-10 * max(1.0, np.abs(ref100).max())


@pytest.mark.parametrize('coordinates,sander_out', [('ligand.crd', 'ligand-min.sander.out'),
                                                     ('ligand-minimized.crd', 'ligand-testenergy.sander.out')])
def test_ligand_gb_energy_on_the_device_matches_sander(coordinates, sander_out):
    s, x = IH.ligand(coordinates=coordinates)
    vac = s.copy(); vac.gb_radius = None
    U = []
    for system in (s, vac):
        e = make_engine(system, [300.0])
        e.set_positions(x[None])
        U.append(e.compute_energies()[0, 0] * KB * 300.0)
        e.close()
    egb = IH.sander_energies(os.path.join(IH.GOLDEN, 't4-' + sander_out))['EGB'] * IH.SANDER_ELEC_SCALE
    assert abs((U[0] - U[1]) / 4.184 - egb) <= 1e-4, ((U[0] - U[1]) / 4.184, egb)


@pytest.mark.parametrize('splitting,n_steps', [('V R O R V', 1), ('V R O R V', 25), ('O V R V O', 10), ('R V O', 7)])
@pytest.mark.parametrize('constraints', ['HBonds', None])
def test_constrained_steps_match_the_oracle_with_the_same_noise(splitting, n_steps, constraints):
    """The bounds of the vacuum test (test_gpu_molecule.py): f32 bonded forces, f64 GB forces."""
    from oracle import implicit
    system, x = IH.implicit_system('alanine-dipeptide', constraints)
    temps = np.array([300.0, 450.0, 600.0])
    K = len(temps)
    rng = np.random.default_rng(8)
    m = implicit.Molecule(system)
    v0 = np.stack([rng.normal(size=x.shape) * np.sqrt(KB * T / m.mass)[:, None] for T in temps])
    e = make_engine(system, temps)
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
    worst = [0.0, 0.0]
    for k in range(K):
        xo, vo = x.copy(), np.ascontiguousarray(v0[k])
        U = oracle_run(m, xo, vo, device_noise(seed, it, k, 22, n_steps * nO), KB * temps[perm[k]], dt, gamma, n_steps, splitting)
        worst = [max(worst[0], np.abs(xg[k] - xo).max()), max(worst[1], np.abs(vg[k] - vo).max())]
        assert np.abs(xg[k] - xo).max() < 3e-7 and np.abs(vg[k] - vo).max() < 1e-4, (k, worst)
        assert abs(pg[k] - U) < 2e-3 and abs(kg[k] - m.kinetic(vo)) < 2e-3
    print('worst: %.2e nm, %.2e nm/ps' % tuple(worst))


@pytest.mark.parametrize('name', ['alanine-dipeptide', 'toluene', 'waters-ion', 'decane'])
def test_long_launch_keeps_constraints_and_is_reproducible(name):
    system, x = SYSTEMS[name]()
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
    assert np.array_equal(xa, xb) and np.array_equal(va, vb) and np.array_equal(pa, pb)
    assert constraint_error(system, xa) < 1e-9
    assert np.all(np.isfinite(pa)) and np.all(ka > 0)
    # the replica energies the launch reports are the energy kernel's (u = beta U: equal up to the rounding of beta)
    e = make_engine(system, temps)
    e.set_positions(xa)
    u = e.compute_energies()
    e.close()
    assert np.abs(u[np.arange(K), np.arange(K)] * KB * temps - pa).max() <= 1e-14 * np.abs(pa).max()


@pytest.mark.parametrize('name', ['alanine-dipeptide', 'waters-ion'])
def test_register_resident_cluster_path_agrees_with_the_general_one(monkeypatch, name):
    system, x = SYSTEMS[name]()
    temps = np.linspace(300.0, 600.0, 6)
    K = len(temps)
    out = []
    for general in (False, True):
        if general:
            monkeypatch.setenv('RX_MOL_NO_STAR', '1')
        e = make_engine(system, temps, constraint_tolerance=1e-12)
        e.set_integrator(0.002, 5.0, 1000, 'V R O R V')
        e.set_positions(np.stack([x] * K)); e.randomize_velocities(5)
        e.propagate(9, 3)
        out.append((e.get_positions(), e.get_velocities()))
        e.close()
    (xs, vs), (xg, vg) = out
    for xx in (xs, xg):
        assert constraint_error(system, xx) < 1e-9
    # 1000 stochastic steps amplify the solvers' different stopping points; 40 steps stay within the vacuum bound
    assert np.all(np.isfinite(xs)) and np.all(np.isfinite(xg))
    out = []
    for general in (False, True):
        monkeypatch.delenv('RX_MOL_NO_STAR', raising=False)
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


@pytest.mark.parametrize('name', ['alanine-dipeptide', 'toluene', 'waters-ion'])
def test_minimizer_reports_the_projected_rms_force(name):
    from oracle import implicit
    system, x = SYSTEMS[name]()
    m = implicit.Molecule(system)
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
        assert abs(rms[k] - ref) <= 1e-12 * ref, (k, rms[k], ref)
        assert rms[k] <= tol and ref <= tol, (k, rms[k], ref, its[k])
        assert U < m.energy(x0[k]) - 1.0
        assert constraint_error(system, xm[k]) < 1e-8


def test_parallel_tempering_docstring_example_runs_stores_and_resumes(tmp_path):
    """paralleltempering.py:61's example on AlanineDipeptideImplicit, with LangevinSplittingDynamicsMove for GHMC."""
    from oracle import implicit
    from openmmtools_b200 import states, mcmc
    from openmmtools_b200.multistate import ParallelTemperingSampler, MultiStateReporter
    testsystem = testsystems.AlanineDipeptideImplicit()
    n_replicas = 3
    T_min, T_max = 298.0 * unit.kelvin, 600.0 * unit.kelvin
    reference_state = states.ThermodynamicState(testsystem.system, T_min)
    move = mcmc.LangevinSplittingDynamicsMove(timestep=2.0 * unit.femtoseconds, n_steps=50)

    def new(path):
        s = ParallelTemperingSampler(mcmc_moves=move, number_of_iterations=4, seed=3)
        s.create(reference_state, states.SamplerState(testsystem.positions), MultiStateReporter(path, checkpoint_interval=1),
                 min_temperature=T_min, max_temperature=T_max, n_temperatures=n_replicas)
        return s
    a = new(str(tmp_path / 'a.nc'))
    a.run()
    assert a.iteration == 4
    m = implicit.Molecule(testsystem.system)
    T = np.array([st.temperature.value_in_unit(unit.kelvin) for st in a._thermodynamic_states])
    u = np.array(a._energy_thermodynamic_states)
    for k, st in enumerate(a.sampler_states):
        U = m.energy(np.ascontiguousarray(st.positions.value_in_unit(unit.nanometer), np.float64))
        assert np.abs(u[k] - U / (KB * T)).max() <= 1e-10 * max(1.0, np.abs(u[k]).max())
    b = new(str(tmp_path / 'b.nc'))
    b.run(2)
    del b
    c = ParallelTemperingSampler.from_storage(str(tmp_path / 'b.nc'))
    assert c.iteration == 2
    c.run()
    assert c.iteration == 4
    assert np.array_equal(c._replica_thermodynamic_states, a._replica_thermodynamic_states)
    assert np.array_equal(c._energy_thermodynamic_states, a._energy_thermodynamic_states)
    assert np.array_equal(np.stack([st._positions for st in c.sampler_states]), np.stack([st._positions for st in a.sampler_states]))


def test_refusals():
    s, x = IH.implicit_system('alanine-dipeptide')
    e = make_engine(s, [300.0])
    for bad in (dict(radius=np.zeros(22)), dict(radius=np.full(22, 0.009))):
        with pytest.raises(_engine.EngineError):
            e.set_implicit_solvent(bad['radius'], s.gb_scale, *s.gb_parameters)
    # a refused call leaves the engine as it was: still in implicit solvent
    e.set_positions(x[None])
    u_gb = e.compute_energies()[0, 0]
    with pytest.raises(_engine.EngineError):
        e.set_implicit_solvent(np.zeros(22), s.gb_scale, *s.gb_parameters)
    assert e.compute_energies()[0, 0] == u_gb
    # set_molecule returns the engine to vacuum
    vac = s.copy(); vac.gb_radius = None
    e.set_molecule(vac)
    e.set_states(np.array([300.0]), np.ones(1))
    e.set_positions(x[None])
    from oracle import oracle
    assert abs(e.compute_energies()[0, 0] * KB * 300.0 - oracle.Molecule(vac).energy(x)) < 1e-9 * abs(oracle.Molecule(vac).energy(x))
    e.close()
    lj = H.gpu_engine(_lib.RX_SYSTEM_HARMONIC, 1, 1, 22)
    with pytest.raises(_engine.EngineError):
        lj.set_implicit_solvent(s.gb_radius, s.gb_scale, *s.gb_parameters)
    lj.close()
