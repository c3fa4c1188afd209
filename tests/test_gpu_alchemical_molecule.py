"""Alchemically decoupled small molecules on the GPU: energy rows against the float64 oracle (oracle/alchemical_molecule.py),
dynamics, HMC, Monte Carlo moves and minimisation at alchemical states, and free energies that are exact by construction --
a constant offset (a rigid charged diatomic in OBC) and 1-D quadrature (a bonded dimer)."""
import numpy as np
import pytest
from openmmtools_b200 import alchemy, mcmc, multistate, states, testsystems, unit, _backend
from openmmtools_b200.alchemy import AbsoluteAlchemicalFactory, AlchemicalRegion, AlchemicalState
from openmmtools_b200.system import System, MOLECULE

pytestmark = pytest.mark.gpu
KB = 8.31446261815324e-3

CASES = {
    'toluene-vacuum': (testsystems.TolueneVacuum, range(15)),
    'toluene-obc1': (testsystems.TolueneImplicit, range(15)),
    'toluene-obc2': (testsystems.TolueneImplicitOBC2, range(15)),
    'toluene-obc1-partial': (testsystems.TolueneImplicit, range(7, 15)),
    'toluene-obc2-partial': (testsystems.TolueneImplicitOBC2, [0, 3, 9, 10]),
    'aladip-vacuum-partial': (testsystems.AlanineDipeptideVacuum, range(6, 12)),
    'aladip-obc1-unconstrained': (lambda: testsystems.AlanineDipeptideImplicit(constraints=None), range(22)),
}
LADDER = [(1.0, 1.0, 300.0), (1.0, 0.6, 300.0), (1.0, 0.0, 310.0), (0.7, 0.0, 300.0), (0.7, 0.0, 300.0), (0.3, 0.0, 320.0),
          (0.0, 0.0, 300.0), (0.0, 0.3, 300.0)]


def _make(name, **region):
    cls, atoms = CASES[name]
    t = cls()
    return t, AbsoluteAlchemicalFactory().create_alchemical_system(t.system, AlchemicalRegion(alchemical_atoms=atoms, **region))


def _protocol(asys, ladder):
    return [states.CompoundThermodynamicState(states.ThermodynamicState(asys, T * unit.kelvin), [_astate(asys, ls, le)])
            for ls, le, T in ladder]


def _astate(asys, ls, le):
    a = AlchemicalState.from_system(asys)
    a.lambda_sterics, a.lambda_electrostatics = ls, le
    return a


def _x(t):
    return np.ascontiguousarray(t.positions.value_in_unit(unit.nanometer), np.float64)


def _oracle_rows(m, xs, ladder):
    return np.array([[m.energy(x, ls, le) / (KB * T) for ls, le, T in ladder] for x in xs])


@pytest.mark.parametrize('name', sorted(CASES))
@pytest.mark.parametrize('annihilate', [(False, True), (True, False)])
def test_energy_rows_match_the_oracle(name, annihilate):
    from oracle.alchemical_molecule import AlchemicalMolecule
    t, asys = _make(name, annihilate_sterics=annihilate[0], annihilate_electrostatics=annihilate[1])
    m = AlchemicalMolecule(asys)
    rng = np.random.default_rng(3)
    K = 5
    xs = np.stack([_x(t) + rng.normal(0, 0.004, _x(t).shape) for _ in range(K)])
    tss = _protocol(asys, LADDER)
    eng = _backend.build_engine(tss, K)
    try:
        eng.set_positions(xs)
        u = eng.compute_energies()
        ref = _oracle_rows(m, xs, LADDER)
        np.testing.assert_allclose(u, ref, rtol=1e-10, atol=0)
        # unsampled states: compute_energies_at on other lambdas, the resident matrix untouched
        other = [(0.5, 0.5, 300.0), (0.1, 1.0, 300.0), (1.0, 0.2, 350.0)]
        _, tab = _backend.engine_tables(_protocol(asys, other))
        ua = eng.compute_energies_at(**tab)
        np.testing.assert_allclose(ua, _oracle_rows(m, xs, other), rtol=1e-10, atol=0)
        assert eng.get_energies().tobytes() == u.tobytes()
    finally:
        eng.close()


def _run(asys, t, ladder, move, n_iterations=3, seed=7):
    s = multistate.ReplicaExchangeSampler(mcmc_moves=move, number_of_iterations=n_iterations, seed=seed)
    s.create(_protocol(asys, ladder), [states.SamplerState(t.positions)])
    s.run()
    return s


def _check_sampler_energies(s, m, ladder, asys):
    """The stored energy matrix is the oracle's at the replicas' final positions; the propagation's potential of each
    replica is the energy at its own state."""
    xs = np.stack([st.positions.value_in_unit(unit.nanometer) for st in s.sampler_states])
    np.testing.assert_allclose(s._energy_thermodynamic_states, _oracle_rows(m, xs, ladder), rtol=1e-10, atol=0)
    for c in np.asarray(asys.constraints).reshape(-1, 3):
        d = np.linalg.norm(xs[:, int(c[0])] - xs[:, int(c[1])], axis=-1)
        assert np.all(np.abs(d - c[2]) < 1e-6 * c[2])


@pytest.mark.parametrize('name', ['toluene-vacuum', 'toluene-obc1', 'toluene-obc2-partial', 'aladip-obc1-unconstrained'])
def test_langevin_hmc_and_mc_moves_at_alchemical_states(name):
    from oracle.alchemical_molecule import AlchemicalMolecule
    t, asys = _make(name)
    m = AlchemicalMolecule(asys)
    ladder = LADDER[:4] + LADDER[5:7]
    lang = mcmc.LangevinSplittingDynamicsMove(timestep=1.0 * unit.femtosecond, n_steps=50)
    s = _run(asys, t, ladder, lang)
    _check_sampler_energies(s, m, ladder, asys)
    hmc = mcmc.HMCMove(timestep=0.5 * unit.femtosecond, n_steps=5)
    s = _run(asys, t, ladder, hmc)
    _check_sampler_energies(s, m, ladder, asys)
    acc, trials = s._engine.get_hmc_statistics()
    assert trials.sum() > 0 and 0 < acc.sum() <= trials.sum()
    e_old, e_new = s._engine.get_hmc_energies()
    assert np.all(np.isfinite(e_old)) and np.all(np.isfinite(e_new))
    seq = mcmc.SequenceMove([mcmc.MCDisplacementMove(displacement_sigma=0.02 * unit.nanometer, atom_subset=list(range(asys.n_particles))),
                             mcmc.MCRotationMove(atom_subset=list(range(asys.n_particles))), lang])
    s = _run(asys, t, ladder, seq)
    _check_sampler_energies(s, m, ladder, asys)


def test_langevin_step_matches_the_oracle_forces():
    """Unconstrained molecules: one V step of the device (f32 forces) against the oracle's f64 forces."""
    from oracle.alchemical_molecule import AlchemicalMolecule
    for name in ('toluene-obc2-partial', 'aladip-obc1-unconstrained'):
        t, asys = _make(name, annihilate_sterics=True)
        if asys.getNumConstraints():
            asys.constraints = np.zeros((0, 3))
        asys.remove_cm_motion = False
        m = AlchemicalMolecule(asys)
        ladder = [(0.6, 0.4, 300.0), (0.2, 0.9, 300.0)]
        eng = _backend.build_engine(_protocol(asys, ladder), 2)
        try:
            x = np.stack([_x(t)] * 2)
            eng.set_replica_states(np.arange(2))
            eng.set_positions(x)
            eng.set_velocities(np.zeros_like(x))
            dt = 1e-4
            eng.set_integrator(dt, 0.0, 1, 'V O R')   # (O: a no-op without friction)
            eng.propagate(1, 0)
            v = eng.get_velocities()
            for k, (ls, le, _) in enumerate(ladder):
                _, F = m.energy(x[k], ls, le, forces=True)
                ref = dt * F / asys.masses[:, None]
                scale = np.abs(ref).max()
                # (f32 terms: 2.1e-5 of the largest force measured on an H100)
                assert np.abs(v[k] - ref).max() <= 1e-4 * scale, (name, k, np.abs(v[k] - ref).max() / scale)
        finally:
            eng.close()


def test_minimize_at_an_alchemical_state_reaches_a_stationary_point_of_the_oracle():
    from oracle.alchemical_molecule import AlchemicalMolecule
    t, asys = _make('aladip-obc1-unconstrained')
    m = AlchemicalMolecule(asys)
    ladder = [(0.5, 0.25, 300.0), (1.0, 0.0, 300.0)]
    eng = _backend.build_engine(_protocol(asys, ladder), 2)
    try:
        eng.set_replica_states(np.arange(2))
        eng.set_positions(np.stack([_x(t)] * 2))
        rms, its = eng.minimize(1.0, 20000)
        x = eng.get_positions()
        for k, (ls, le, _) in enumerate(ladder):
            _, F = m.energy(x[k], ls, le, forces=True)
            assert np.sqrt((F ** 2).mean()) == pytest.approx(rms[k], rel=1e-6, abs=1e-8)
            assert rms[k] <= 1.0
            assert m.energy(x[k], ls, le) < m.energy(_x(t), ls, le)
    finally:
        eng.close()


def test_non_alchemical_molecule_runs_unchanged_with_an_electrostatic_lambda_in_its_states():
    """A molecule without a region ignores lambda_electrostatics: the same bits whatever the table holds."""
    t = testsystems.TolueneImplicit()
    tss = [states.ThermodynamicState(t.system, T * unit.kelvin) for T in (300.0, 330.0)]
    out = []
    for le in (None, [0.0, 0.5]):
        eng = _backend.build_engine(tss, 2)
        try:
            _, tab = _backend.engine_tables(tss)
            eng.set_states(**tab, lambda_electrostatics=le)
            eng.set_positions(np.stack([_x(t)] * 2))
            eng.randomize_velocities(5)
            eng.set_integrator(1e-3, 1.0, 20)
            eng.propagate(3, 1)
            out.append((eng.get_positions().tobytes(), eng.get_velocities().tobytes(), eng.compute_energies().tobytes()))
        finally:
            eng.close()
    assert out[0] == out[1]


# -- exact free energies ----------------------------------------------------------------------------------------------
def _dimer(rigid, obc, d=0.2):
    """Two atoms with charges of one sign: rigid (one constraint, the pair excluded) or harmonically bonded (the pair
    interacting through soft-core LJ, Coulomb and GB)."""
    s = System(MOLECULE, [12.0, 16.0])
    s.charge = np.array([0.4, 0.3]); s.sigma = np.array([0.2, 0.22]); s.epsilon = np.array([0.4, 0.6])
    s.angles = np.zeros((0, 5)); s.torsions = np.zeros((0, 7)); s.exceptions = np.zeros((0, 5))
    if rigid:
        s.bonds = np.zeros((0, 4)); s.constraints = np.array([[0, 1, d]]); s.exclusions = np.array([[0, 1]])
    else:
        s.bonds = np.array([[0, 1, 3000.0, 0.25]]); s.constraints = np.zeros((0, 3)); s.exclusions = np.zeros((0, 2), np.int64)
    s.remove_cm_motion = False
    if obc:
        from openmmtools_b200.amber import obc_parameters
        s.gb_parameters = obc_parameters(implicitSolvent=obc)
        s.gb_radius = np.array([0.17, 0.15]); s.gb_scale = np.array([0.72, 0.85])
    x = np.array([[0.0, 0.0, 0.0], [d if rigid else 0.25, 0.0, 0.0]])
    return s, x


def _free_energy(asys, x0, ladder, unsampled, n_iterations, path, move):
    s = multistate.ReplicaExchangeSampler(mcmc_moves=move, number_of_iterations=n_iterations, seed=17)
    s.create(_protocol(asys, ladder), [states.SamplerState(unit.Quantity(x0, unit.nanometer))],
             storage=multistate.MultiStateReporter(str(path), checkpoint_interval=50),
             unsampled_thermodynamic_states=_protocol(asys, unsampled))
    s.run()
    a = multistate.ReplicaExchangeAnalyzer(multistate.MultiStateReporter(str(path), open_mode='r'))
    D, dD = a.get_free_energy()
    return s, D, dD


@pytest.mark.parametrize('obc', ['OBC1', 'OBC2'])
def test_free_energy_of_a_rigid_diatomic_is_the_energy_offset(obc, tmp_path):
    from oracle.alchemical_molecule import AlchemicalMolecule
    sysd, x0 = _dimer(True, obc)
    asys = AbsoluteAlchemicalFactory().create_alchemical_system(sysd, AlchemicalRegion(alchemical_atoms=[0]))
    m = AlchemicalMolecule(asys)
    T = 300.0
    ladder = [(1.0, le, T) for le in (1.0, 0.75, 0.5, 0.25, 0.0)]
    move = mcmc.LangevinSplittingDynamicsMove(timestep=1.0 * unit.femtosecond, n_steps=20)
    s, D, dD = _free_energy(asys, x0, ladder[1:-1], [ladder[0], ladder[-1]], 100, tmp_path / 'rigid', move)
    beta = 1.0 / (KB * T)
    xr = lambda r: np.array([[0.0, 0.0, 0.0], [r, 0.0, 0.0]])
    dU = np.array([m.energy(xr(0.2), 1.0, le) - m.energy(xr(0.2), 1.0, 1.0) for _, le, _ in ladder])
    h = 1e-6
    slope = np.array([(m.energy(xr(0.2 + h), 1.0, le) - m.energy(xr(0.2 + h), 1.0, 1.0)
                       - m.energy(xr(0.2 - h), 1.0, le) + m.energy(xr(0.2 - h), 1.0, 1.0)) / (2 * h) for _, le, _ in ladder])
    xs = np.stack([st.positions.value_in_unit(unit.nanometer) for st in s.sampler_states])
    dr = np.abs(np.linalg.norm(xs[:, 0] - xs[:, 1], axis=-1) - 0.2).max()
    bound = 2 * beta * np.abs(slope) * max(dr, 1e-9) + 1e-9
    assert np.all(np.abs(D[0] - beta * dU) <= bound), (D[0], beta * dU, bound)
    assert np.abs(beta * dU).max() > 1.0    # (an offset worth measuring)


@pytest.mark.parametrize('obc', [None, 'OBC2'])
def test_free_energies_of_a_bonded_dimer_match_quadrature(obc, tmp_path):
    from oracle.alchemical_molecule import AlchemicalMolecule
    sysd, x0 = _dimer(False, obc)
    asys = AbsoluteAlchemicalFactory().create_alchemical_system(sysd, AlchemicalRegion(alchemical_atoms=[0]))
    m = AlchemicalMolecule(asys)
    T = 300.0
    beta = 1.0 / (KB * T)
    ends = [(1.0, 1.0, T), (0.0, 0.0, T)]
    ladder = [(1.0, 0.8, T), (1.0, 0.45, T), (1.0, 0.1, T), (0.75, 0.0, T), (0.5, 0.0, T), (0.25, 0.0, T), (0.05, 0.0, T)]
    move = mcmc.LangevinSplittingDynamicsMove(timestep=1.0 * unit.femtosecond, n_steps=50)
    _, D, dD = _free_energy(asys, x0, ladder, ends, 1500, tmp_path / 'dimer', move)
    r = np.linspace(0.05, 0.6, 4001)
    xr = lambda q: np.array([[0.0, 0.0, 0.0], [q, 0.0, 0.0]])
    every = [ends[0]] + ladder + [ends[1]]
    logZ = []
    for ls, le, _ in every:
        u = np.array([m.energy(xr(q), ls, le) for q in r]) * beta
        w = r ** 2 * np.exp(-(u - u.min()))
        logZ.append(np.log(np.trapezoid(w, r)) - u.min())
    exact = -(np.array(logZ)[None, :] - np.array(logZ)[:, None])
    n = len(every)
    off = ~np.eye(n, dtype=bool)
    assert np.all(np.abs(D - exact)[off] <= 4 * dD[off]), (D[0], exact[0], dD[0])
    assert np.abs(exact[0, -1]) > 2.0


# -- storage and sharding ---------------------------------------------------------------------------------------------
def toluene_sampler(n_iterations=1000, storage=None, communicator=None):
    """Replica exchange over a joint lambda ladder of a partly alchemical TolueneImplicitOBC2, with unsampled end states."""
    t = testsystems.TolueneImplicitOBC2()
    asys = AbsoluteAlchemicalFactory().create_alchemical_system(t.system, AlchemicalRegion(alchemical_atoms=range(7, 15)))
    ladder = [(1.0, 0.8, 300.0), (1.0, 0.4, 300.0), (1.0, 0.0, 300.0), (0.6, 0.0, 300.0), (0.3, 0.0, 300.0), (0.1, 0.0, 300.0)]
    kw = {} if communicator is None else dict(communicator=communicator)
    s = multistate.ReplicaExchangeSampler(mcmc_moves=mcmc.LangevinSplittingDynamicsMove(n_steps=20), seed=5,
                                          number_of_iterations=n_iterations, **kw)
    s.create(_protocol(asys, ladder), [states.SamplerState(t.positions)], storage=storage,
             unsampled_thermodynamic_states=_protocol(asys, [(1.0, 1.0, 300.0), (0.0, 0.0, 300.0)]))
    return s


def test_resumed_alchemical_molecule_run_stores_the_same_data(tmp_path):
    full = toluene_sampler(40, multistate.MultiStateReporter(str(tmp_path / 'full.nc'), checkpoint_interval=10))
    full.run()
    part = toluene_sampler(40, multistate.MultiStateReporter(str(tmp_path / 'part.nc'), checkpoint_interval=10))
    part.run(25)
    del part
    resumed = multistate.ReplicaExchangeSampler.from_storage(str(tmp_path / 'part.nc'))
    resumed.run()
    a = multistate.MultiStateReporter(str(tmp_path / 'full.nc'), open_mode='r')
    b = multistate.MultiStateReporter(str(tmp_path / 'part.nc'), open_mode='r')
    for it in range(0, 41):
        ea, eb = a.read_energies(it), b.read_energies(it)
        for x, y in zip(ea, eb):
            assert np.asarray(x).tobytes() == np.asarray(y).tobytes(), it
        assert np.array_equal(a.read_replica_thermodynamic_states(it), b.read_replica_thermodynamic_states(it))
    for it in (10, 20, 30, 40):
        pa = [s.positions.value_in_unit(unit.nanometer) for s in a.read_sampler_states(it)]
        pb = [s.positions.value_in_unit(unit.nanometer) for s in b.read_sampler_states(it)]
        assert all(np.asarray(x).tobytes() == np.asarray(y).tobytes() for x, y in zip(pa, pb)), it
    fa = multistate.ReplicaExchangeAnalyzer(a).get_free_energy()
    fb = multistate.ReplicaExchangeAnalyzer(b).get_free_energy()
    assert fa[0].tobytes() == fb[0].tobytes()


TWO_RANK_WORKER = r'''
import os, sys
sys.path.insert(0, %(root)r)
sys.path.insert(0, os.path.join(%(root)r, 'tests'))
import numpy as np
import torch.distributed as dist
dist.init_process_group('gloo')
from test_gpu_alchemical_molecule import toluene_sampler
from openmmtools_b200._dist import TorchCommunicator
s = toluene_sampler(communicator=TorchCommunicator())
s.run(4)
np.savez(%(out)r + '_%%d.npz' %% dist.get_rank(), u=s._energy_thermodynamic_states, uu=s._energy_unsampled_states,
         perm=s._replica_thermodynamic_states, x=s._engine.get_positions(), k0=s._engine.k0)
dist.barrier()
'''


def test_two_ranks_reproduce_one_gpu(tmp_path):
    import ctypes
    import os
    import subprocess
    import sys
    try:
        cuda = ctypes.CDLL('libcudart.so.12')
    except OSError:
        cuda = ctypes.CDLL('libcudart.so')
    n = ctypes.c_int()
    cuda.cudaGetDeviceCount(ctypes.byref(n))
    if n.value < 2:
        pytest.skip('needs 2 GPUs')
    s = toluene_sampler()
    s.run(4)
    u1, uu1, p1, x1 = (s._energy_thermodynamic_states.copy(), s._energy_unsampled_states.copy(),
                       s._replica_thermodynamic_states.copy(), s._engine.get_positions())
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script, out = tmp_path / 'w.py', str(tmp_path / 'res')
    script.write_text(TWO_RANK_WORKER % {'root': root, 'out': out})
    r = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2',
                        '--master-addr', '127.0.0.1', '--master-port', '29547', str(script)],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    for rank in range(2):
        d = np.load(out + '_%d.npz' % rank)
        assert np.array_equal(d['perm'], p1) and np.array_equal(d['u'], u1)
        k0 = int(d['k0'])
        assert np.array_equal(d['uu'][k0:k0 + d['x'].shape[0]], uu1[k0:k0 + d['x'].shape[0]])
        assert np.array_equal(d['x'], x1[k0:k0 + d['x'].shape[0]])
