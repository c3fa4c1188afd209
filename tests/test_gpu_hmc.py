"""Hybrid Monte Carlo on the device (k_propagate_hmc, rx_set_hmc_integrator) against the host oracle of tests/hmc_oracle.py
fed the device's own draws, its rejection and NaN rules, its stationary distribution on the harmonic oscillator, its
invariance under the launch layout, and the samplers that run it."""
import os
import subprocess
import sys
import numpy as np
import pytest
import hmc_oracle as ho
from helpers import KB, lj_setup, oracle_system, min_image, wrap, gpu_engine, scattered_alch
from regions_ref import RegionsReference
from openmmtools_b200 import _lib, mcmc, unit, states, alchemy, testsystems, multistate

pytestmark = pytest.mark.gpu

SEED, IT = 0x1234_5678_9ABC, 7


def lj_engine(s, K, lambdas, temps, dt, n_steps, use_switch=True):
    eng = gpu_engine(_lib.RX_SYSTEM_LJ_ALCH, K, len(lambdas), s['N'], box=tuple(s['box']), r_cutoff=s['rc'], r_switch=s['rs'],
                     use_switch=use_switch)
    eng.set_particles(s['sigma'], s['eps'], s['mass'], s['alch'])
    eng.set_states(temps, lambda_sterics=lambdas)
    eng.set_hmc_integrator(dt, n_steps)
    return eng


def f32(a):
    return np.asarray(a, np.float32).astype(np.float64)


def check_replica(eng, k, x0, mass, kT, ef, dt, n_steps, xg, vg, box=None, tol_x=5e-4, tol_v=5e-3, cons=None,
                  iterations=(IT,)):
    """The device's replica k against the oracle run on the same draws: positions, the velocities the last trajectory ended
    with (kept also after a rejection), the last trial's energies, the number of accepted trials, and the last accept bit
    as the oracle decides it from the device's dH and uniform.  `iterations`: the launches the device ran from x0, in order;
    the oracle runs on from its own end state (wrapped into the box between launches, as the device wraps it).  Returns
    the (Eold, Enew, accepted) of every trial in launch order, n_steps per launch."""
    x = f32(x0) if cons is None else np.array(x0, np.float64)
    trials = []
    for q, it in enumerate(iterations):
        if q and box is not None:
            x = wrap(x, box)
        gauss, u = ho.draws(SEED, it, k, len(mass), n_steps)
        x, v, tr = ho.run(x, mass, kT, ef, gauss, u, dt, n_steps, cons)
        trials += tr
    d = xg[k] - x if box is None else min_image(xg[k] - wrap(x, box), box)
    assert np.abs(d).max() < tol_x
    assert np.abs(vg[k] - v).max() < tol_v
    e_old, e_new = eng.get_hmc_energies()
    e0, e1, last = trials[-1]
    assert abs(e_old[k] - e0) < 1e-5 * abs(e0) + 2e-3 and abs(e_new[k] - e1) < 1e-5 * abs(e1) + 2e-3
    acc, n = eng.get_hmc_statistics()
    assert n[k] == len(iterations) * n_steps and acc[k] == sum(t[2] for t in trials)
    assert (u[-1] <= np.exp(-(e_new[k] - e_old[k]) / kT)) == last
    return trials


@pytest.mark.parametrize('N,cl,switch,sort,regions', [
    (256, 1, True, True, False), (300, 2, True, True, False), (300, 4, True, True, False), (300, 4, True, False, False),
    (256, 1, False, True, False), (1100, None, True, True, False), (256, 1, True, True, True), (300, 4, True, True, True)])
def test_lj_trials_match_oracle(monkeypatch, N, cl, switch, sort, regions):
    if cl is not None:
        monkeypatch.setenv('RX_CLUSTER', str(cl))
    if not sort:
        monkeypatch.setenv('RX_NO_SORT', '1')
    K, n_steps, dt = 2, 4, 0.002
    lambdas, temps = np.array([1.0, 0.4]), np.array([300.0, 330.0])
    perm = np.array([1, 0])
    if regions:   # two alchemical regions (the REG instantiations), second region at 1 - lambda
        s = lj_setup(N=N, seed=N, alch=scattered_alch(N))
        ids = np.where(s['alch'] != 0, 1 + np.arange(N) % 2, 0).astype(np.uint8)
        eng = gpu_engine(_lib.RX_SYSTEM_LJ_ALCH, K, 2, N, box=tuple(s['box']), r_cutoff=s['rc'], r_switch=s['rs'], use_switch=True)
        eng.set_particles(s['sigma'], s['eps'], s['mass'], (ids != 0).astype(np.uint8))
        eng.set_alchemical_regions(ids, False, False)
        eng.set_states(temps, lambda_sterics=lambdas, lambda_sterics_2=1.0 - lambdas)
        eng.set_hmc_integrator(dt, n_steps)
        ref = RegionsReference(s, ids)
        ef = [lambda y, l=l: ref.energy(y, lambdas[l], 1.0 - lambdas[l], forces=True) for l in range(2)]
    else:
        s = lj_setup(N=N, n_alch=6, seed=N)
        eng = lj_engine(s, K, lambdas, temps, dt, n_steps, use_switch=switch)
        osys = oracle_system(s, use_switch=switch)
        ef = [ho.lj(osys, lam) for lam in lambdas]
    x0 = np.stack([s['x']] * K)
    eng.set_positions(x0); eng.set_velocities(np.zeros_like(x0))
    eng.set_replica_states(perm)
    eng.propagate(SEED, IT)
    xg, vg = eng.get_positions(), eng.get_velocities()
    for k in range(K):
        check_replica(eng, k, x0[k], s['mass'], KB * temps[perm[k]], ef[perm[k]], dt, n_steps, xg, vg, s['box'])


def harmonic_engine(K, N, Ks, x0s, temps, dt, n_steps):
    eng = gpu_engine(_lib.RX_SYSTEM_HARMONIC, K, len(Ks), N)
    eng.set_particles(None, None, np.full(N, 39.948), None)
    eng.set_states(temps, None, np.zeros(len(Ks)), Ks, x0s)
    eng.set_hmc_integrator(dt, n_steps)
    return eng


def test_harmonic_trials_match_oracle():
    K, N, n_steps, dt = 3, 5, 6, 0.4
    Ks, x0s, temps = np.array([40.0, 90.0, 160.0]), np.array([[0.0, 0, 0], [0.1, 0, 0], [0.0, -0.1, 0.05]]), np.array([300.0, 310.0, 320.0])
    eng = harmonic_engine(K, N, Ks, x0s, temps, dt, n_steps)
    rng = np.random.default_rng(4)
    x0 = rng.normal(scale=0.1, size=(K, N, 3))
    eng.set_positions(x0); eng.set_velocities(np.zeros_like(x0))
    perm = np.array([2, 0, 1])
    eng.set_replica_states(perm)
    eng.propagate(SEED, IT)
    xg, vg = eng.get_positions(), eng.get_velocities()
    decisions = []
    for k in range(K):
        l = perm[k]
        decisions += [t[2] for t in check_replica(eng, k, x0[k], np.full(N, 39.948), KB * temps[l], ho.harmonic(Ks[l], x0s[l]),
                                                  dt, n_steps, xg, vg, tol_x=2e-5, tol_v=2e-4)]
    assert 0 < sum(decisions) < len(decisions)   # both branches ran


def test_rejected_trials_leave_positions_bit_identical():
    K, N = 2, 4
    eng = harmonic_engine(K, N, np.array([4.184e4, 4.184e4]), np.zeros((2, 3)), np.array([300.0, 300.0]), 0.1, 3)
    x0 = f32(np.random.default_rng(1).normal(scale=0.05, size=(K, N, 3)))
    eng.set_positions(x0); eng.set_velocities(np.zeros_like(x0))
    eng.propagate(SEED, IT)
    acc, n = eng.get_hmc_statistics()
    assert list(acc) == [0, 0] and list(n) == [3, 3]
    e0, e1 = eng.get_hmc_energies()
    assert np.all(e1 - e0 > 1e3)
    assert np.array_equal(eng.get_positions(), x0)


def test_harmonic_oscillator_samples_boltzmann_exactly():
    """<x^2> per degree of freedom = kT/K at a timestep where about half the trials are accepted; velocity Verlet with
    velocities redrawn the same way (numpy's generator, on the host) but no Metropolis test inflates it by
    1/(1 - (omega dt / 2)^2) = 4/3 there, which the same bound detects."""
    K, N, n_steps, T = 128, 32, 10, 300.0
    m = 39.948
    Kc = m                       # omega = 1 / ps
    dt = 1.0                     # omega dt = 1
    kT = KB * T
    eng = harmonic_engine(K, N, np.array([Kc]), np.zeros((1, 3)), np.array([T]), dt, n_steps)
    rng = np.random.default_rng(5)
    eng.set_positions(rng.normal(scale=np.sqrt(kT / Kc), size=(K, N, 3)))
    eng.set_velocities(np.zeros((K, N, 3)))
    eng.set_replica_states(np.zeros(K, np.int64))
    per = []
    for it in range(220):
        eng.propagate(SEED, it)
        if it >= 20:
            x = eng.get_positions()
            per.append((x * x).mean(axis=(1, 2)))
    r = np.mean(per, axis=0) / (kT / Kc)             # per replica (independent chains)
    mean, sem = r.mean(), r.std(ddof=1) / np.sqrt(K)
    acc, n = eng.get_hmc_statistics()
    rate = acc.sum() / n.sum()
    assert 0.2 < rate < 0.8, rate
    assert abs(mean - 1.0) < 5 * sem + 0.005, (mean, sem)
    # the same bound fails without the Metropolis test (host, vectorised over chains)
    x = rng.normal(scale=np.sqrt(kT / Kc), size=(K, N, 3))
    acc_u = []
    for it in range(220):
        for _ in range(n_steps):
            v = rng.normal(size=x.shape) * np.sqrt(kT / m)
            for _ in range(n_steps):
                v = v - 0.5 * dt * Kc * x / m; x = x + dt * v; v = v - 0.5 * dt * Kc * x / m
        if it >= 20:
            acc_u.append((x * x).mean(axis=(1, 2)))
    ru = np.mean(acc_u, axis=0) / (kT / Kc)
    assert abs(ru.mean() - 1.0) > 5 * ru.std(ddof=1) / np.sqrt(K) + 0.005


def test_same_bits_at_every_layout(monkeypatch):
    s = lj_setup(N=600, n_alch=6, seed=3)
    K, lambdas, temps = 3, np.array([1.0, 0.5, 0.0]), np.array([300.0, 300.0, 300.0])
    x0 = np.stack([s['x']] * K)
    out = []
    for cl, sort in ((1, True), (2, True), (4, True), (4, False)):
        monkeypatch.setenv('RX_CLUSTER', str(cl))
        if sort:
            monkeypatch.delenv('RX_NO_SORT', raising=False)
        else:
            monkeypatch.setenv('RX_NO_SORT', '1')
        eng = lj_engine(s, K, lambdas, temps, 0.003, 12)
        eng.set_positions(x0); eng.set_velocities(np.zeros_like(x0))
        eng.propagate(SEED, IT)
        eng.propagate(SEED, IT + 1)
        out.append((eng.get_positions(), eng.get_velocities(), eng.get_hmc_statistics(), eng.get_hmc_energies()))
        eng.close()
    for o in out[1:]:
        assert np.array_equal(o[0], out[0][0]) and np.array_equal(o[1], out[0][1])
        assert all(np.array_equal(a, b) for a, b in zip(o[2], out[0][2]))
        assert all(np.array_equal(a, b) for a, b in zip(o[3], out[0][3]))
    assert 0 < out[0][2][0].sum() <= out[0][2][1].sum() == K * 24


def test_per_state_hmc_moves_and_refusals():
    s = lj_setup(N=128, n_alch=4, seed=2)
    K, lambdas, temps = 2, np.array([1.0, 0.5]), np.array([300.0, 300.0])
    eng = lj_engine(s, K, lambdas, temps, 0.002, 3)
    eng.set_state_hmc_integrator(1, 0.001, 3)
    x0 = np.stack([s['x']] * K)
    eng.set_positions(x0); eng.set_velocities(np.zeros_like(x0))
    eng.set_replica_states(np.array([0, 1]))
    eng.propagate(SEED, IT)
    xg, vg = eng.get_positions(), eng.get_velocities()
    osys = oracle_system(s)
    for k, dt in ((0, 0.002), (1, 0.001)):
        check_replica(eng, k, x0[k], s['mass'], KB * 300.0, ho.lj(osys, lambdas[k]), dt, 3, xg, vg, s['box'])
    from openmmtools_b200._engine import EngineError
    eng.set_state_integrator(0, 0.002, 1.0, 3, 'V R O R V')   # a Langevin state among HMC states: refused at launch
    with pytest.raises(EngineError) as e:
        eng.propagate(SEED, IT)
    assert e.value.code == _lib.RX_ERR_UNSUPPORTED
    eng.set_pressures(np.full(2, 0.06), np.zeros(2))
    with pytest.raises(EngineError) as e:
        eng.set_hmc_integrator(0.002, 3)
    assert e.value.code == _lib.RX_ERR_UNSUPPORTED


def hmc_sampler(tmp, seed=11, K=6, **kw):
    fluid = testsystems.LennardJonesFluid(nparticles=128)
    ligand = list(range(4))
    asys = alchemy.AbsoluteAlchemicalFactory(disable_alchemical_dispersion_correction=True).create_alchemical_system(
        fluid.system, alchemy.AlchemicalRegion(alchemical_atoms=ligand))
    tstates = states.create_thermodynamic_state_protocol(
        asys, {'lambda_sterics': [1.0 - l / (K - 1) for l in range(K)]}, constants={'temperature': 300.0 * unit.kelvin},
        composable_states=alchemy.AlchemicalState.from_system(asys))
    sstate = states.SamplerState(fluid.positions, box_vectors=asys.getDefaultPeriodicBoxVectors())
    move = mcmc.SequenceMove([mcmc.MCDisplacementMove(displacement_sigma=0.05 * unit.nanometer, atom_subset=ligand),
                              mcmc.HMCMove(timestep=2.0 * unit.femtosecond, n_steps=5)])
    s = multistate.ReplicaExchangeSampler(mcmc_moves=move, number_of_iterations=6, seed=seed, **kw)
    storage = None if tmp is None else multistate.MultiStateReporter(os.path.join(str(tmp), 'run'), checkpoint_interval=2)
    s.create(tstates, [sstate], storage=storage)
    return s


def test_sampler_runs_hmc_fused_and_phase_by_phase_alike():
    a, b = hmc_sampler(None), hmc_sampler(None)
    a.run(3)
    b._compute_energies()
    b._engine.run_iterations(3, 'swap-all', b._seed, 1)
    for f in ('get_replica_states', 'get_energies', 'get_positions', 'get_velocities', 'get_hmc_statistics'):
        ra, rb = getattr(a._engine, f)(), getattr(b._engine, f)()
        assert all(np.array_equal(p, q) for p, q in zip(ra, rb)) if isinstance(ra, tuple) else np.array_equal(ra, rb), f
    acc, n = a._engine.get_hmc_statistics()
    assert list(n) == [3 * 5] * 6 and 0 < acc.sum() <= n.sum()


def test_stored_hmc_run_resumes_bit_for_bit(tmp_path):
    a = hmc_sampler(tmp_path / 'a')
    a.run(6)
    b = hmc_sampler(tmp_path / 'b')
    b.run(4)
    b._reporter.close()
    del b
    c = multistate.ReplicaExchangeSampler.from_storage(multistate.MultiStateReporter(os.path.join(str(tmp_path / 'b'), 'run')))
    assert c.iteration == 4
    assert isinstance(mcmc.split_move(c._mcmc_moves[0])[1], mcmc.HMCMove)
    c.run(2)
    assert np.array_equal(a._engine.get_positions(), c._engine.get_positions())


def test_move_apply_runs_one_replica():
    fluid = testsystems.LennardJonesFluid(nparticles=64)
    ts = states.ThermodynamicState(fluid.system, temperature=300.0 * unit.kelvin)
    ss = states.SamplerState(fluid.positions, box_vectors=fluid.system.getDefaultPeriodicBoxVectors())
    x0 = ss.positions.value_in_unit(unit.nanometer).copy()
    move = mcmc.HMCMove(timestep=2.0 * unit.femtosecond, n_steps=4)
    move.apply(ts, ss)
    assert not np.allclose(ss.positions.value_in_unit(unit.nanometer), x0)
    assert ss.kinetic_energy is not None


# ---- molecules (k_propagate_mol_hmc): alanine dipeptide with HBonds and without constraints, in vacuum and in OBC1 ---------
def aladip_system(constraints, implicit):
    a = testsystems.AlanineDipeptideVacuum(constraints=constraints)
    x = np.ascontiguousarray(a.positions.value_in_unit(unit.nanometer), np.float64)
    system = a.system
    if implicit:
        from implicit_helpers import obc
        system = obc(system, 'OBC1')
    return system, x


def oracle_molecule(system, implicit):
    if implicit:
        from oracle import implicit as oi
        return oi.Molecule(system)
    from oracle import oracle
    return oracle.Molecule(system)


@pytest.mark.parametrize('constraints', ['HBonds', None])
@pytest.mark.parametrize('implicit', [False, True])
def test_molecule_trials_match_oracle(constraints, implicit):
    system, x = aladip_system(constraints, implicit)
    temps = np.array([300.0, 450.0])
    K, n_steps, dt = 2, 5, 0.001
    e = gpu_engine(_lib.RX_SYSTEM_MOLECULE, K, K, system.n_particles)
    e.set_molecule(system, constraint_tolerance=1e-10)
    e.set_states(temps, np.ones(K))
    e.set_hmc_integrator(dt, n_steps)
    rng = np.random.default_rng(2)
    x0 = np.stack([x + rng.normal(0, 0.002, x.shape) for _ in range(K)])
    m = oracle_molecule(system, implicit)
    if constraints is not None:   # start on the constraints (the first trial may be rejected back to the start)
        x0 = np.stack([ho.shake(m.cons, m.mass, xk, xk, 1e-12) for xk in x0])
    e.set_positions(x0); e.set_velocities(np.zeros_like(x0))
    perm = np.array([1, 0])
    e.set_replica_states(perm)
    e.propagate(SEED, IT)
    xg, vg = e.get_positions(), e.get_velocities()
    cons = m.cons if constraints is not None else None
    decisions = []
    for k in range(K):
        decisions += [t[2] for t in check_replica(e, k, x0[k], m.mass, KB * temps[perm[k]], ho.molecule(m), dt, n_steps, xg, vg,
                                                  tol_x=2e-6, tol_v=2e-3, cons=cons)]
    assert sum(decisions) > 0
    if cons is not None:
        i, j = cons[:, 0].astype(int), cons[:, 1].astype(int)
        assert np.abs(np.linalg.norm(xg[:, i] - xg[:, j], axis=-1) - cons[:, 2]).max() < 1e-10
    e.close()


def test_molecule_constraints_hold_over_a_long_launch():
    system, x = aladip_system('HBonds', False)
    from oracle import oracle
    m = oracle.Molecule(system)
    K = 4
    e = gpu_engine(_lib.RX_SYSTEM_MOLECULE, K, K, system.n_particles)
    e.set_molecule(system, constraint_tolerance=1e-10)
    e.set_states(np.linspace(300.0, 500.0, K), np.ones(K))
    e.set_hmc_integrator(0.002, 40)   # 40 trials of 40 steps
    x0 = ho.shake(m.cons, m.mass, x, x, 1e-12)
    e.set_positions(np.stack([x0] * K)); e.set_velocities(np.zeros((K,) + x.shape))
    e.propagate(SEED, IT)
    xg = e.get_positions()
    i, j = m.cons[:, 0].astype(int), m.cons[:, 1].astype(int)
    assert np.abs(np.linalg.norm(xg[:, i] - xg[:, j], axis=-1) - m.cons[:, 2]).max() < 1e-10
    acc, n = e.get_hmc_statistics()
    assert list(n) == [40] * K and 0 < acc.sum() < n.sum()
    e.close()


def test_molecule_move_apply():
    a = testsystems.AlanineDipeptideVacuum()
    ts = states.ThermodynamicState(a.system, temperature=298.0 * unit.kelvin)
    ss = states.SamplerState(a.positions)
    x0 = ss.positions.value_in_unit(unit.nanometer).copy()
    mcmc.HMCMove(timestep=0.5 * unit.femtosecond, n_steps=10).apply(ts, ss)
    assert not np.allclose(ss.positions.value_in_unit(unit.nanometer), x0)


TWO_RANK_WORKER = r'''
import os, sys
sys.path.insert(0, %(root)r)
sys.path.insert(0, os.path.join(%(root)r, 'tests'))
import numpy as np
import torch.distributed as dist
dist.init_process_group('gloo')
from test_gpu_hmc import hmc_sampler
from openmmtools_b200._dist import TorchCommunicator
s = hmc_sampler(None, seed=321, communicator=TorchCommunicator())
s.run(3)
acc, n = s._engine.get_hmc_statistics()
np.savez(%(out)r + '_%%d.npz' %% dist.get_rank(), perm=s._replica_thermodynamic_states, u=s._energy_thermodynamic_states,
         x=s._engine.get_positions(), k0=s._engine.k0, acc=acc, n=n)
dist.barrier()
'''


def test_two_gpus_reproduce_single_gpu_with_hmc(tmp_path):
    from test_multi_gpu_mc import _two_devices
    if not _two_devices():
        pytest.skip('needs 2 GPUs')
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    s = hmc_sampler(None, seed=321)
    s.run(3)
    u1, p1, x1 = s._energy_thermodynamic_states.copy(), s._replica_thermodynamic_states.copy(), s._engine.get_positions()
    acc1, n1 = s._engine.get_hmc_statistics()
    script = tmp_path / 'g.py'
    out = str(tmp_path / 'res')
    script.write_text(TWO_RANK_WORKER % {'root': root, 'out': out})
    r = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2',
                        '--master-addr', '127.0.0.1', '--master-port', '29573', str(script)],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    for rank in range(2):
        d = np.load(out + '_%d.npz' % rank)
        assert np.array_equal(d['perm'], p1) and np.array_equal(d['u'], u1)
        k0 = int(d['k0'])
        kn = d['x'].shape[0]
        assert np.array_equal(d['x'], x1[k0:k0 + kn])
        assert np.array_equal(d['acc'][k0:k0 + kn], acc1[k0:k0 + kn]) and np.array_equal(d['n'][k0:k0 + kn], n1[k0:k0 + kn])
