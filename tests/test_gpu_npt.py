"""Constant pressure on the GPU: the energy matrix with per-replica boxes and pV, the Monte Carlo barostat inside
k_propagate (its decisions on the device's own uniforms, its independence of the launch plan, the ideal gas's volume law,
the cutoff limit), the NaN restart, and stored ReplicaExchangeSampler runs with a pressure ladder."""
import os
import numpy as np
import pytest
from helpers import lj_setup, oracle_system, gpu_engine, KB, philox4x32_10, device_noise, min_image, wrap
from test_npt_host import BAR, alchemical_fluid
from oracle import npt as onpt

pytestmark = pytest.mark.gpu
RTOL = 1e-10


def npt_engine(s, K, M, lambdas, temps, pressures, disp, eps=None, alch=None):
    e = gpu_engine(1, K, M, s['N'], box=tuple(s['box']), r_cutoff=s['rc'], r_switch=s['rs'], use_switch=True)
    e.set_particles(s['sigma'], s['eps'] if eps is None else eps, s['mass'], s['alch'] if alch is None else alch)
    e.set_states(temps, lambdas)
    e.set_pressures(pressures, disp)
    return e


def barostat_uniforms(seed, iteration, replica, attempt):
    key = (seed & 0xFFFFFFFF, ((seed >> 32) ^ (iteration >> 32)) & 0xFFFFFFFF)
    r = philox4x32_10(np.array([attempt, 0xA0000000, replica, iteration & 0xFFFFFFFF], np.uint32), key)
    return (float(r[0]) + 0.5) * 2.0 ** -32, (float(r[1]) + 0.5) * 2.0 ** -32


class cluster_width:
    """RX_CLUSTER for the launches inside the block (the planner's override)."""

    def __init__(self, cl):
        self.cl = cl

    def __enter__(self):
        self.old = os.environ.get('RX_CLUSTER')
        if self.cl is None:
            os.environ.pop('RX_CLUSTER', None)
        else:
            os.environ['RX_CLUSTER'] = str(self.cl)

    def __exit__(self, *a):
        if self.old is None:
            os.environ.pop('RX_CLUSTER', None)
        else:
            os.environ['RX_CLUSTER'] = self.old


@pytest.mark.parametrize('with_dispersion', [True, False])
def test_energy_matrix_per_replica_boxes_and_pv(with_dispersion):
    N, K, M = 512, 6, 9
    s = lj_setup(N=N, n_alch=10, seed=5)
    scales = np.linspace(0.9, 1.15, K)
    xs = np.stack([(s['x'] * f).astype(np.float32).astype(np.float64) for f in scales])
    boxes = np.outer(scales, s['box'])
    lambdas, temps = np.linspace(1.0, 0.0, M), np.linspace(300.0, 330.0, M)
    pressures = np.linspace(1.0, 80.0, M) * BAR
    disp = np.linspace(-40.0, -10.0, M) if with_dispersion else np.zeros(M)
    e = npt_engine(s, K, M, lambdas, temps, pressures, disp)
    e.set_positions(xs)
    e.set_boxes(boxes)
    assert np.array_equal(e.get_boxes(), boxes)
    u = e.compute_energies()
    # unsampled states: their own temperatures, lambdas, pressures and coefficients, the same per-replica boxes
    ul, ut, up, uc = np.array([0.37, 0.9]), np.array([290.0, 350.0]), np.array([5.0, 120.0]) * BAR, disp[:2] * 1.5
    uu = e.compute_energies_at(ut, ul, pressure=up, dispersion=uc)
    e.close()
    osys = oracle_system(s)
    for got, lam, T, p, c in ((u, lambdas, temps, pressures, disp), (uu, ul, ut, up, uc)):
        ref = onpt.energy_matrix(osys, xs, boxes, lam, 1.0 / (KB * T), p, c)
        assert (np.abs(got - ref) / np.maximum(1.0, np.abs(ref))).max() <= RTOL
    for k in range(K):     # and through the NVT oracle at each box, pV and c / V added by hand
        V = np.prod(boxes[k])
        ref = oracle_system(dict(s, box=boxes[k])).energy_row(xs[k], lambdas, 1.0 / (KB * temps), disp / V + pressures * V)
        assert (np.abs(u[k] - ref) / np.maximum(1.0, np.abs(ref))).max() <= RTOL


@pytest.mark.parametrize('N,cl', [(512, 1), (512, 4), (2048, None)])
def test_barostat_decisions_on_device_uniforms(N, cl):
    """Ideal gas (epsilon = 0, so dU = 0 exactly): 75 steps are three attempts, whose outcome is a function of the
    device's Philox uniforms alone; the boxes and the barostat state follow the host restatement."""
    K, seed, it = 8, 99, 3
    s = lj_setup(N=N, n_alch=0, seed=2)
    kT = KB * 300.0
    V0 = np.prod(s['box'])
    p = (N + 1) * kT / V0 * 1.3      # above the box's ideal-gas pressure: compressions are favoured
    e = npt_engine(s, K, 1, [1.0], [300.0], [p], [0.0], eps=np.zeros(N))
    e.set_positions(np.stack([s['x']] * K))
    e.randomize_velocities(seed)
    e.set_integrator(0.002, 1.0, 75)
    st0 = e.get_barostat()
    st0['volume_scale'] = st0['volume_scale'] * 5.0     # large moves, so that both outcomes occur
    e.set_barostat(st0)
    with cluster_width(cl):
        e.propagate(seed, it)
    boxes, bst = e.get_boxes(), e.get_barostat()
    e.close()
    outcomes = []
    osys = oracle_system(dict(s, eps=np.zeros(N)))
    for k in range(K):
        box, x = np.array(s['box']), s['x'].copy()
        st = onpt.barostat_state(st0['volume_scale'][k])
        for a in range(3):
            u1, u2 = barostat_uniforms(seed, it, k, a)
            outcomes.append(onpt.barostat_step(osys, x, box, st, u1, u2, 1.0, kT, p, 0.0, 2 * s['rc'])[0])
        assert np.allclose(boxes[k], box, rtol=1e-13, atol=0), k
        assert bst['n_attempted'][k] == st.n_attempted and bst['n_accepted'][k] == st.n_accepted
        assert bst['volume_scale'][k] == pytest.approx(st.volume_scale, rel=1e-15) and bst['step'][k] == 0
    assert 1 in outcomes and 0 in outcomes


@pytest.mark.parametrize('N,cl', [(512, 1), (512, 4), (2048, None)])
def test_interacting_fluid_steps_and_barostat_match_oracle(monkeypatch, N, cl):
    """75 steps (three attempts) of the alchemical LJ fluid with the device's Philox noise and uniforms restated on the
    host: the oracle (f64) takes the same accept/reject decisions, and positions, velocities, boxes and the potential
    agree within the tolerances of the NVT step tests."""
    K = 4
    s = lj_setup(N=N, n_alch=6, seed=11)
    if cl is not None:
        monkeypatch.setenv('RX_CLUSTER', str(cl))
    lambdas, temps = np.array([1.0, 0.6, 0.3, 0.0]), np.array([300.0, 310.0, 320.0, 330.0])
    pressures, disp = np.array([30.0, 45.0, 60.0, 80.0]) * BAR, np.array([-30.0, -25.0, -20.0, -15.0])
    dt, gamma, n_steps, seed, it = 0.002, 10.0, 75, 0x1234567890ABCDEF, 7
    e = npt_engine(s, K, K, lambdas, temps, pressures, disp)
    e.set_integrator(dt, gamma, n_steps, 'V R O R V')
    x0 = np.stack([s['x']] * K)
    v0 = np.random.default_rng(2).normal(scale=0.25, size=(K, N, 3)).astype(np.float32).astype(np.float64)
    e.set_positions(x0); e.set_velocities(v0)
    st0 = e.get_barostat()
    st0['volume_scale'] = st0['volume_scale'] * 3.0
    e.set_barostat(st0)
    e.propagate(seed, it)
    xg, vg, bg, bst = e.get_positions(), e.get_velocities(), e.get_boxes(), e.get_barostat()
    pot = e.get_replica_energies()[0]
    e.close()
    osys = oracle_system(s)
    accepted = 0
    for k in range(K):
        x, v, box = x0[k].copy(), v0[k].copy(), np.array(s['box'], np.float64)
        st = onpt.barostat_state(st0['volume_scale'][k])
        uni = np.array([barostat_uniforms(seed, it, k, a) for a in range(3)]).ravel()
        dec, U = onpt.langevin(osys, x, v, device_noise(seed, it, k, N, n_steps), box, st, uni, lambdas[k], KB * temps[k], dt,
                               gamma, n_steps, pressures[k], disp[k], 2 * s['rc'])
        assert len(dec) == 3 and bst['n_attempted'][k] == 3 and bst['n_accepted'][k] == dec.count(1), (k, dec, bst)
        accepted += dec.count(1)
        assert np.allclose(bg[k], box, rtol=1e-12, atol=0), (k, bg[k], box)
        assert np.abs(min_image(xg[k] - wrap(x, box), box)).max() < 2e-5, k
        assert np.abs(vg[k] - v).max() < 2e-4, k
        assert abs(pot[k] - U) < 1e-3 * max(1.0, abs(U)), (pot[k], U)
    assert accepted > 0


def fluid_run(cl, N=512, K=4, launches=2, n_steps=100):
    s = lj_setup(N=N, n_alch=10, seed=11)
    M = K
    e = npt_engine(s, K, M, np.linspace(1.0, 0.0, M), np.full(M, 300.0), np.linspace(20.0, 80.0, M) * BAR,
                   np.full(M, -25.0))
    e.set_positions(np.stack([s['x']] * K))
    e.randomize_velocities(3)
    e.set_integrator(0.002, 5.0, n_steps)
    with cluster_width(cl):
        for it in range(launches):
            e.propagate(17, it)
    out = (e.get_positions(), e.get_velocities(), e.get_boxes(), e.get_barostat(), e.get_replica_energies()[0])
    e.close()
    return out


def test_trajectory_boxes_and_barostat_do_not_depend_on_the_cluster_width():
    ref = fluid_run(1)
    assert not np.array_equal(ref[2], np.tile(lj_setup(N=512, n_alch=10, seed=11)['box'], (4, 1))), 'no move accepted'
    for cl in (2, 4):
        got = fluid_run(cl)
        for a, b in zip(ref[:3], got[:3]):
            assert np.array_equal(a, b), cl
        for f in ref[3]:
            assert np.array_equal(ref[3][f], got[3][f]), (cl, f)


def test_compact_plan_trajectory_independent_of_cluster_width():
    a = fluid_run(2, N=2048, K=2, launches=1, n_steps=50)
    b = fluid_run(4, N=2048, K=2, launches=1, n_steps=50)
    for x, y in zip(a[:3], b[:3]):
        assert np.array_equal(x, y)


def test_ideal_gas_volume_distribution():
    """epsilon = 0, 512 atoms, 64 replicas: after equilibration V has mean (N+1) kT/p and variance (N+1) (kT/p)^2."""
    N, K = 512, 64
    s = lj_setup(N=N, n_alch=0, seed=4)
    kT = KB * 300.0
    p = (N + 1) * kT / np.prod(s['box'])       # the box is the mean volume: edges ~ 7 nm, far above 2 rc ~ 2 nm
    e = npt_engine(s, K, 1, [1.0], [300.0], [p], [0.0], eps=np.zeros(N))
    e.set_positions(np.stack([s['x']] * K))
    e.randomize_velocities(1)
    e.set_integrator(0.004, 5.0, 500)          # 20 attempts per launch
    vols = []
    for it in range(60):
        e.propagate(5, it)
        if it >= 10:
            vols.append(np.prod(e.get_boxes(), axis=1))
    e.close()
    v = np.array(vols).T                       # [K, samples]
    Vm, Vv = (N + 1) * kT / p, (N + 1) * (kT / p) ** 2
    means, variances = v.mean(axis=1), v.var(axis=1)
    se_m, se_v = means.std(ddof=1) / np.sqrt(K), variances.std(ddof=1) / np.sqrt(K)
    assert abs(means.mean() - Vm) < 4 * se_m, (means.mean(), Vm, se_m)
    assert abs(variances.mean() - Vv) < 4 * se_v, (variances.mean(), Vv, se_v)


def test_box_never_below_twice_the_cutoff():
    N, K = 256, 16
    s = lj_setup(N=N, n_alch=0, seed=6)
    kT = KB * 300.0
    p = (N + 1) * kT / (1.6 * s['rc']) ** 3    # the ideal-gas volume lies below the limit
    e = npt_engine(s, K, 1, [1.0], [300.0], [p], [0.0], eps=np.zeros(N))
    e.set_positions(np.stack([s['x']] * K))
    e.randomize_velocities(1)
    e.set_integrator(0.004, 5.0, 500)
    for it in range(40):
        e.propagate(8, it)
        assert e.get_boxes().min() >= 2 * s['rc']
    assert e.get_boxes().min() < 2.1 * s['rc']    # the run did reach the limit
    e.close()


def nan_engine():
    N, K = 512, 4
    s = lj_setup(N=N, n_alch=10, seed=11)
    e = npt_engine(s, K, K, np.linspace(1.0, 0.0, K), np.full(K, 300.0), np.full(K, 40.0 * BAR), np.full(K, -25.0))
    e.set_positions(np.stack([s['x']] * K))
    e.randomize_velocities(3)
    e.set_integrator(0.002, 5.0, 100)
    e.propagate(17, 0)
    bad = e.get_positions()
    bad[2, 5] = np.inf                     # replica 2 starts the next propagation from a non-finite position
    e.set_positions(bad)
    return e


def test_nan_restart_restores_box_and_barostat():
    """Only the failed replica runs again, from the snapshot of its positions, velocities, box and barostat state: its
    result equals a plain propagation with the retry's seed from that same start."""
    from openmmtools_b200 import _lib
    from openmmtools_b200._engine import EngineError
    e = nan_engine()
    snap_box = e.get_boxes()
    with pytest.raises(EngineError) as err:
        e.propagate(17, 1)
    assert err.value.code == _lib.RX_ERR_NAN and list(err.value.nan_flags) == [0, 0, 1, 0]
    after = (e.get_positions(), e.get_boxes(), e.get_barostat())
    assert not np.array_equal(after[1][2], snap_box[2]), 'the failed run left the box as it was: no restore is shown'
    with pytest.raises(EngineError):
        e.propagate_retry(18, 1)
    retry = (e.get_positions(), e.get_boxes(), e.get_barostat())
    e.close()
    ref_e = nan_engine()
    with pytest.raises(EngineError):
        ref_e.propagate(18, 1)
    ref = (ref_e.get_positions(), ref_e.get_boxes(), ref_e.get_barostat())
    ref_e.close()
    for k in (0, 1, 3):                    # the replicas that came through keep their result
        assert np.array_equal(retry[0][k], after[0][k]) and np.array_equal(retry[1][k], after[1][k])
        assert all(retry[2][f][k] == after[2][f][k] for f in retry[2])
    assert np.array_equal(retry[0][2], ref[0][2], equal_nan=True) and np.array_equal(retry[1][2], ref[1][2])
    assert all(retry[2][f][2] == ref[2][f][2] for f in retry[2])


def test_minimize_at_per_replica_boxes():
    """FIRE descent of every replica at its own box: the oracle's forces at the returned positions and that box meet the
    tolerance, the positions are wrapped into the replica's box, and the boxes are left as they were."""
    N, K = 512, 4
    s = lj_setup(N=N, n_alch=10, seed=8)
    scales = np.array([0.85, 0.95, 1.05, 1.2])
    boxes = np.outer(scales, s['box'])
    xs = np.stack([(s['x'] * f).astype(np.float32).astype(np.float64) for f in scales])
    lambdas = np.array([1.0, 0.7, 0.4, 0.0])
    rms0 = [np.sqrt((oracle_system(dict(s, box=boxes[k])).energy(xs[k], lambdas[k], forces=True)[2] ** 2).mean())
            for k in range(K)]
    tol = 0.1 * min(rms0)       # every replica has to descend
    e = npt_engine(s, K, K, lambdas, np.full(K, 300.0), np.full(K, 40.0 * BAR), np.full(K, -25.0))
    e.set_positions(xs)
    e.set_boxes(boxes)
    rms, its = e.minimize(tol)
    x = e.get_positions()
    assert np.array_equal(e.get_boxes(), boxes)
    e.close()
    for k in range(K):
        assert its[k] > 0 and rms[k] <= tol
        assert (x[k] >= 0).all() and (x[k] < boxes[k]).all()
        f = oracle_system(dict(s, box=boxes[k])).energy(x[k], lambdas[k], forces=True)[2]
        assert np.sqrt((f ** 2).mean()) <= 1.05 * tol, (k, np.sqrt((f ** 2).mean()))


def test_reduced_potential_of_an_npt_state():
    """ThermodynamicState.reduced_potential on a SamplerState with its own box: beta (U + c / V + p V) (states.py:1909-1917)."""
    from openmmtools_b200 import unit, states, alchemy, _backend
    from oracle import oracle
    asys = alchemical_fluid(N=128, dispersion=True)
    from openmmtools_b200 import testsystems
    x = np.asarray(testsystems.LennardJonesFluid(nparticles=128).positions.value_in_unit(unit.nanometer), np.float64)
    ts = states.create_thermodynamic_state_protocol(asys, {'lambda_sterics': [0.4], 'pressure': [35.0] * unit.bar},
                                                    constants={'temperature': 310.0 * unit.kelvin},
                                                    composable_states=alchemy.AlchemicalState.from_system(asys))[0]
    f = 1.07
    edges = np.diag(asys.box_vectors) * f
    ss = states.SamplerState(x * f, box_vectors=unit.Quantity(np.diag(edges), unit.nanometer))
    u = ts.reduced_potential(ss)
    osys = oracle.LJSystem(asys.sigma, asys.epsilon, asys.masses, asys.alchemical_mask(), tuple(edges), asys.cutoff,
                           asys.switching_distance)
    U = osys.energy((x * f).astype(np.float32).astype(np.float64), 0.4)[0]
    V = np.prod(edges)
    c = _backend.pressure_tables([ts])[1][0]
    ref = (U + c / V + 35.0 * BAR * V) / (KB * 310.0)
    assert u == pytest.approx(ref, rel=1e-9)


def npt_sampler(path, K=4, N=128, iterations=4):
    from openmmtools_b200 import unit, states, alchemy, mcmc, multistate
    from openmmtools_b200.multistate import MultiStateReporter
    asys = alchemical_fluid(N=N, dispersion=True)
    from openmmtools_b200 import testsystems
    fluid = testsystems.LennardJonesFluid(nparticles=N)
    tstates = states.create_thermodynamic_state_protocol(
        asys, {'pressure': list(np.linspace(20.0, 60.0, K)) * unit.bar}, constants={'temperature': 300.0 * unit.kelvin,
                                                                                 'lambda_sterics': 0.5},
        composable_states=alchemy.AlchemicalState.from_system(asys))
    unsampled = states.create_thermodynamic_state_protocol(
        asys, {'pressure': [50.0] * unit.bar}, constants={'temperature': 320.0 * unit.kelvin, 'lambda_sterics': 1.0},
        composable_states=alchemy.AlchemicalState.from_system(asys))
    sstate = states.SamplerState(fluid.positions, box_vectors=asys.getDefaultPeriodicBoxVectors())
    move = mcmc.LangevinSplittingDynamicsMove(timestep=2.0 * unit.femtosecond, n_steps=100)
    smp = multistate.ReplicaExchangeSampler(mcmc_moves=move, number_of_iterations=iterations, seed=21)
    smp.create(tstates, [sstate], storage=MultiStateReporter(path, checkpoint_interval=2),
               unsampled_thermodynamic_states=unsampled)
    return smp, asys, tstates + unsampled


def test_sampler_run_stores_boxes_energies_and_resumes(tmp_path):
    from openmmtools_b200 import multistate, _backend, unit
    from openmmtools_b200.multistate import MultiStateReporter
    a, asys, tstates = npt_sampler(str(tmp_path / 'a.store'))
    a.run()
    xa = np.stack([st._positions for st in a.sampler_states])
    ba = np.stack([st._box_vectors for st in a.sampler_states])
    assert len({tuple(np.diag(b)) for b in ba}) > 1, 'every replica kept the initial box'
    r = MultiStateReporter(str(tmp_path / 'a.store'), open_mode='r')
    stored = r.read_sampler_states(4)
    assert np.array_equal(np.stack([s._box_vectors for s in stored]), ba)
    ua, _, uu = r.read_energies(4)
    assert np.array_equal(r.read_volumes(4), np.prod(np.einsum('kii->ki', ba), axis=1))
    assert r.read_volumes().shape == (5, len(xa))
    p, c = _backend.pressure_tables(tstates)
    lams = np.array([t.lambda_sterics for t in tstates])
    betas = np.array([1.0 / (KB * t.temperature.value_in_unit(unit.kelvin)) for t in tstates])
    s = dict(sigma=asys.sigma, eps=asys.epsilon, mass=asys.masses, alch=asys.alchemical_mask(), box=np.diag(ba[0]),
             rc=asys.cutoff, rs=asys.switching_distance)
    ref = onpt.energy_matrix(oracle_system(s), xa, np.einsum('kii->ki', ba), lams, betas, p, c)
    M = len(xa)
    for got, want in ((ua, ref[:, :M]), (uu, ref[:, M:])):
        assert (np.abs(got - want) / np.maximum(1.0, np.abs(want))).max() <= RTOL
    # the device loop gives the same bits as the host loop
    d, _, _ = npt_sampler(str(tmp_path / 'd.store'))
    d._compute_energies()
    d._engine.run_iterations(4, 'swap-all', d._seed, 1)
    assert np.array_equal(d._engine.get_positions(), a._engine.get_positions())
    assert np.array_equal(d._engine.get_boxes(), a._engine.get_boxes())
    # interrupted after 3 iterations (last checkpoint 2), resumed from storage: the same bits as the uninterrupted run
    b, _, _ = npt_sampler(str(tmp_path / 'b.store'))
    b.run(3)
    del b
    c2 = multistate.ReplicaExchangeSampler.from_storage(str(tmp_path / 'b.store'))
    assert c2.iteration == 2
    c2.run()
    assert np.array_equal(np.stack([st._positions for st in c2.sampler_states]), xa)
    assert np.array_equal(np.stack([st._box_vectors for st in c2.sampler_states]), ba)
    assert np.array_equal(c2._energy_thermodynamic_states, a._energy_thermodynamic_states)
