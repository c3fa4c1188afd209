"""The anisotropic Monte Carlo barostat on the GPU: its decisions, axes, positions and boxes against the oracle on the
device's own Philox draws (every launch layout, three axis masks, replicas in other states), unscaled edges that never
move, per-axis step-size adaptation, independence of the cluster width, the z-only ideal gas's volume law, the cutoff
limit on the scaled edge, the NaN restart, stored / fused / resumed ReplicaExchangeSampler runs, the reduced potential
of an anisotropic state and two ranks."""
import os
import subprocess
import sys
import numpy as np
import pytest
from helpers import lj_setup, oracle_system, gpu_engine, KB, philox4x32_10, device_noise, min_image, wrap
from test_npt_host import BAR, alchemical_fluid
from test_gpu_npt import cluster_width
from oracle import npt_aniso

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 0x1234567890ABCDEF
MASKS = {'xyz': 7, 'z': 4, 'xy': 3}


def draw(seed, iteration, replica, attempt, mask):
    """(axis, u1, u2) of an anisotropic attempt: the isotropic attempt's Philox draw, its third word picking the
    floor(rr.z n / 2^32)-th of the n scaled axes."""
    key = (seed & 0xFFFFFFFF, ((seed >> 32) ^ (iteration >> 32)) & 0xFFFFFFFF)
    r = philox4x32_10(np.array([attempt, 0xA0000000, replica, iteration & 0xFFFFFFFF], np.uint32), key)
    axes = [d for d in range(3) if mask >> d & 1]
    return axes[(int(r[2]) * len(axes)) >> 32], (float(r[0]) + 0.5) * 2.0 ** -32, (float(r[1]) + 0.5) * 2.0 ** -32


def aniso_engine(s, K, M, lambdas, temps, pressures, disp, mask, eps=None):
    e = gpu_engine(1, K, M, s['N'], box=tuple(s['box']), r_cutoff=s['rc'], r_switch=s['rs'], use_switch=True)
    e.set_particles(s['sigma'], s['eps'] if eps is None else eps, s['mass'], s['alch'])
    e.set_states(temps, lambdas)
    e.set_pressures(pressures, disp)
    e.set_anisotropic_barostat([bool(mask >> d & 1) for d in range(3)])
    return e


def oracle_state(dev, k):
    st = npt_aniso.barostat_state(dev['volume_scale'][k], int(dev['scale_mask'][k]), int(dev['step'][k]))
    st.n_attempted[:] = [int(v) for v in dev['n_attempted'][k]]
    st.n_accepted[:] = [int(v) for v in dev['n_accepted'][k]]
    return st


def assert_same_state(dev, k, st):
    assert list(dev['n_attempted'][k]) == list(st.n_attempted) and list(dev['n_accepted'][k]) == list(st.n_accepted), k
    assert dev['step'][k] == st.step and dev['scale_mask'][k] == st.scale_mask
    assert np.allclose(dev['volume_scale'][k], list(st.volume_scale), rtol=1e-15, atol=0), k


def oracle_launch(osys, x, v, box, st, seed, it, k, n_steps, lam, T, p, c, dt, gamma):
    """One launch of replica k on the oracle with the device's noise and draws; returns (decisions, axes, potential)."""
    N = len(x)
    n_max = n_steps // 25 + 1
    d = [draw(seed, it, k, a, st.scale_mask) for a in range(n_max)]
    axes, uni = [a for a, _, _ in d], np.array([(u1, u2) for _, u1, u2 in d]).ravel()
    dec, U = npt_aniso.langevin(osys, x, v, device_noise(seed, it, k, N, n_steps), box, st, axes, uni, lam, KB * T, dt,
                                 gamma, n_steps, p, c, 2 * osys.p.r_cutoff)
    return dec, axes[:len(dec)], U


# ---- 1. the oracle on the device's draws ---------------------------------------------------------------------------------
@pytest.mark.parametrize('mask', list(MASKS), ids=list(MASKS))
@pytest.mark.parametrize('N,cl', [(512, 1), (512, 4), (2048, None)], ids=['cl1', 'cl4', 'compact'])
def test_decisions_axes_positions_and_boxes_match_oracle(N, cl, mask):
    """75 steps (three attempts) of the alchemical fluid with replicas in states other than their own index: the
    oracle (f64) on the device's noise, axes and uniforms takes the same decisions on the same axes, the boxes and the
    per-axis state agree, and the f32 positions, velocities and potential stay within the f32 dynamics' drift."""
    K, m = 4, MASKS[mask]
    s = lj_setup(N=N, n_alch=6, seed=11)
    lambdas, temps = np.array([1.0, 0.6, 0.3, 0.0]), np.array([300.0, 310.0, 320.0, 330.0])
    pressures, disp = np.array([30.0, 45.0, 60.0, 80.0]) * BAR, np.array([-30.0, -25.0, -20.0, -15.0])
    perm = np.array([2, 0, 3, 1])
    dt, gamma, n_steps, it = 0.002, 10.0, 75, 7
    e = aniso_engine(s, K, K, lambdas, temps, pressures, disp, m)
    e.set_integrator(dt, gamma, n_steps, 'V R O R V')
    e.set_replica_states(perm)
    x0 = np.stack([s['x']] * K)
    v0 = np.random.default_rng(2).normal(scale=0.25, size=(K, N, 3)).astype(np.float32).astype(np.float64)
    e.set_positions(x0); e.set_velocities(v0)
    st0 = e.get_barostat_anisotropic()
    st0['volume_scale'] = st0['volume_scale'] * np.array([3.0, 2.0, 4.0])
    e.set_barostat_anisotropic(st0)
    with cluster_width(cl):
        e.propagate(SEED, it)
    xg, vg, bg, dev = e.get_positions(), e.get_velocities(), e.get_boxes(), e.get_barostat_anisotropic()
    pot = e.get_replica_energies()[0]
    e.close()
    osys = oracle_system(s)
    decisions, seen = [], set()
    for k in range(K):
        l = perm[k]
        x, v, box, st = x0[k].copy(), v0[k].copy(), np.array(s['box'], np.float64), oracle_state(st0, k)
        dec, axes, U = oracle_launch(osys, x, v, box, st, SEED, it, k, n_steps, lambdas[l], temps[l], pressures[l], disp[l],
                                     dt, gamma)
        assert len(dec) == 3 and all(m >> a & 1 for a in axes)
        decisions += dec
        seen |= set(axes)
        assert_same_state(dev, k, st)
        assert np.allclose(bg[k], box, rtol=1e-12, atol=0), (k, bg[k], box)
        assert np.abs(min_image(xg[k] - wrap(x, box), box)).max() < 3e-5, k
        assert np.abs(vg[k] - v).max() < 2e-4, k
        assert abs(pot[k] - U) < 1e-3 * max(1.0, abs(U)), (pot[k], U)
    assert 1 in decisions, decisions
    assert len(seen) > 1 or m == 4, seen


# ---- 2. unscaled edges ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('mask', ['z', 'xy'])
def test_unscaled_edges_never_move(mask):
    """2000 steps (80 attempts) in one launch: the unscaled edges are the start's bits, the scaled ones moved."""
    N, K, m = 512, 8, MASKS[mask]
    s = lj_setup(N=N, n_alch=10, seed=11)
    e = aniso_engine(s, K, K, np.linspace(1.0, 0.0, K), np.full(K, 300.0), np.linspace(20.0, 80.0, K) * BAR,
                     np.full(K, -25.0), m)
    e.set_positions(np.stack([s['x']] * K))
    e.randomize_velocities(3)
    e.set_integrator(0.002, 5.0, 2000)
    fresh = e.get_barostat_anisotropic()
    e.propagate(17, 0)
    b = e.get_boxes()
    dev = e.get_barostat_anisotropic()
    e.close()
    for d in range(3):
        if m >> d & 1:
            assert not np.array_equal(b[:, d], np.full(K, s['box'][d])), d
        else:
            assert np.array_equal(b[:, d], np.full(K, s['box'][d])), d
            for f in ('volume_scale', 'n_attempted', 'n_accepted'):
                assert np.array_equal(dev[f][:, d], fresh[f][:, d]), (d, f)


# ---- 3. per-axis adaptation ----------------------------------------------------------------------------------------------
def test_per_axis_adaptation_at_the_tenth_attempt():
    """Every axis of every replica is one attempt short of ten; one attempt (25 steps) reaches the tenth on the drawn
    axis only: 0 of 9 accepted shrinks its scale by 1.1, 9 of 9 grows it by 1.1, 9 of 9 from 0.29 V stops at the cap
    0.3 V, 5 of 9 keeps it and its counters; the other two axes keep their records.  Ideal gas, so that the decisions
    follow the uniforms alone; the oracle restates every record."""
    N, K = 512, 12
    s = lj_setup(N=N, n_alch=0, seed=4)
    V0 = float(np.prod(s['box']))
    p = (N + 1) * KB * 300.0 / V0
    e = aniso_engine(s, K, 1, [1.0], [300.0], [p], [0.0], 7, eps=np.zeros(N))
    e.set_positions(np.stack([s['x']] * K))
    e.randomize_velocities(1)
    e.set_integrator(0.002, 5.0, 25)
    kinds = [(0.05, 0), (0.05, 9), (0.29, 9), (0.05, 5)] * 3
    st0 = e.get_barostat_anisotropic()
    st0['volume_scale'] = np.array([[vs * V0] * 3 for vs, _ in kinds])
    st0['n_attempted'] = np.full((K, 3), 9)
    st0['n_accepted'] = np.array([[acc] * 3 for _, acc in kinds])
    e.set_barostat_anisotropic(st0)
    e.propagate(SEED, 5)
    dev, boxes = e.get_barostat_anisotropic(), e.get_boxes()
    e.close()
    osys = oracle_system(dict(s, eps=np.zeros(N)))
    axes = set()
    for k, (vs, acc) in enumerate(kinds):
        axis, u1, u2 = draw(SEED, 5, k, 0, 7)
        axes.add(axis)
        st = oracle_state(st0, k)
        x, box = s['x'].copy(), np.array(s['box'], np.float64)
        npt_aniso.barostat_step(osys, x, box, st, axis, u1, u2, 1.0, KB * 300.0, p, 0.0, 2 * s['rc'])
        assert np.allclose(boxes[k], box, rtol=1e-13, atol=0)
        st.step = 0
        assert_same_state(dev, k, st)
        want = {0: vs * V0 / 1.1, 9: vs * V0 * 1.1 if vs < 0.29 else 0.3 * V0, 5: vs * V0}[acc]
        assert dev['volume_scale'][k, axis] == pytest.approx(want, rel=1e-15), (k, axis)
        assert dev['n_attempted'][k, axis] == (10 if acc == 5 else 0)
        for d in set(range(3)) - {axis}:
            assert dev['volume_scale'][k, d] == vs * V0 and dev['n_attempted'][k, d] == 9 and dev['n_accepted'][k, d] == acc
    assert len(axes) > 1


# ---- 4. cluster width ----------------------------------------------------------------------------------------------------
def aniso_run(cl, mask, N=2048, K=4, n_steps=100):
    s = lj_setup(N=N, n_alch=10, seed=11)
    e = aniso_engine(s, K, K, np.linspace(1.0, 0.0, K), np.full(K, 300.0), np.linspace(20.0, 80.0, K) * BAR,
                     np.full(K, -25.0), mask)
    e.set_positions(np.stack([s['x']] * K))
    e.randomize_velocities(3)
    e.set_integrator(0.002, 5.0, n_steps)
    with cluster_width(cl):
        e.propagate(17, 0)
    out = (e.get_positions(), e.get_velocities(), e.get_boxes(), e.get_barostat_anisotropic(), e.get_replica_energies()[0])
    e.close()
    return out, s['box']


@pytest.mark.parametrize('mask', ['xyz', 'z'])
def test_trajectory_boxes_and_axis_state_do_not_depend_on_the_cluster_width(mask):
    """2048 atoms at CL = 2 and 8: positions, velocities, boxes and every per-axis record are the same bits."""
    (a, box0), (b, _) = aniso_run(2, MASKS[mask]), aniso_run(8, MASKS[mask])
    assert not np.array_equal(a[2], np.tile(box0, (4, 1))), 'no move accepted'
    for x, y in zip(a[:3], b[:3]):
        assert np.array_equal(x, y)
    for f in a[3]:
        assert np.array_equal(a[3][f], b[3][f]), f


# ---- 5. volume law and cutoff limit --------------------------------------------------------------------------------------
def test_z_only_ideal_gas_volume_law():
    """epsilon = 0, 512 atoms, 64 replicas, z scaled only: V has mean (N+1) kT/p and variance (N+1) (kT/p)^2 after
    equilibration, and x and y keep their edges."""
    N, K = 512, 64
    s = lj_setup(N=N, n_alch=0, seed=4)
    kT = KB * 300.0
    p = (N + 1) * kT / np.prod(s['box'])
    e = aniso_engine(s, K, 1, [1.0], [300.0], [p], [0.0], 4, eps=np.zeros(N))
    e.set_positions(np.stack([s['x']] * K))
    e.randomize_velocities(1)
    e.set_integrator(0.004, 5.0, 500)
    vols = []
    for it in range(80):
        e.propagate(5, it)
        if it >= 15:
            b = e.get_boxes()
            assert np.array_equal(b[:, :2], np.tile(s['box'][:2], (K, 1)))
            vols.append(np.prod(b, axis=1))
    e.close()
    v = np.array(vols).T
    Vm, Vv = (N + 1) * kT / p, (N + 1) * (kT / p) ** 2
    means, variances = v.mean(axis=1), v.var(axis=1)
    se_m, se_v = means.std(ddof=1) / np.sqrt(K), variances.std(ddof=1) / np.sqrt(K)
    assert abs(means.mean() - Vm) < 4 * se_m, (means.mean(), Vm, se_m)
    assert abs(variances.mean() - Vv) < 4 * se_v, (variances.mean(), Vv, se_v)


def test_scaled_edge_never_below_twice_the_cutoff():
    N, K = 256, 16
    s = lj_setup(N=N, n_alch=0, seed=6)
    kT = KB * 300.0
    p = (N + 1) * kT / (s['box'][0] * s['box'][1] * 1.6 * s['rc'])   # the ideal gas's mean z edge lies below the limit
    e = aniso_engine(s, K, 1, [1.0], [300.0], [p], [0.0], 4, eps=np.zeros(N))
    e.set_positions(np.stack([s['x']] * K))
    e.randomize_velocities(1)
    e.set_integrator(0.004, 5.0, 500)
    for it in range(40):
        e.propagate(8, it)
        assert e.get_boxes()[:, 2].min() >= 2 * s['rc']
    assert e.get_boxes()[:, 2].min() < 2.1 * s['rc']
    e.close()


# ---- 6. NaN restart ------------------------------------------------------------------------------------------------------
def nan_engine():
    N, K = 512, 4
    s = lj_setup(N=N, n_alch=10, seed=11)
    e = aniso_engine(s, K, K, np.linspace(1.0, 0.0, K), np.full(K, 300.0), np.full(K, 40.0 * BAR), np.full(K, -25.0), 5)
    e.set_positions(np.stack([s['x']] * K))
    e.randomize_velocities(3)
    e.set_integrator(0.002, 5.0, 100)
    e.propagate(17, 0)
    bad = e.get_positions()
    bad[2, 5] = np.inf
    e.set_positions(bad)
    return e


def test_nan_restart_restores_the_axis_state():
    from openmmtools_b200 import _lib
    from openmmtools_b200._engine import EngineError
    e = nan_engine()
    snap = e.get_barostat_anisotropic()
    with pytest.raises(EngineError) as err:
        e.propagate(17, 1)
    assert err.value.code == _lib.RX_ERR_NAN and list(err.value.nan_flags) == [0, 0, 1, 0]
    after = e.get_barostat_anisotropic()
    assert not np.array_equal(after['n_attempted'][2], snap['n_attempted'][2]), 'the failed run left the record as it was'
    with pytest.raises(EngineError):
        e.propagate_retry(18, 1)
    retry = e.get_barostat_anisotropic()
    e.close()
    ref_e = nan_engine()
    with pytest.raises(EngineError):
        ref_e.propagate(18, 1)
    ref = ref_e.get_barostat_anisotropic()
    ref_e.close()
    for f in retry:
        for k in (0, 1, 3):
            assert np.array_equal(retry[f][k], after[f][k]), (f, k)
        assert np.array_equal(retry[f][2], ref[f][2]), f


# ---- 7. the sampler ------------------------------------------------------------------------------------------------------
def aniso_sampler(path, K=4, N=128, iterations=4, scale=(False, False, True)):
    from openmmtools_b200 import unit, states, alchemy, mcmc, multistate, testsystems
    from openmmtools_b200.multistate import MultiStateReporter
    from openmmtools_b200.system import MonteCarloAnisotropicBarostat
    asys = alchemical_fluid(N=N, dispersion=True)
    asys.addForce(MonteCarloAnisotropicBarostat(1.0 * unit.bar, 300 * unit.kelvin, *scale))
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


def test_sampler_run_stores_fuses_and_resumes(tmp_path):
    from openmmtools_b200 import multistate
    from openmmtools_b200.multistate import MultiStateReporter
    a, asys, _ = aniso_sampler(str(tmp_path / 'a.store'))
    a.run()
    xa = np.stack([st._positions for st in a.sampler_states])
    ba = np.stack([st._box_vectors for st in a.sampler_states])
    edges = np.einsum('kii->ki', ba)
    assert len({tuple(b) for b in edges}) > 1, 'every replica kept the initial box'
    assert np.array_equal(edges[:, :2], np.tile(np.diag(asys.box_vectors)[:2], (len(edges), 1)))
    aa = a._engine.get_barostat_anisotropic()
    assert (aa['scale_mask'] == 4).all() and aa['n_attempted'][:, :2].sum() == 0
    r = MultiStateReporter(str(tmp_path / 'a.store'), open_mode='r')
    assert np.array_equal(r.read_volumes(4), np.prod(edges, axis=1))
    assert r.read_energies(4)[2].shape[1] == 1
    # the fused device loop gives the same bits as the host loop
    d, _, _ = aniso_sampler(str(tmp_path / 'd.store'))
    d._compute_energies()
    d._engine.run_iterations(4, 'swap-all', d._seed, 1)
    assert np.array_equal(d._engine.get_positions(), a._engine.get_positions())
    assert np.array_equal(d._engine.get_boxes(), a._engine.get_boxes())
    da = d._engine.get_barostat_anisotropic()
    assert all(np.array_equal(da[f], aa[f]) for f in aa)
    # interrupted after 3 iterations (last checkpoint 2), resumed from storage: the same bits as the uninterrupted run
    b, _, _ = aniso_sampler(str(tmp_path / 'b.store'))
    b.run(3)
    del b
    c2 = multistate.ReplicaExchangeSampler.from_storage(str(tmp_path / 'b.store'))
    assert c2.iteration == 2
    c2.run()
    assert np.array_equal(np.stack([st._positions for st in c2.sampler_states]), xa)
    assert np.array_equal(np.stack([st._box_vectors for st in c2.sampler_states]), ba)
    assert np.array_equal(c2._energy_thermodynamic_states, a._energy_thermodynamic_states)
    assert np.array_equal(c2._energy_unsampled_states, a._energy_unsampled_states)
    ca = c2._engine.get_barostat_anisotropic()
    assert all(np.array_equal(ca[f], aa[f]) for f in aa)


def test_reduced_potential_of_an_anisotropic_state():
    """beta (U + c / V + p V) at a SamplerState's own rectangular box (states.py:1909-1917), as for the isotropic one."""
    from openmmtools_b200 import unit, states, alchemy, _backend, testsystems
    from openmmtools_b200.system import MonteCarloAnisotropicBarostat
    from oracle import oracle
    asys = alchemical_fluid(N=128, dispersion=True)
    asys.addForce(MonteCarloAnisotropicBarostat([35.0, 1.0, 35.0] * unit.bar, 310 * unit.kelvin, True, False, True))
    x = np.asarray(testsystems.LennardJonesFluid(nparticles=128).positions.value_in_unit(unit.nanometer), np.float64)
    ts = states.create_thermodynamic_state_protocol(asys, {'lambda_sterics': [0.4]},
                                                    constants={'temperature': 310.0 * unit.kelvin},
                                                    composable_states=alchemy.AlchemicalState.from_system(asys))[0]
    assert ts.pressure == 35.0 * unit.bar and ts._barostat_scale == (True, False, True)
    f = np.array([1.07, 1.0, 0.96])
    edges = np.diag(asys.box_vectors) * f
    ss = states.SamplerState(x * f, box_vectors=unit.Quantity(np.diag(edges), unit.nanometer))
    u = ts.reduced_potential(ss)
    osys = oracle.LJSystem(asys.sigma, asys.epsilon, asys.masses, asys.alchemical_mask(), tuple(edges), asys.cutoff,
                           asys.switching_distance)
    U = osys.energy((x * f).astype(np.float32).astype(np.float64), 0.4)[0]
    V = np.prod(edges)
    c = _backend.pressure_tables([ts])[1][0]
    assert u == pytest.approx((U + c / V + 35.0 * BAR * V) / (KB * 310.0), rel=1e-9)


# ---- 8. two GPUs ---------------------------------------------------------------------------------------------------------
def aniso_sharded_run(prefix):
    """8 replicas, z scaled, 3 iterations: the owned rows of positions, boxes and per-axis records, the energy matrix
    and the replica->state map, and the records rank 0 gathered."""
    a, _, _ = aniso_sampler(prefix + 'a.store', K=8, iterations=3, scale=(True, False, True))
    a.run()
    e = a._engine
    out = dict(k0=e.k0, x=e.get_positions(), box=e.get_boxes(), u=np.array(a._energy_thermodynamic_states),
               perm=np.array(a._replica_thermodynamic_states),
               **{'aniso_' + f: v for f, v in e.get_barostat_anisotropic().items()})
    if a._last_aniso_records is not None:
        out['records'] = a._last_aniso_records
    return out


WORKER = r'''
import os, sys
sys.path.insert(0, %(root)r)
sys.path.insert(0, os.path.join(%(root)r, 'tests'))
import numpy as np
import torch.distributed as dist
dist.init_process_group('gloo')
from test_gpu_npt_anisotropic import aniso_sharded_run
rank = dist.get_rank()
np.savez(%(out)r + '_%%d.npz' %% rank, **aniso_sharded_run(%(out)r + '_%%d_' %% rank))
dist.barrier()
'''


def test_two_gpus_reproduce_single_gpu(tmp_path):
    from test_multi_gpu import _two_devices
    if not _two_devices():
        pytest.skip('needs 2 GPUs')
    ref = aniso_sharded_run(str(tmp_path / 'one_'))
    script = tmp_path / 'aniso2.py'
    out = str(tmp_path / 'two')
    script.write_text(WORKER % {'root': ROOT, 'out': out})
    r = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2',
                        '--master-addr', '127.0.0.1', '--master-port', '29541', str(script)],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    for rank in range(2):
        d = np.load(out + '_%d.npz' % rank)
        k0, n = int(d['k0']), d['x'].shape[0]
        assert n == 4, n
        for key in ref:
            if key in ('k0', 'records'):
                continue
            want = ref[key] if key in ('u', 'perm') else ref[key][k0:k0 + n]
            assert np.array_equal(d[key], want), (rank, key)
        if rank == 0:
            assert np.array_equal(d['records'], ref['records'])
