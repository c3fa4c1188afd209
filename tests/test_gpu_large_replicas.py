"""Replicas of 1025 to 4096 atoms (DESIGN 4.2): k_propagate over a cluster of 2, 4 or 8 blocks in the compact shared-memory
layout, k_minimize with four atoms per thread and k_energy_rows, against the double-precision oracle and against
themselves at every cluster width that can hold the atoms.  Systems: three atom types, a rectangular box, alchemical atoms
scattered over the blocks of an 8-block cluster."""
import numpy as np
import pytest
from helpers import (lj_setup, oracle_system, gpu_engine, KB, device_noise, THREE_TYPES, RECT, scattered_alch, wrap,
                     min_image)

pytestmark = pytest.mark.gpu
RTOL = 1e-10
N_SM, OPTIN = 132, 227 * 1024        # H100 SXM: multiprocessors, opt-in shared memory per block


def big(N, seed, box='rect', **kw):
    return lj_setup(N=N, seed=seed, types=THREE_TYPES, box_ratio=RECT if box == 'rect' else (1.0, 1.0, 1.0),
                    alch=scattered_alch(N, cluster=8), **kw)


def feasible_clusters(s, K):
    """The cluster widths of 2, 4, 8 blocks rx_propagate accepts as RX_CLUSTER for this system (they hold the atoms and a
    list of 48 entries)."""
    from openmmtools_b200._engine import Engine
    from openmmtools_b200._lib import RX_SYSTEM_LJ_ALCH
    return [c for c in (2, 4, 8) if Engine.plan_propagate(RX_SYSTEM_LJ_ALCH, s['N'], K, N_SM, OPTIN, box=tuple(s['box']),
                                                           r_cutoff=s['rc'], cluster=c)['cluster'] == c]


def make_engine(s, K, M, lambdas, temps, dt, gamma, n_steps, splitting):
    e = gpu_engine(1, K, M, s['N'], box=tuple(s['box']), r_cutoff=s['rc'], r_switch=s['rs'], use_switch=True)
    e.set_particles(s['sigma'], s['eps'], s['mass'], s['alch'])
    e.set_states(temps, lambdas)
    e.set_integrator(dt, gamma, n_steps, splitting)
    return e


def max_image_dev(xg, x, box):
    return np.abs(min_image(xg - wrap(x, box), box)).max()


def perturbed(s, K, seed):
    rng = np.random.default_rng(seed)
    return np.stack([(s['x'] + rng.normal(scale=0.03, size=(s['N'], 3))).astype(np.float32).astype(np.float64)
                     for _ in range(K)])


# ---- 1. energies --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('N,annihilate,c,M', [(1025, False, 6.0, 7), (1500, True, 6.0, 600), (2048, False, 4.0, 64),
                                              (3000, True, 4.0, 513), (4096, False, 6.0, 600)])
def test_energy_matrix_above_1024_atoms_matches_oracle(N, annihilate, c, M):
    K = 3
    s = big(N, seed=N)
    xs = perturbed(s, K, N + 1)
    lambdas = np.linspace(1.0, 0.0, M); temps = np.linspace(290.0, 340.0, M); offsets = np.linspace(-2.5, 1.5, M)
    e = gpu_engine(1, K, M, N, box=tuple(s['box']), r_cutoff=s['rc'], r_switch=s['rs'], use_switch=True,
                   annihilate_sterics=annihilate, softcore_c=c)
    e.set_particles(s['sigma'], s['eps'], s['mass'], s['alch'])
    e.set_states(temps, lambdas, offsets)
    e.set_positions(xs)
    u = e.compute_energies()
    # and at 600 other states (rx_compute_energies_at)
    la2, t2, o2 = np.linspace(0.0, 1.0, 600), np.linspace(280.0, 360.0, 600), np.linspace(1.0, -1.0, 600)
    u2 = e.compute_energies_at(t2, la2, o2)
    e.close()
    osys = oracle_system(s, annihilate=annihilate, c=c)
    for got, ref in ((u, osys.energy_matrix(xs, lambdas, 1.0 / (KB * temps), offsets)),
                     (u2, osys.energy_matrix(xs, la2, 1.0 / (KB * t2), o2))):
        err = np.abs(got - ref) / np.maximum(1.0, np.abs(ref))
        assert err.max() <= RTOL, err.max()


# ---- 2. steps against the oracle fed with the device's noise ------------------------------------------------------------
def steps_vs_oracle(s, K, n_steps, dt, gamma, temps, lambdas, seed, iteration, v0, bx=2e-5, bv=2e-4, rel_v=False):
    N = s['N']
    e = make_engine(s, K, K, lambdas, temps, dt, gamma, n_steps, 'V R O R V')
    x0 = np.stack([s['x']] * K)
    e.set_positions(x0); e.set_velocities(v0); e.set_replica_states(np.arange(K))
    e.propagate(seed, iteration)
    xg, vg = e.get_positions(), e.get_velocities()
    pot, kin = e.get_replica_energies()
    e.close()
    osys = oracle_system(s)
    moved = 0.0
    for k in range(K):
        x = x0[k].copy(); v = v0[k].copy()
        U = osys.langevin(x, v, device_noise(seed, iteration, k, N, n_steps), lambdas[k], KB * temps[k], dt, gamma, n_steps,
                          'VRORV')
        moved = max(moved, np.sqrt(((x - x0[k]) ** 2).sum(axis=1)).max())
        assert max_image_dev(xg[k], x, s['box']) < bx, (k, max_image_dev(xg[k], x, s['box']))
        vb = bv * max(1.0, np.abs(v).max()) if rel_v else bv
        assert np.abs(vg[k] - v).max() < vb, (k, np.abs(vg[k] - v).max())
        assert abs(pot[k] - U) < 1e-3 * max(1.0, abs(U)), (pot[k], U)
        ke = 0.5 * (s['mass'][:, None] * v * v).sum()
        assert abs(kin[k] - ke) < 1e-4 * ke
    return moved


STEP_CASES = [(N, cl) for N in (1025, 2047, 2048) for cl in (2, 4, 8)] + [(4096, 8)]


@pytest.mark.parametrize('N,cl', STEP_CASES)
def test_steps_above_1024_atoms_match_oracle_with_same_noise(monkeypatch, N, cl):
    K = 4
    s = big(N, seed=N)
    assert cl in feasible_clusters(s, K)
    monkeypatch.setenv('RX_CLUSTER', str(cl))
    v0 = np.random.default_rng(2).normal(scale=0.25, size=(K, N, 3)).astype(np.float32).astype(np.float64)
    steps_vs_oracle(s, K, 6, 0.002, 10.0, np.array([300.0, 310.0, 320.0, 330.0]), np.array([1.0, 0.6, 0.3, 0.0]),
                    0x1234567890ABCDEF, 7, v0)


def test_cluster_of_4096_atoms_is_8_blocks_only():
    assert feasible_clusters(big(4096, seed=4096), 4) == [8]


@pytest.mark.parametrize('N,cl', [(2048, 2), (2048, 8), (4096, 8)])
def test_steps_across_outer_rebuilds_above_1024_atoms_match_oracle(monkeypatch, N, cl):
    """Skins shrunk to 0.09 / 0.03 nm: 25 hot steps with light atoms cross several outer rebuilds, each re-dealing the
    atoms to threads inside every block of the cluster."""
    K, n_steps = 2, 25
    s = big(N, seed=71)
    monkeypatch.setenv('RX_CLUSTER', str(cl))
    monkeypatch.setenv('RX_SKIN', '0.09')
    monkeypatch.setenv('RX_SKIN_IN', '0.03')
    rng = np.random.default_rng(9)
    v0 = (rng.normal(size=(K, N, 3)) * np.sqrt(KB * 600.0 / s['mass'])[:, None]).astype(np.float32).astype(np.float64)
    moved = steps_vs_oracle(s, K, n_steps, 0.002, 1.0, np.array([600.0, 600.0]), np.array([1.0, 0.4]), 0x5EED0F0DDBA11, 4,
                            v0, bx=1e-4, bv=1e-3)
    assert moved > 2 * 0.03, moved


def test_dense_fluid_of_2048_atoms_falls_back_to_all_pairs_and_matches_oracle():
    """Liquid density: more neighbours than a list column holds -> the whole cluster switches to the all-pairs loop."""
    K, N = 2, 2048
    s = big(N, seed=31, box='cubic', reduced_density=0.6)
    v0 = np.random.default_rng(8).normal(scale=0.2, size=(K, N, 3)).astype(np.float32).astype(np.float64)
    # (forces of a dense, roughly packed start are large: velocities to float32 accuracy of those forces)
    steps_vs_oracle(s, K, 4, 0.001, 10.0, np.array([300.0, 300.0]), np.array([1.0, 0.4]), 5, 1, v0, rel_v=True)


# ---- 3. bit for bit -------------------------------------------------------------------------------------------------------
def _hot_run(s, K, n_steps, seed=1234, iteration=9):
    lambdas = np.linspace(1.0, 0.0, K); temps = np.full(K, 500.0)
    v0 = np.random.default_rng(15).normal(scale=0.3, size=(K, s['N'], 3)).astype(np.float32).astype(np.float64)
    e = make_engine(s, K, K, lambdas, temps, 0.002, 1.0, n_steps, 'V R O R V')
    e.set_positions(np.stack([s['x']] * K)); e.set_velocities(v0)
    e.set_replica_states((np.arange(K) + 1) % K)
    e.propagate(seed, iteration)
    out = (e.get_positions(), e.get_velocities(), e.get_replica_energies())
    e.close()
    return out


def assert_same_trajectory(a, b):
    (xa, va, (pa, ka)), (xb, vb, (pb, kb)) = a, b
    assert np.array_equal(xa, xb) and np.array_equal(va, vb), (np.abs(xa - xb).max(), np.abs(va - vb).max())
    # (other block partitions sum the f64 energies in other partial sums: last-bit differences)
    assert np.allclose(pa, pb, rtol=1e-12, atol=1e-9) and np.allclose(ka, kb, rtol=1e-12, atol=1e-9)


@pytest.mark.parametrize('N', [1025, 2048])
def test_trajectory_above_1024_atoms_does_not_depend_on_cluster_width(monkeypatch, N):
    """200 hot steps (re-partitions and outer rebuilds) at every feasible cluster width give the same trajectory.  (4096
    atoms fit with a list only in 8 blocks: test_cluster_of_4096_atoms_is_8_blocks_only.)"""
    K = 3
    s = big(N, seed=51)
    out = []
    for c in feasible_clusters(s, K):
        monkeypatch.setenv('RX_CLUSTER', str(c))
        out.append(_hot_run(s, K, 200))
    assert len(out) == 3
    for o in out[1:]:
        assert_same_trajectory(out[0], o)


@pytest.mark.parametrize('N,cl', [(2048, 2), (4096, 8)])
def test_unsorted_atom_deal_above_1024_atoms_reproduces_sorted_trajectory(monkeypatch, N, cl):
    s = big(N, seed=81)
    monkeypatch.setenv('RX_CLUSTER', str(cl))
    a = _hot_run(s, 3, 250)
    monkeypatch.setenv('RX_NO_SORT', '1')
    assert_same_trajectory(a, _hot_run(s, 3, 250))


# ---- 4. per-state moves ---------------------------------------------------------------------------------------------------
def test_per_state_moves_of_2048_atoms_equal_single_move_engines():
    K, N = 4, 2048
    s = big(N, seed=61)
    lambdas = np.array([1.0, 0.7, 0.3, 0.0]); temps = np.array([300.0, 320.0, 340.0, 360.0])
    A = (0.002, 1.0, 40, 'V R O R V', False)
    B = (0.001, 5.0, 25, 'O V R V O', True)
    v0 = np.random.default_rng(16).normal(scale=0.3, size=(K, N, 3)).astype(np.float32).astype(np.float64)
    perm = np.array([2, 0, 3, 1])

    def run(moves):
        e = make_engine(s, K, K, lambdas, temps, *moves[0][:4])
        if any(m != moves[0] for m in moves):
            for l, m in enumerate(moves):
                e.set_state_integrator(l, *m)
        e.set_positions(np.stack([s['x']] * K)); e.set_velocities(v0)
        e.set_replica_states(perm)
        e.propagate(77, 3, moves[0][4] if all(m == moves[0] for m in moves) else False)
        out = (e.get_positions(), e.get_velocities(), e.get_replica_energies())
        e.close()
        return out
    xm, vm, (pm, km) = run([A, A, B, B])
    xa, va, (pa, ka) = run([A] * 4)
    xb, vb, (pb, kb) = run([B] * 4)
    for k in range(K):
        x_ref, v_ref, p_ref, k_ref = (xa, va, pa, ka) if perm[k] < 2 else (xb, vb, pb, kb)
        assert np.array_equal(xm[k], x_ref[k]) and np.array_equal(vm[k], v_ref[k]), k
        assert np.isclose(pm[k], p_ref[k], rtol=1e-12, atol=1e-9) and np.isclose(km[k], k_ref[k], rtol=1e-12, atol=1e-9), k
    assert not np.array_equal(xa[0], xb[0])


# ---- 5. NaN restart -------------------------------------------------------------------------------------------------------
def test_nan_restart_of_2048_atoms_retries_only_the_failed_replica():
    """rx_propagate reports the replica whose velocities were made absurd; rx_propagate_retry puts only that replica back to
    the start of the call and propagates it again; the others keep their result of the first call."""
    from openmmtools_b200._engine import EngineError
    K, N = 4, 2048
    s = big(N, seed=91)
    lambdas = np.linspace(1.0, 0.0, K); temps = np.full(K, 300.0)

    def engine():
        e = make_engine(s, K, K, lambdas, temps, 0.002, 5.0, 20, 'V R O R V')
        e.set_positions(np.stack([s['x']] * K))
        e.set_velocities(np.random.default_rng(3).normal(scale=0.3, size=(K, N, 3)))
        e.set_replica_states(np.arange(K))
        return e
    clean, sick = engine(), engine()
    clean.propagate(5, 1)
    v = sick.get_velocities()
    v[2] = 1e30
    sick.set_velocities(v[2:3], first=2)
    x_start = sick.get_positions()
    with pytest.raises(EngineError) as first:
        sick.propagate(5, 1)
    xs1 = sick.get_positions()
    with pytest.raises(EngineError) as retry:
        sick.propagate_retry(6, 1)
    assert first.value.nan_flags.tolist() == [0, 0, 1, 0] and retry.value.nan_flags.tolist() == [0, 0, 1, 0]
    xs2, xc = sick.get_positions(), clean.get_positions()
    for k in range(K):
        if k != 2:
            assert np.array_equal(xs1[k], xc[k]) and np.array_equal(xs2[k], xc[k]), k   # propagated once, not retried
    assert not np.array_equal(xs2[2], x_start[2])    # (retried from the start and failed again)
    clean.close(); sick.close()


# ---- 6. minimiser ---------------------------------------------------------------------------------------------------------
def test_minimize_2048_atoms_meets_force_tolerance():
    N, K, tol = 2048, 2, 1.0
    s = big(N, seed=14)
    lambdas = np.array([1.0, 0.3])
    e = make_engine(s, K, K, lambdas, np.full(K, 300.0), 0.001, 10.0, 1, 'V R O R V')
    x0 = np.stack([s['x'] + np.random.default_rng(k).normal(scale=0.02, size=(N, 3)) for k in range(K)])
    x0 = x0.astype(np.float32).astype(np.float64)
    e.set_positions(x0); e.set_replica_states(np.arange(K))
    rms, its = e.minimize(tol)
    x1 = e.get_positions()
    e.close()
    assert np.all(x1 >= 0) and np.all(x1 < s['box'])
    osys = oracle_system(s)
    for k in range(K):
        e1, _, f1 = osys.energy(x1[k], lambdas[k], forces=True)
        rms_ref = np.sqrt(np.mean(f1 ** 2))
        assert e1 < osys.energy(x0[k], lambdas[k])[0] and its[k] > 0
        assert rms[k] <= tol and rms_ref < tol * 1.02, (k, rms[k], rms_ref)
        assert abs(rms[k] - rms_ref) < 1e-3 * tol, (k, rms[k], rms_ref)


# ---- 7. sampler level -----------------------------------------------------------------------------------------------------
def test_replica_exchange_of_2048_atom_fluid_stores_oracle_energies_and_resumes_bit_identically(tmp_path):
    from openmmtools_b200 import unit, states, alchemy, mcmc, testsystems, multistate, _backend
    from openmmtools_b200.multistate import MultiStateReporter
    from oracle import oracle
    K, N = 4, 2048
    fluid = testsystems.LennardJonesFluid(nparticles=N)
    asys = alchemy.AbsoluteAlchemicalFactory(disable_alchemical_dispersion_correction=True).create_alchemical_system(
        fluid.system, alchemy.AlchemicalRegion(alchemical_atoms=range(8)))
    lambdas = [1.0 - l / (K - 1) for l in range(K)]
    tstates = states.create_thermodynamic_state_protocol(asys, {'lambda_sterics': lambdas}, constants={'temperature': 300.0 * unit.kelvin},
                                                         composable_states=alchemy.AlchemicalState.from_system(asys))
    sstate = states.SamplerState(fluid.positions, box_vectors=asys.getDefaultPeriodicBoxVectors())
    move = mcmc.LangevinSplittingDynamicsMove(timestep=1.0 * unit.femtosecond, n_steps=25)

    def new_sampler(path):
        s = multistate.ReplicaExchangeSampler(mcmc_moves=move, number_of_iterations=4, replica_mixing_scheme='swap-all', seed=7)
        s.create(tstates, [sstate], storage=MultiStateReporter(path, checkpoint_interval=2))
        return s
    a = new_sampler(str(tmp_path / 'a.store'))
    a.run()
    assert a.iteration == 4
    xa = np.stack([st._positions for st in a.sampler_states])
    ra = MultiStateReporter(str(tmp_path / 'a.store'), open_mode='r')
    ua = ra.read_energies(4)[0]
    L = asys.box_vectors[0, 0]
    osys = oracle.LJSystem(asys.sigma, asys.epsilon, asys.masses, asys.alchemical_mask(), (L, L, L), asys.cutoff,
                           asys.switching_distance, use_switch=True)
    ref = osys.energy_matrix(xa, np.array(lambdas), np.full(K, 1.0 / (KB * 300.0)), np.full(K, _backend.lj_dispersion_correction(asys)))
    err = np.abs(ua - ref) / np.maximum(1.0, np.abs(ref))
    assert err.max() <= RTOL, err.max()
    # interrupted after 3 iterations (last checkpoint 2), resumed from storage
    b = new_sampler(str(tmp_path / 'b.store'))
    b.run(3)
    del b
    c = multistate.ReplicaExchangeSampler.from_storage(str(tmp_path / 'b.store'))
    assert c.iteration == 2
    c.run()
    assert c.iteration == 4
    assert np.array_equal(c._replica_thermodynamic_states, a._replica_thermodynamic_states)
    assert np.array_equal(c._energy_thermodynamic_states, a._energy_thermodynamic_states)
    assert np.array_equal(np.stack([st._positions for st in c.sampler_states]), xa)
