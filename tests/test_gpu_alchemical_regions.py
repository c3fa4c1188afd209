"""Two alchemical regions on the device: the energy matrix (k_energy_rows, f64) against the inclusion-exclusion of the
one-region oracle (regions_ref.py), the force kernels (k_propagate in every layout, k_minimize) against the one-region
kernels where the two must agree bit for bit, steps with both regions visible against the f64 reference fed the device's
noise, and the samplers through the public API (replica exchange with storage and resume, SAMS, two GPUs)."""
import numpy as np
import pytest
from helpers import lj_setup, gpu_engine, KB, THREE_TYPES, RECT, scattered_alch, device_noise, min_image, wrap
from regions_ref import RegionsReference

pytestmark = pytest.mark.gpu
RTOL = 1e-10


def assert_close(u, ref):
    err = np.abs(u - ref) / np.maximum(1.0, np.abs(ref))
    assert err.max() <= RTOL, err.max()


def regions_of(N):
    """Region 1: the scattered atoms (the last atom of every cluster block, the last warp, atom N-1); region 2: five
    atoms next to them."""
    r1 = scattered_alch(N)
    rest = np.setdiff1d(np.arange(N), r1)
    r2 = rest[np.linspace(0, len(rest) - 1, min(5, len(rest))).astype(int)]
    ids = np.zeros(N, np.uint8)
    ids[r1] = 1
    ids[r2] = 2
    return ids


def system(N, seed, box='rect'):
    return lj_setup(N=N, seed=seed, types=THREE_TYPES, box_ratio=RECT if box == 'rect' else (1.0, 1.0, 1.0),
                    alch=scattered_alch(N))


def engine(s, K, M, ids, ann, c=6.0, a=1.0, b=1.0, regions=True):
    e = gpu_engine(1, K, M, s['N'], box=tuple(s['box']), r_cutoff=s['rc'], r_switch=s['rs'], use_switch=True,
                   annihilate_sterics=ann[0], softcore_c=c, softcore_a=a, softcore_b=b)
    e.set_particles(s['sigma'], s['eps'], s['mass'], (ids != 0).astype(np.uint8) if regions else (ids == 1).astype(np.uint8))
    if regions:
        e.set_alchemical_regions(ids, *ann)
    return e


def perturbed(s, K, seed):
    rng = np.random.default_rng(seed)
    return np.stack([(s['x'] + rng.normal(scale=0.03, size=(s['N'], 3))).astype(np.float32).astype(np.float64)
                     for _ in range(K)])


def grid(n):
    """A (lambda_1, lambda_2) grid of about n states with 0 and 1 on both axes."""
    m = max(2, int(round(np.sqrt(n))))
    g1, g2 = np.meshgrid(np.linspace(0.0, 1.0, m), np.linspace(1.0, 0.0, m), indexing='ij')
    return g1.ravel(), g2.ravel()


@pytest.mark.parametrize('N,M,ann,c', [(64, 16, (False, True), 6.0), (512, 600, (True, False), 6.0),
                                       (1000, 64, (False, False), 4.0), (2048, 36, (True, True), 6.0),
                                       (4096, 9, (False, True), 6.0)])
def test_energy_matrix_matches_oracle(N, M, ann, c):
    K = 3
    s = system(N, seed=N)
    ids = regions_of(N)
    xs = perturbed(s, K, N + 1)
    l1, l2 = grid(M)
    M = len(l1)
    temps = np.linspace(290.0, 340.0, M)
    offsets = np.linspace(-2.5, 1.5, M)
    e = engine(s, K, M, ids, ann, c=c)
    e.set_states(temps, l1, offsets, lambda_sterics_2=l2)
    e.set_positions(xs)
    u = e.compute_energies()
    # the unsampled-state path takes the second lambda as well
    u_at = e.compute_energies_at(temps[::-1], l1[::-1], offsets[::-1], lambda_sterics_2=l2[::-1])
    e.close()
    ref = RegionsReference(s, ids, *ann, c=c)
    betas = 1.0 / (KB * temps)
    assert_close(u, ref.energy_matrix(xs, l1, l2, betas, offsets))
    assert_close(u_at, ref.energy_matrix(xs, l1[::-1], l2[::-1], betas[::-1], offsets[::-1]))


@pytest.mark.parametrize('N', [512, 2048])
def test_energy_matrix_at_constant_pressure(N):
    K, M = 3, 25
    s = system(N, seed=3 * N)
    ids = regions_of(N)
    xs = perturbed(s, K, 5)
    l1, l2 = grid(M)
    temps = np.full(M, 300.0)
    pressure = np.linspace(0.05, 0.1, M); dispersion = np.linspace(-3.0, -1.0, M)
    boxes = np.stack([s['box'] * f for f in (1.0, 1.02, 0.985)])
    e = engine(s, K, M, ids, (False, True))
    e.set_states(temps, l1, None, lambda_sterics_2=l2)
    e.set_pressures(pressure, dispersion)
    e.set_positions(xs)
    e.set_boxes(boxes)
    u = e.compute_energies()
    u_at = e.compute_energies_at(temps[:4], l1[:4], None, pressure=pressure[:4], dispersion=dispersion[:4],
                                 lambda_sterics_2=l2[::-1][:4])
    e.close()
    betas = 1.0 / (KB * temps)
    for k in range(K):
        V = np.prod(boxes[k])
        ref = RegionsReference(s, ids, False, True, box=boxes[k])
        row = ref.energy_matrix(xs[k:k + 1], l1, l2, betas)[0] + betas * (dispersion / V + pressure * V)
        assert_close(u[k], row)
        row_at = ref.energy_matrix(xs[k:k + 1], l1[:4], l2[::-1][:4], betas[:4])[0] + betas[:4] * (
            dispersion[:4] / V + pressure[:4] * V)
        assert_close(u_at[k], row_at)


def run_pair(s, ids_two, ann_two, l_two, ids_one, ann_one, l_one, K, steps, monkeypatch, cl=None, npt=False,
             per_state=False, minimize=False):
    """Propagate the same replicas with the two-region kernels and with the one-region kernels; both engines' outputs."""
    if cl is not None:
        monkeypatch.setenv('RX_CLUSTER', str(cl))
    out = []
    M = K
    temps = np.linspace(300.0, 330.0, M)
    for regions, ids, ann, lam in ((True, ids_two, ann_two, l_two), (False, ids_one, ann_one, l_one)):
        e = engine(s, K, M, ids, ann, regions=regions)
        if regions:
            e.set_states(temps, lam[0], None, lambda_sterics_2=lam[1])
        else:
            e.set_states(temps, lam, None)
        if npt:
            e.set_pressures(np.full(M, 0.06), np.full(M, -2.0))
        e.set_integrator(0.002, 5.0, steps)
        if per_state:
            for l in range(M):
                e.set_state_integrator(l, 0.001 + 0.0005 * l, 2.0 + l, steps - l % 2)
        e.set_positions(perturbed(s, K, 9))
        e.randomize_velocities(7)
        if minimize:
            e.minimize(50.0, 200)
        for it in range(2):
            e.propagate(1234, it)
        pot, kin = e.get_replica_energies()
        out.append((e.get_positions(), e.get_velocities(), pot, kin, e.get_boxes() if npt else None))
        e.close()
    return out


# Region B with epsilon 0 contributes nothing in either kernel, so a two-region engine with region A as region 1 (or as
# region 2, with the lambdas swapped) must reproduce the one-region engine of region A bit for bit: every pair of A is
# the same float expression, every pair of B adds exactly zero.
LAYOUTS = [(256, None, False, False), (300, 1, False, False), (300, 2, False, False), (777, 4, False, False),
           (1024, 1, True, False), (2048, 2, False, False), (2100, 4, False, True), (4096, 8, False, False),
           (512, 1, False, True), (1500, 2, True, True)]


@pytest.mark.parametrize('N,cl,per_state,npt', LAYOUTS)
@pytest.mark.parametrize('a_is', [1, 2])
def test_propagate_with_an_invisible_region_reproduces_one_region(monkeypatch, N, cl, per_state, npt, a_is):
    K = 4
    s = system(N, seed=N + a_is)
    ids = regions_of(N)                      # 1: region A (scattered), 2: region B
    s['eps'] = np.where(ids == 2, 0.0, s['eps'])
    lam_a, lam_b = np.linspace(1.0, 0.0, K), np.linspace(0.2, 0.9, K)
    if a_is == 1:
        two = dict(ids_two=ids, ann_two=(True, False), l_two=(lam_a, lam_b))
    else:
        swapped = np.where(ids == 1, 2, np.where(ids == 2, 1, 0)).astype(np.uint8)
        two = dict(ids_two=swapped, ann_two=(False, True), l_two=(lam_b, lam_a))
    (x2, v2, p2, k2, b2), (x1, v1, p1, k1, b1) = run_pair(
        s, ids_one=ids, ann_one=(True, False), l_one=lam_a, K=K, steps=30, monkeypatch=monkeypatch, cl=cl, npt=npt,
        per_state=per_state, **two)
    assert np.array_equal(x2, x1) and np.array_equal(v2, v1)
    assert np.array_equal(p2, p1) and np.array_equal(k2, k1)
    if npt:
        assert np.array_equal(b2, b1)


@pytest.mark.parametrize('N', [300, 2048])
def test_minimize_with_an_invisible_region_reproduces_one_region(monkeypatch, N):
    K = 3
    s = system(N, seed=N)
    ids = regions_of(N)
    s['eps'] = np.where(ids == 2, 0.0, s['eps'])
    lam = np.linspace(1.0, 0.0, K)
    (x2, _, _, _, _), (x1, _, _, _, _) = run_pair(s, ids, (False, True), (lam, lam[::-1]), ids, (False, False), lam,
                                                  K, 1, monkeypatch, minimize=True)
    assert np.array_equal(x2, x1)


@pytest.mark.parametrize('N,cl,npt', [(512, None, False), (1000, 4, False), (2048, None, True)])
def test_propagated_potential_matches_oracle(monkeypatch, N, cl, npt):
    """Both regions interacting with the environment and across pairs present: the float kernel's potential of the
    final positions against the f64 reference (float32 resolution), and the energy matrix of those positions."""
    if cl is not None:
        monkeypatch.setenv('RX_CLUSTER', str(cl))
    K = M = 4
    s = system(N, seed=N + 7)
    ids = regions_of(N)
    l1, l2 = np.array([1.0, 0.7, 0.3, 0.0]), np.array([0.0, 0.4, 0.8, 1.0])
    temps = np.full(M, 300.0)
    e = engine(s, K, M, ids, (False, True))
    e.set_states(temps, l1, None, lambda_sterics_2=l2)
    if npt:
        e.set_pressures(np.full(M, 0.06), np.zeros(M))
    e.set_integrator(0.002, 5.0, 50)
    e.set_positions(perturbed(s, K, 2))
    e.randomize_velocities(3)
    e.propagate(99, 0)
    pot, _ = e.get_replica_energies()
    x = e.get_positions()
    boxes = e.get_boxes() if npt else np.tile(s['box'], (K, 1))
    states = e.get_replica_states()
    u = e.compute_energies()
    e.close()
    for k in range(K):
        ref = RegionsReference(s, ids, False, True, box=boxes[k])
        l = states[k]
        U = ref.energy(x[k], l1[l], l2[l])
        assert abs(pot[k] - U) <= 1e-4 * max(1.0, abs(U)), (k, pot[k], U)
        row = ref.energy_matrix(x[k:k + 1], l1, l2, 1.0 / (KB * temps))[0]
        if npt:
            row = row + 0.06 * np.prod(boxes[k]) / (KB * temps)
        assert_close(u[k], row)


@pytest.mark.parametrize('N,cl', [(256, None), (777, 4), (2048, 2)])
def test_steps_match_the_reference_fed_the_device_noise(monkeypatch, N, cl):
    """Both regions visible (every epsilon non-zero, across pairs within the cutoff): VRORV steps against the f64
    reference's forces with the device's Philox noise, within the float32 bounds of test_gpu_propagate.py."""
    if cl is not None:
        monkeypatch.setenv('RX_CLUSTER', str(cl))
    K = M = 4
    s = system(N, seed=N + 3)
    ids = regions_of(N)
    l1, l2 = np.array([1.0, 0.6, 0.3, 0.0]), np.array([0.2, 1.0, 0.5, 0.0])
    temps = np.array([300.0, 310.0, 320.0, 330.0])
    dt, gamma, n_steps = 0.002, 10.0, 8
    e = engine(s, K, M, ids, (True, False))
    e.set_states(temps, l1, None, lambda_sterics_2=l2)
    e.set_integrator(dt, gamma, n_steps)
    rng = np.random.default_rng(2)
    x0 = np.stack([s['x']] * K)
    v0 = rng.normal(scale=0.25, size=(K, N, 3)).astype(np.float32).astype(np.float64)
    e.set_positions(x0); e.set_velocities(v0)
    st = np.array([2, 0, 3, 1])
    e.set_replica_states(st)
    seed, iteration = 0x1234567890ABCDEF, 7
    e.propagate(seed, iteration)
    xg, vg = e.get_positions(), e.get_velocities()
    pot, _ = e.get_replica_energies()
    e.close()
    ref = RegionsReference(s, ids, True, False)
    m = s['mass'][:, None]
    a, b = np.exp(-gamma * dt), np.sqrt(1.0 - np.exp(-2.0 * gamma * dt))
    for k in range(K):
        l = st[k]
        x, v = x0[k].copy(), v0[k].copy()
        noise = device_noise(seed, iteration, k, N, n_steps)
        f = ref.energy(x, l1[l], l2[l], forces=True)[1]
        for q in range(n_steps):     # V R O R V
            v += 0.5 * dt * f / m
            x += 0.5 * dt * v
            v = a * v + b * np.sqrt(KB * temps[l] / m) * noise[q]
            x += 0.5 * dt * v
            f = ref.energy(x, l1[l], l2[l], forces=True)[1]
            v += 0.5 * dt * f / m
        U = ref.energy(x, l1[l], l2[l])
        assert np.abs(min_image(xg[k] - wrap(x, s['box']), s['box'])).max() < 2e-5, k
        assert np.abs(vg[k] - v).max() < 2e-4, (k, np.abs(vg[k] - v).max())
        assert abs(pot[k] - U) < 1e-3 * max(1.0, abs(U)), (pot[k], U)


def test_across_pairs_at_zero_separation_contribute_nothing():
    """Dual topology may place an atom of each region at the same point: the pair has no interaction, so the propagation
    and the energies stay finite."""
    N, K = 256, 2
    s = system(N, seed=12)
    ids = regions_of(N)
    i, j = np.nonzero(ids == 1)[0][0], np.nonzero(ids == 2)[0][0]
    xs = perturbed(s, K, 4)
    xs[:, j] = xs[:, i]
    e = engine(s, K, K, ids, (False, False))
    e.set_states(np.full(K, 300.0), np.array([1.0, 0.5]), None, lambda_sterics_2=np.array([1.0, 0.0]))
    e.set_integrator(0.001, 5.0, 10)
    e.set_positions(xs)
    u0 = e.compute_energies()
    e.minimize(1e9, 1)        # one force evaluation at the coincident configuration
    e.set_positions(xs)
    flags = e.propagate(5, 0)
    pot, _ = e.get_replica_energies()
    e.close()
    # (the one-region oracle cannot be the reference here: its soft-core term of the epsilon-0 pair is 0 * inf at r = 0)
    assert np.all(np.isfinite(u0)) and not flags.any() and np.all(np.isfinite(pot))


def dual_sampler(K=6, N=128, iterations=3, storage=None, seed=4321, communicator=None):
    """A ReplicaExchangeSampler on the dual-topology ladder lambda_B = 1 - lambda_A (K not a power of two, swap-all)."""
    from openmmtools_b200 import testsystems, alchemy, states, mcmc, multistate, unit
    fluid = testsystems.LennardJonesFluid(nparticles=N)
    regions = [alchemy.AlchemicalRegion(alchemical_atoms=range(0, 4), name='A'),
               alchemy.AlchemicalRegion(alchemical_atoms=range(4, 8), name='B', annihilate_sterics=True)]
    asys = alchemy.AbsoluteAlchemicalFactory().create_alchemical_system(fluid.system, regions)
    la = np.linspace(1.0, 0.0, K)
    comp = [alchemy.AlchemicalState.from_system(asys, parameters_name_suffix=n) for n in ('A', 'B')]
    tstates = states.create_thermodynamic_state_protocol(
        asys, {'lambda_sterics_A': list(la), 'lambda_sterics_B': list(1.0 - la)},
        constants={'temperature': 300.0 * unit.kelvin}, composable_states=comp)
    sstate = states.SamplerState(fluid.positions, box_vectors=asys.getDefaultPeriodicBoxVectors())
    move = mcmc.LangevinSplittingDynamicsMove(timestep=1.0 * unit.femtosecond, n_steps=20)
    kw = {} if communicator is None else dict(communicator=communicator)
    sampler = multistate.ReplicaExchangeSampler(mcmc_moves=move, number_of_iterations=iterations, seed=seed,
                                                replica_mixing_scheme='swap-all', **kw)
    if storage is not None:
        from openmmtools_b200.multistate import MultiStateReporter
        storage = MultiStateReporter(storage, checkpoint_interval=2)
    sampler.create(tstates, [sstate], storage=storage)
    return sampler, asys, tstates, la


def regions_ref_of(asys):
    L = asys.box_vectors[0, 0]
    s = dict(N=asys.n_particles, sigma=np.asarray(asys.sigma), eps=np.asarray(asys.epsilon), mass=np.asarray(asys.masses),
             box=np.array([L, L, L]), rc=asys.cutoff, rs=asys.switching_distance)
    return RegionsReference(s, asys.alchemical_region_ids(), *[a for _, _, a in asys.alchemical_regions])


def test_replica_exchange_on_a_dual_topology_ladder_stores_and_resumes(tmp_path):
    """Through the public API: the stored energies equal the reference's on the device's positions, the suffixed states
    come back from storage, and a run interrupted after 3 iterations and resumed gives the same bits as the whole run."""
    from openmmtools_b200 import multistate, _backend
    from openmmtools_b200.multistate import MultiStateReporter
    a, asys, tstates, la = dual_sampler(iterations=4, storage=str(tmp_path / 'a.store'))
    a.run()
    u = a._energy_thermodynamic_states.copy()
    x = np.stack([st._positions for st in a.sampler_states])
    _, tab = _backend.engine_tables(tstates)
    betas = 1.0 / (KB * tab['temperature'])
    assert_close(u, regions_ref_of(asys).energy_matrix(x, la, 1.0 - la, betas, tab['energy_offset']))
    assert sorted(a._replica_thermodynamic_states) == list(range(len(la)))
    r = MultiStateReporter(str(tmp_path / 'a.store'), open_mode='r')
    assert np.array_equal(r.read_energies(4)[0], u)
    back, _ = r.read_thermodynamic_states()
    assert [t.lambda_sterics_A for t in back] == list(la) and [t.lambda_sterics_B for t in back] == list(1.0 - la)
    b, _, _, _ = dual_sampler(iterations=4, storage=str(tmp_path / 'b.store'))
    b.run(3)
    del b
    c = multistate.ReplicaExchangeSampler.from_storage(str(tmp_path / 'b.store'))
    assert c.iteration == 2
    c.run()
    assert np.array_equal(np.stack([st._positions for st in c.sampler_states]), x)
    assert np.array_equal(c._energy_thermodynamic_states, u)


def test_sams_with_device_weight_update_over_a_2d_grid():
    from openmmtools_b200 import testsystems, alchemy, states, mcmc, multistate, unit, _backend
    N, n_rep = 128, 4
    fluid = testsystems.LennardJonesFluid(nparticles=N)
    regions = [alchemy.AlchemicalRegion(alchemical_atoms=range(0, 4), name='A'),
               alchemy.AlchemicalRegion(alchemical_atoms=range(4, 8), name='B')]
    asys = alchemy.AbsoluteAlchemicalFactory().create_alchemical_system(fluid.system, regions)
    l1, l2 = grid(9)
    comp = [alchemy.AlchemicalState.from_system(asys, parameters_name_suffix=n) for n in ('A', 'B')]
    tstates = states.create_thermodynamic_state_protocol(
        asys, {'lambda_sterics_A': list(l1), 'lambda_sterics_B': list(l2)}, constants={'temperature': 300.0 * unit.kelvin},
        composable_states=comp)
    move = mcmc.LangevinSplittingDynamicsMove(timestep=1.0 * unit.femtosecond, n_steps=20)
    smp = multistate.SAMSSampler(mcmc_moves=move, number_of_iterations=10 ** 6, seed=99, device_weight_update=True,
                                 flatness_criteria='minimum-visits')
    sstate = states.SamplerState(fluid.positions, box_vectors=asys.getDefaultPeriodicBoxVectors())
    smp.create(tstates, [sstate] * n_rep)
    smp.run(6)
    smp.run_fused(4)
    u = smp._energy_thermodynamic_states.copy()
    x = smp._engine.get_positions()
    _, tab = _backend.engine_tables(tstates)
    assert_close(u, regions_ref_of(asys).energy_matrix(x, l1, l2, 1.0 / (KB * tab['temperature']), tab['energy_offset']))
    assert np.all(np.isfinite(smp._logZ)) and sum(smp._state_histogram) > 0


TWO_GPU_WORKER = r"""
import os, sys
sys.path.insert(0, %(root)r)
sys.path.insert(0, os.path.join(%(root)r, 'tests'))
import numpy as np
import torch.distributed as dist
dist.init_process_group('gloo')
from openmmtools_b200._dist import TorchCommunicator
from test_gpu_alchemical_regions import dual_sampler
s = dual_sampler(K=6, iterations=3, communicator=TorchCommunicator())[0]
s.run()
np.savez(%(out)r + '_%%d.npz' %% dist.get_rank(), u=s._energy_thermodynamic_states, perm=s._replica_thermodynamic_states,
         x=s._engine.get_positions(), k0=s._engine.k0)
dist.barrier()
"""


def test_two_gpus_reproduce_one(tmp_path):
    import os, subprocess, sys
    from test_multi_gpu import _two_devices, ROOT
    if not _two_devices():
        pytest.skip('needs 2 GPUs')
    s = dual_sampler(K=6, iterations=3)[0]
    s.run()
    u1, p1, x1 = s._energy_thermodynamic_states.copy(), s._replica_thermodynamic_states.copy(), s._engine.get_positions()
    script = tmp_path / 'g.py'
    out = str(tmp_path / 'res')
    script.write_text(TWO_GPU_WORKER % {'root': ROOT, 'out': out})
    r = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2',
                        '--master-addr', '127.0.0.1', '--master-port', '29541', str(script)],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    for rank in range(2):
        d = np.load(out + '_%d.npz' % rank)
        assert np.array_equal(d['perm'], p1) and np.array_equal(d['u'], u1)
        k0 = int(d['k0'])
        assert np.array_equal(d['x'], x1[k0:k0 + d['x'].shape[0]])
