"""Monte Carlo rigid-body moves on the device (rx_mc.cuh) against the host restatement of tests/mc_oracle.py, their
stationary distribution, and the samplers that run them before the Langevin steps."""
import os
import numpy as np
import pytest
import mc_oracle as mo
from helpers import KB, lj_setup, oracle_system, scattered_alch, waters, gpu_engine
from openmmtools_b200 import _lib, mcmc, unit, states, alchemy, testsystems, multistate

pytestmark = pytest.mark.gpu

SEED, IT = 0x1234_5678_9ABC, 7


def run_moves(eng, x, moves, seed=SEED, iteration=IT):
    """The moves of every state (list of (kind, sigma, subset)) once on every replica: zero dynamics steps."""
    eng.set_integrator(0.001, 1.0, 0, 'VRO')
    eng.set_positions(x)
    eng.set_velocities(np.zeros_like(x))
    eng.set_mc_moves(moves)
    eng.propagate(seed, iteration)
    return eng.get_positions(), eng.get_mc_statistics()


def replay(x, moves, perm, energy_of, betas, box_of=lambda k: None, store=np.float32):
    """The oracle's positions and decisions [K][slot] for the same draws."""
    out, dec = np.array(x, np.float64), []
    for k in range(len(x)):
        l, row = perm[k], []
        for j, (kind, sigma, subset) in enumerate(moves[l]):
            words, u = mo.draws(SEED, IT, k, j)
            out[k], yes, _ = mo.step(lambda y: energy_of(l, k, y), out[k], subset, kind, mo.proposal(kind, words, sigma), u,
                                     betas[l], box_of(k), store)
            row.append(yes)
        dec.append(row)
    return out, dec


def lj_engine(s, K, lambdas, T=300.0, two=None):
    M = len(lambdas)
    eng = gpu_engine(_lib.RX_SYSTEM_LJ_ALCH, K, M, s['N'], box=tuple(s['box']), r_cutoff=s['rc'], r_switch=s['rs'],
                     use_switch=True)
    eng.set_particles(s['sigma'], s['eps'], s['mass'], s['alch'])
    if two is not None:
        eng.set_alchemical_regions(two, False, False)
        eng.set_states([T] * M, lambda_sterics=lambdas, lambda_sterics_2=lambdas[::-1])
    else:
        eng.set_states([T] * M, lambda_sterics=lambdas)
    return eng


def configurations(s, K, spread=0.02, seed=3):
    rng = np.random.default_rng(seed)
    x = s['x'][None] + rng.normal(0.0, spread, (K, s['N'], 3))
    return (x - s['box'] * np.floor(x / s['box'])).astype(np.float32).astype(np.float64)


def check(xd, xo, dec, stats, moves, perm):
    assert np.abs(xd - xo).max() < 2e-6
    acc = np.zeros_like(stats[0]); prop = np.zeros_like(stats[1])
    for k, row in enumerate(dec):
        for j, yes in enumerate(row):
            prop[perm[k], j] += 1
            acc[perm[k], j] += yes
    assert np.array_equal(acc, stats[0]) and np.array_equal(prop, stats[1])


@pytest.mark.parametrize('case', ['compact', 'scattered', 'all-atoms', 'large'])
def test_lj_moves_match_oracle(case):
    N = 4096 if case == 'large' else 512
    s = lj_setup(N=N, n_alch=8, reduced_density=0.3 if case == 'large' else 0.05)
    K, lambdas = 8, [1.0, 0.8, 0.5, 0.2]
    sub = {'compact': np.arange(8), 'scattered': scattered_alch(N), 'all-atoms': np.arange(N), 'large': np.arange(8)}[case]
    sigma = 0.01 if case == 'all-atoms' else 0.05
    moves = [[(mo.DISPLACEMENT, sigma, sub), (mo.ROTATION, 0.0, sub), (mo.DISPLACEMENT, 2 * sigma, sub[:3])]] * 4
    moves[1] = moves[1][:1]     # the states carry different moves
    x = configurations(s, K)
    eng = lj_engine(s, K, lambdas)
    xd, stats = run_moves(eng, x, moves)
    osys = oracle_system(s)
    perm = np.arange(K) % 4
    xo, dec = replay(x, moves, perm, lambda l, k, y: osys.energy(y, lambdas[l])[0], np.full(4, 1.0 / (KB * 300.0)),
                     lambda k: s['box'])
    check(xd, xo, dec, stats, moves, perm)
    if case in ('scattered', 'all-atoms'):   # the whole-making rule rejects the rotations of a spread-out subset
        words = [mo.draws(SEED, IT, k, 1)[0] for k in range(K) if perm[k] != 1]
        assert all(not mo.propose(mo.ROTATION, x[0], sub, mo.proposal(mo.ROTATION, w), s['box'])[1] for w in words)
    if case == 'compact':
        assert 0 < stats[0].sum() < stats[1].sum()


def test_two_regions_and_npt_match_oracle():
    from regions_ref import RegionsReference
    s = lj_setup(N=512, n_alch=0)
    region = np.zeros(512, np.uint8); region[:5] = 1; region[5:9] = 2
    K, lambdas = 4, [1.0, 0.7, 0.4, 0.1]
    x = configurations(s, K)
    moves = [[(mo.DISPLACEMENT, 0.05, np.arange(5)), (mo.ROTATION, 0.0, np.arange(5, 9))]] * 4
    eng = lj_engine(s, K, lambdas, two=region)
    xd, stats = run_moves(eng, x, moves)
    ref = RegionsReference(s, region)
    xo, dec = replay(x, moves, np.arange(K), lambda l, k, y: ref.energy(y, lambdas[l], lambdas[::-1][l]),
                     np.full(4, 1.0 / (KB * 300.0)), lambda k: s['box'])
    check(xd, xo, dec, stats, moves, np.arange(K))
    # NPT: every replica in its own box
    eng = lj_engine(s, K, lambdas)
    eng.set_pressures(np.full(4, 0.0602214076), np.zeros(4))
    boxes = s['box'][None] * np.array([1.0, 1.02, 0.98, 1.05])[:, None]
    eng.set_boxes(boxes)
    xd, stats = run_moves(eng, x, moves)

    def energy(l, k, y):
        t = dict(s); t['box'] = boxes[k]
        return oracle_system(t).energy(y, lambdas[l])[0]
    xo, dec = replay(x, moves, np.arange(K), energy, np.full(4, 1.0 / (KB * 300.0)), lambda k: boxes[k])
    wrap = lambda y: y - boxes[:, None] * np.floor(y / boxes[:, None])   # (every replica in its own box)
    check(wrap(xd), wrap(xo), dec, stats, moves, np.arange(K))


@pytest.mark.parametrize('case', ['one-region', 'two-regions', 'npt'])
def test_kernel_energy_change_is_the_difference_of_energy_rows(case):
    """The dU k_mc_move takes its decision on (rx_get_mc_energy_changes) equals the change of the replica's own entry of
    rx_compute_energies, divided by beta, to 1e-10 relative: displacements (alchemical atoms, their pairs with the fluid in
    the soft core and the switch) and rotations of a compact triple.  At 1e9 K the states accept nearly every proposal, so
    each is compared; the lambdas still span the soft-core range."""
    s = lj_setup(N=512, n_alch=8)
    K, lambdas, T = 16, [1.0, 0.8, 0.5, 0.2], 1e9
    x = configurations(s, K)
    d = x[0] - x[0][0]
    d -= s['box'] * np.round(d / s['box'])
    triple = np.argsort(np.einsum('ij,ij->i', d, d))[:3]            # atom 0 and its two nearest neighbours
    region = None
    if case == 'two-regions':
        region = np.zeros(512, np.uint8); region[:4] = 1; region[4:8] = 2
    eng = lj_engine(s, K, lambdas, T=T, two=region)
    if case == 'npt':
        boxes = s['box'][None] * np.linspace(0.97, 1.04, K)[:, None]
        eng.set_pressures(np.full(4, 0.0602214076), np.zeros(4))
        eng.set_boxes(boxes)
        # every replica's positions inside its own box, in f32 as the propagation wraps them (so that it moves nothing)
        L, iL = boxes.astype(np.float32)[:, None], (1.0 / boxes).astype(np.float32)[:, None]
        x32 = x.astype(np.float32)
        x = (x32 - L * np.floor(x32 * iL)).astype(np.float32).astype(np.float64)
    eng.set_positions(x)
    u0 = eng.compute_energies()
    moves = [[(mo.DISPLACEMENT, 0.03, np.arange(8))], [(mo.ROTATION, 0.0, triple)]] * 2
    _, stats = run_moves(eng, x, moves)
    u1 = eng.compute_energies()
    du = eng.get_mc_energy_changes()
    beta = 1.0 / (KB * T)
    assert np.isnan(du[:, 1:]).all()
    compared = 0
    for k in range(K):
        l = k % 4
        assert np.isfinite(du[k, 0])
        if u1[k, l] != u0[k, l]:      # accepted
            row = (u1[k, l] - u0[k, l]) / beta
            assert abs(du[k, 0] - row) <= 1e-10 * max(abs(row), 1.0), (k, du[k, 0], row)
            compared += 1
    assert compared >= K - 2 and stats[0].sum() == compared
    assert np.abs(du[:, 0]).max() > 1.0      # (moves that change the energy by more than a kJ/mol)


def test_rotation_samples_the_boltzmann_distribution_of_a_rigid_pair():
    """MCRotationMove alone on a rigid LJ pair (0.4 nm) about its centre, next to a fixed third atom, with the pair across
    the periodic boundary (the subset is made whole by minimum image): the histogram of the nearer pair-atom distance to the
    third atom over independent replicas matches the Boltzmann integral over uniform rotations (chi-squared)."""
    from scipy.stats import chi2
    K, T, L, sig, eps = 4096, 300.0, 2.4, 0.34, 5.0
    rc, rs = 3 * sig, 2 * sig
    h, D = 0.2, 0.55
    c = np.array([0.02, 1.2, 1.2])
    x0 = np.array([c + [h, 0, 0], c - [h, 0, 0], c - [D, 0, 0]])
    x0 -= L * np.floor(x0 / L)                     # atom 1 and atom 2 wrap to the far side of the box
    eng = gpu_engine(_lib.RX_SYSTEM_LJ_ALCH, K, 1, 3, box=(L, L, L), r_cutoff=rc, r_switch=rs, use_switch=True)
    eng.set_particles(np.full(3, sig), np.full(3, eps), np.full(3, 40.0), np.zeros(3, np.uint8))
    eng.set_states([T], lambda_sterics=[1.0])
    eng.set_integrator(0.001, 1.0, 0, 'VRO')
    eng.set_positions(np.broadcast_to(x0, (K, 3, 3)).astype(np.float32).astype(np.float64).copy())
    eng.set_velocities(np.zeros((K, 3, 3)))
    eng.set_mc_moves([[(mo.ROTATION, 0.0, [0, 1])]])

    def nearer(x):
        r = [x[:, i] - x[:, 2] for i in (0, 1)]
        return np.minimum(*[np.linalg.norm(v - L * np.round(v / L), axis=-1) for v in r])
    samples, it = [], 1
    for _ in range(4):
        eng.run_iterations(25, None, 17, it)
        it += 25
        samples.append(nearer(eng.get_positions()))
    r = np.concatenate(samples)
    acc, prop = eng.get_mc_statistics()
    assert 0.2 < acc.sum() / prop.sum() < 0.95

    def lj(q):
        s6 = (sig / q) ** 6
        t = np.clip((q - rs) / (rc - rs), 0.0, 1.0)
        return 4 * eps * (s6 * s6 - s6) * (1.0 + t ** 3 * (-10.0 + t * (15.0 - 6.0 * t)))
    mu = (np.arange(1_000_000) + 0.5) / 1_000_000       # |cos| of the pair axis to the third atom: uniform under rotations
    near, far = np.sqrt(D * D + h * h - 2 * D * h * mu), np.sqrt(D * D + h * h + 2 * D * h * mu)
    w = np.exp(-(lj(near) + lj(far)) / (KB * T))
    edges = np.linspace(D - h, np.sqrt(D * D + h * h), 11)
    p = np.histogram(near, edges, weights=w)[0] / w.sum()
    obs = np.histogram(r, edges)[0]
    assert obs.sum() == len(r)
    stat = np.sum((obs - len(r) * p) ** 2 / (len(r) * p))
    assert chi2.sf(stat, len(p) - 1) > 1e-3, (stat, obs, len(r) * p)
    # the rotation changes the distribution away from the uniform-rotation one (the test can tell them apart)
    p0 = np.histogram(near, edges)[0] / len(near)
    assert chi2.sf(np.sum((obs - len(r) * p0) ** 2 / (len(r) * p0)), len(p) - 1) < 1e-6


def test_rigid_water_and_toluene_match_oracle():
    from oracle import oracle, implicit
    from implicit_helpers import implicit_system
    sysw, xw = waters(10)
    sub = np.array([3, 4, 5])
    for system, x0, subset, make in ((sysw, xw, sub, oracle.Molecule),
                                     implicit_system('toluene') + (None, implicit.Molecule)):
        N = system.n_particles
        subset = np.arange(N) if subset is None else subset
        K = 4
        eng = gpu_engine(_lib.RX_SYSTEM_MOLECULE, K, 2, N)
        eng.set_molecule(system)
        eng.set_states([300.0, 400.0])
        rng = np.random.default_rng(1)
        x = np.stack([x0 + rng.normal(0, 0.02, 3) for _ in range(K)])
        moves = [[(mo.DISPLACEMENT, 0.05, subset), (mo.ROTATION, 0.0, subset)]] * 2
        xd, stats = run_moves(eng, x, moves)
        om = make(system)
        xo, dec = replay(x, moves, np.arange(K) % 2, lambda l, k, y: om.energy(y), 1.0 / (KB * np.array([300.0, 400.0])),
                         store=np.float64)
        check(xd, xo, dec, stats, moves, np.arange(K) % 2)
        for i, j, d in system.constraints:     # rigid moves of whole clusters keep every constraint
            r = np.linalg.norm(xd[:, int(i)] - xd[:, int(j)], axis=-1)
            assert np.abs(r - np.linalg.norm(x[:, int(i)] - x[:, int(j)], axis=-1)).max() < 1e-10


def test_subsets_are_validated():
    sysw, xw = waters(3)
    eng = gpu_engine(_lib.RX_SYSTEM_MOLECULE, 2, 1, 9)
    eng.set_molecule(sysw)
    eng.set_states([300.0])
    with pytest.raises(Exception) as e:
        eng.set_mc_moves([[(mo.ROTATION, 0.0, [0, 1])]])       # half a water
    assert e.value.code == _lib.RX_ERR_UNSUPPORTED
    for bad in ([(mo.DISPLACEMENT, -1.0, [0, 1, 2])], [(mo.DISPLACEMENT, np.inf, [0, 1, 2])], [(mo.ROTATION, 0.0, [0, 1, 9])],
                [(mo.ROTATION, 0.0, [0, 1, 2, 2])], [(mo.ROTATION, 0.0, [0, 1, 2])] * 5):
        with pytest.raises(Exception) as e:
            eng.set_mc_moves([bad])
        assert e.value.code == _lib.RX_ERR_INVALID
    eng.set_mc_moves([[(mo.ROTATION, 0.0, [3, 4, 5, 0, 1, 2])]])


@pytest.mark.parametrize('sigma_factor', [0.3, 1.0, 3.0])
def test_displacement_samples_the_harmonic_boltzmann_distribution(sigma_factor):
    """MCDisplacementMove alone on a harmonic well: per-axis mean x0 and variance kT/K, within 5 sigma of the sampling
    error of independent replicas."""
    K, T, Kf, x0 = 4096, 300.0, 500.0, np.array([0.1, -0.2, 0.3])
    kT = KB * T
    eng = gpu_engine(_lib.RX_SYSTEM_HARMONIC, K, 1, 1)
    eng.set_particles(None, None, np.array([10.0]), None)
    eng.set_states([T], ho_K=[Kf], ho_x0=[x0])
    eng.set_integrator(0.001, 1.0, 0, 'VRO')
    eng.set_positions(np.broadcast_to(x0, (K, 1, 3)).copy())
    eng.set_velocities(np.zeros((K, 1, 3)))
    eng.set_mc_moves([[(mo.DISPLACEMENT, sigma_factor * np.sqrt(kT / Kf), [0])]])
    eng.run_iterations(300, None, 99, 1)
    x = eng.get_positions()[:, 0]
    var = kT / Kf
    assert np.all(np.abs(x.mean(0) - x0) < 5 * np.sqrt(var / K))
    assert np.all(np.abs(x.var(0) - var) < 5 * var * np.sqrt(2.0 / K))


def yank_sampler(tmp, seed=11, n_steps=20, K=8, **kw):
    fluid = testsystems.LennardJonesFluid(nparticles=128)
    ligand = list(range(4))
    asys = alchemy.AbsoluteAlchemicalFactory(disable_alchemical_dispersion_correction=True).create_alchemical_system(
        fluid.system, alchemy.AlchemicalRegion(alchemical_atoms=ligand))
    lambdas = [1.0 - l / (K - 1) for l in range(K)]
    tstates = states.create_thermodynamic_state_protocol(
        asys, {'lambda_sterics': lambdas}, constants={'temperature': 300.0 * unit.kelvin},
        composable_states=alchemy.AlchemicalState.from_system(asys))
    sstate = states.SamplerState(fluid.positions, box_vectors=asys.getDefaultPeriodicBoxVectors())
    move = mcmc.SequenceMove([mcmc.MCDisplacementMove(displacement_sigma=0.05 * unit.nanometer, atom_subset=ligand),
                              mcmc.MCRotationMove(atom_subset=ligand),
                              mcmc.LangevinSplittingDynamicsMove(timestep=2.0 * unit.femtosecond, n_steps=n_steps)])
    s = multistate.ReplicaExchangeSampler(mcmc_moves=move, number_of_iterations=6, seed=seed, **kw)
    storage = None if tmp is None else multistate.MultiStateReporter(os.path.join(str(tmp), 'run'), checkpoint_interval=2)
    s.create(tstates, [sstate], storage=storage)
    return s


def test_sampler_runs_the_sequence_fused_and_phase_by_phase_alike(tmp_path):
    a, b = yank_sampler(None), yank_sampler(None)
    a.run(3)
    b._compute_energies()
    b._engine.run_iterations(3, 'swap-all', b._seed, 1)
    for f in ('get_replica_states', 'get_energies', 'get_positions', 'get_mc_statistics'):
        ra, rb = getattr(a._engine, f)(), getattr(b._engine, f)()
        assert all(np.array_equal(p, q) for p, q in zip(ra, rb)) if isinstance(ra, tuple) else np.array_equal(ra, rb), f
    # the statistics the move objects carry are the device counts, state by state
    a._pull_mc_statistics()
    acc, prop = a._engine.get_mc_statistics()
    assert prop[:, :2].sum() == 2 * 3 * 8 and prop[:, 2:].sum() == 0
    for l, mv in enumerate(a._mcmc_moves):
        assert [st for st in mv.statistics[:2]] == [dict(n_accepted=int(acc[l, j]), n_proposed=int(prop[l, j])) for j in range(2)]
    assert len({tuple(mv.statistics[0].values()) for mv in a._mcmc_moves}) > 1


def test_stored_run_resumes_bit_for_bit(tmp_path):
    a = yank_sampler(tmp_path / 'a')
    a.run(6)
    b = yank_sampler(tmp_path / 'b')
    b.run(4)
    b._reporter.close()
    del b
    c = multistate.ReplicaExchangeSampler.from_storage(multistate.MultiStateReporter(os.path.join(str(tmp_path / 'b'), 'run')))
    assert c.iteration == 4
    c.run(2)
    assert np.array_equal(a._engine.get_positions(), c._engine.get_positions())
    assert np.array_equal(a._engine.get_mc_statistics()[1], c._engine.get_mc_statistics()[1])
    stored = multistate.MultiStateReporter(os.path.join(str(tmp_path / 'a'), 'run'), open_mode='r').read_mcmc_moves()
    acc, prop = a._engine.get_mc_statistics()
    assert stored[0].statistics[0] == dict(n_accepted=int(acc[0, 0]), n_proposed=int(prop[0, 0]))


def test_sams_runs_the_sequence_on_the_device():
    fluid = testsystems.LennardJonesFluid(nparticles=128)
    asys = alchemy.AbsoluteAlchemicalFactory(disable_alchemical_dispersion_correction=True).create_alchemical_system(
        fluid.system, alchemy.AlchemicalRegion(alchemical_atoms=range(4)))
    tstates = states.create_thermodynamic_state_protocol(
        asys, {'lambda_sterics': [1.0, 0.6, 0.3, 0.0]}, constants={'temperature': 300.0 * unit.kelvin},
        composable_states=alchemy.AlchemicalState.from_system(asys))
    move = mcmc.SequenceMove([mcmc.MCDisplacementMove(displacement_sigma=0.02 * unit.nanometer, atom_subset=[0, 1, 2, 3]),
                              mcmc.LangevinSplittingDynamicsMove(timestep=2.0 * unit.femtosecond, n_steps=10)])
    s = multistate.SAMSSampler(mcmc_moves=move, number_of_iterations=10, seed=3, device_weight_update=True)
    s.create(tstates, [states.SamplerState(fluid.positions, box_vectors=asys.getDefaultPeriodicBoxVectors())] * 4)
    s.run_fused(5)
    acc, prop = s._engine.get_mc_statistics()
    assert prop[:, 0].sum() == 5 * 4 and 0 < acc.sum() <= prop.sum()


def test_nan_retry_reruns_the_dynamics_from_the_post_mc_state():
    """A replica that fails goes back to the snapshot rx_propagate took after the Monte Carlo moves: the retry keeps the
    moved positions and does not repeat (or count) the moves."""
    from openmmtools_b200._engine import EngineError
    s = lj_setup(N=512, n_alch=8)
    K, lambdas = 4, [1.0, 0.8, 0.5, 0.2]
    x = configurations(s, K)
    moves = [[(mo.DISPLACEMENT, 0.002, np.arange(8)), (mo.ROTATION, 0.0, np.arange(8))]] * 4
    xt, st = run_moves(lj_engine(s, K, lambdas), x, moves)
    eng = lj_engine(s, K, lambdas)
    eng.set_integrator(0.001, 1.0, 0, 'VRO')
    eng.set_positions(x)
    v = np.zeros_like(x)
    v[1] = np.nan
    eng.set_velocities(v)
    eng.set_mc_moves(moves)
    with pytest.raises(EngineError) as e:
        eng.propagate(SEED, IT)
    assert e.value.nan_flags.tolist() == [0, 1, 0, 0]
    eng.propagate_retry(SEED + 1, IT, reassign_velocities=True)
    assert np.array_equal(eng.get_positions(), xt)
    assert all(np.array_equal(a, b) for a, b in zip(eng.get_mc_statistics(), st))
    assert st[0].sum() > 0


def test_no_launch_without_mc_moves():
    s = lj_setup(N=256, n_alch=4)
    eng = lj_engine(s, 4, [1.0, 0.5, 0.2, 0.0])
    eng.set_integrator(0.001, 1.0, 5, 'VRORV')
    eng.set_positions(configurations(s, 4))
    eng.set_velocities(np.zeros((4, 256, 3)))
    eng.phase_times(reset=True)
    eng.propagate(1, 1)
    assert eng.phase_times()['launches_by_phase'][1] == 1
    eng.set_mc_moves([[(mo.ROTATION, 0.0, [0, 1, 2])], [], [], []])
    eng.phase_times(reset=True)
    eng.propagate(1, 2)
    assert eng.phase_times()['launches_by_phase'][1] == 2
    eng.set_mc_moves([[]] * 4)
    eng.phase_times(reset=True)
    eng.propagate(1, 3)
    assert eng.phase_times()['launches_by_phase'][1] == 1


def test_single_replica_apply_updates_statistics():
    fluid = testsystems.LennardJonesFluid(nparticles=128)
    ts = states.ThermodynamicState(fluid.system, 300.0 * unit.kelvin)
    ss = states.SamplerState(fluid.positions, box_vectors=fluid.system.getDefaultPeriodicBoxVectors())
    move = mcmc.SequenceMove([mcmc.MCDisplacementMove(displacement_sigma=0.01 * unit.nanometer, atom_subset=[0]),
                              mcmc.LangevinSplittingDynamicsMove(n_steps=5)])
    move.apply(ts, ss)
    move.apply(ts, ss)
    assert move.statistics[0]['n_proposed'] == 2
    m = mcmc.MCRotationMove(atom_subset=[0, 1])
    m.apply(ts, ss)
    assert m.n_proposed == 1
