"""The Monte Carlo barostat of k_propagate beyond one launch of an identity replica->state map: replicas in other states
than their own index (the state's lambda, kT, pressure and dispersion, the replica's box, barostat record and Philox
stream), the step-size adaptation, launches that split the 25-step interval, per-state moves, the NPT instantiations of
every (C6, SW) pair and layout, k_energy_rows<NPT> above 1024 atoms and 512 states, k_minimize<APT = 4, NPT> and two
ranks.  The oracle is the f64 one of test_gpu_npt.py (oracle/npt.py), fed with the device's noise and uniforms.

Every engine here has at least as many states as replicas."""
import os
import subprocess
import sys
import numpy as np
import pytest
from helpers import lj_setup, oracle_system, gpu_engine, device_noise, device_reassign_noise, min_image, wrap, KB
from test_gpu_npt import barostat_uniforms, cluster_width, npt_sampler
from test_gpu_propagate import mixed
from test_npt_host import BAR
from oracle import npt as onpt

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RTOL = 1e-10
SEED = 0x1234567890ABCDEF


def engine(s, K, M, lambdas, temps, pressures, disp, eps=None, use_switch=True, softcore_c=6.0, annihilate=False):
    e = gpu_engine(1, K, M, s['N'], box=tuple(s['box']), r_cutoff=s['rc'], r_switch=s['rs'], use_switch=use_switch,
                   softcore_c=softcore_c, annihilate_sterics=annihilate)
    e.set_particles(s['sigma'], s['eps'] if eps is None else eps, s['mass'], s['alch'])
    e.set_states(temps, lambdas)
    e.set_pressures(pressures, disp)
    return e


class Replica:
    """One replica on the oracle: f64 positions (unwrapped), velocities, box and Barostat record, carried from launch to
    launch."""

    def __init__(self, x, v, box, volume_scale, step=0, n_attempted=0, n_accepted=0):
        self.x, self.v, self.box = np.array(x, np.float64), np.array(v, np.float64), np.array(box, np.float64)
        self.st = onpt.barostat_state(volume_scale, step, n_attempted, n_accepted)

    def launch(self, osys, seed, iteration, k, n_steps, lam, kT, pressure, dispersion, dt, gamma, program='VRORV',
               reassign_mass=None):
        """One launch of replica k (its noise, its uniforms (seed, iteration, k, a), a = 0, 1, ... restarting here).
        reassign_mass: velocities drawn first from the device's reassignment normals at kT.  Returns (decisions,
        potential, the step of the launch whose start took the first attempt or None)."""
        N = len(self.x)
        if reassign_mass is not None:
            self.v = np.sqrt(kT / reassign_mass)[:, None] * device_reassign_noise(seed, iteration, k, N)
        first = (24 - self.st.step) if n_steps > 24 - self.st.step else None
        n_max = n_steps // 25 + 1
        uni = np.array([barostat_uniforms(seed, iteration, k, a) for a in range(n_max)]).ravel()
        noise = device_noise(seed, iteration, k, N, n_steps * program.count('O'))
        dec, U = onpt.langevin(osys, self.x, self.v, noise, self.box, self.st, uni, lam, kT, dt, gamma, n_steps, pressure,
                               dispersion, min_edge=2 * osys.p.r_cutoff, program=program)
        return dec, U, first


def device_state(e):
    return dict(x=e.get_positions(), v=e.get_velocities(), box=e.get_boxes(), baro=e.get_barostat(),
                pot=e.get_replica_energies()[0])


def assert_replica(dev, k, rep, U, what=''):
    """The device's replica k against the oracle's: counters exactly, box 1e-12, volume_scale 1e-15, positions 2e-5 nm
    (minimum image), velocities 2e-4 nm/ps, potential 1e-3 relative."""
    b = dev['baro']
    tag = (what, k)
    assert (b['step'][k], b['n_attempted'][k], b['n_accepted'][k]) == (rep.st.step, rep.st.n_attempted, rep.st.n_accepted), \
        (tag, {f: b[f][k] for f in b}, (rep.st.step, rep.st.n_attempted, rep.st.n_accepted, rep.st.volume_scale))
    assert b['volume_scale'][k] == pytest.approx(rep.st.volume_scale, rel=1e-15, abs=0), (tag, b['volume_scale'][k], rep.st.volume_scale)
    assert np.allclose(dev['box'][k], rep.box, rtol=1e-12, atol=0), (tag, dev['box'][k], rep.box)
    dx = np.abs(min_image(dev['x'][k] - wrap(rep.x, rep.box), rep.box)).max()
    assert dx < 2e-5, (tag, dx)
    assert np.abs(dev['v'][k] - rep.v).max() < 2e-4, (tag, np.abs(dev['v'][k] - rep.v).max())
    assert abs(dev['pot'][k] - U) < 1e-3 * max(1.0, abs(U)), (tag, dev['pot'][k], U)


def assert_energy_matrix(u, osys, x, boxes, lambdas, temps, pressures, disp):
    ref = onpt.energy_matrix(osys, x, boxes, lambdas, 1.0 / (KB * np.asarray(temps)), pressures, disp)
    assert (np.abs(u - ref) / np.maximum(1.0, np.abs(ref))).max() <= RTOL


def start_velocities(K, N, seed=2):
    return np.random.default_rng(seed).normal(scale=0.25, size=(K, N, 3)).astype(np.float32).astype(np.float64)


# ---- 1. replicas in states other than their own index ----------------------------------------------------------------
@pytest.mark.parametrize('cl', [1, 4])
def test_swapped_replicas_take_the_state_parameters_and_keep_their_box(cl):
    """K = 4 replicas over M = 6 states (each its own T, lambda, p, c) in the map [4, 0, 5, 2], then in another map under
    the next iteration: the oracle runs replica k with state perm[k]'s parameters and replica k's noise, uniforms, box and
    barostat record, which stay with the replica when its state changes."""
    N, K, M = 512, 4, 6
    s = lj_setup(N=N, n_alch=6, seed=11)
    lambdas = np.array([1.0, 0.8, 0.6, 0.45, 0.3, 0.0])
    temps = np.array([300.0, 315.0, 330.0, 345.0, 290.0, 360.0])
    pressures = np.array([30.0, 150.0, 45.0, 400.0, 60.0, 5.0]) * BAR
    disp = np.array([-30.0, -12.0, -25.0, -40.0, -20.0, -15.0])
    maps = [np.array([4, 0, 5, 2]), np.array([1, 3, 0, 5])]
    dt, gamma, n_steps, it0 = 0.002, 10.0, 75, 7
    e = engine(s, K, M, lambdas, temps, pressures, disp)
    e.set_integrator(dt, gamma, n_steps, 'V R O R V')
    x0, v0 = np.stack([s['x']] * K), start_velocities(K, N)
    e.set_positions(x0); e.set_velocities(v0)
    st0 = e.get_barostat()
    vs0 = st0['volume_scale'] * 3.0
    st0['volume_scale'] = vs0
    e.set_barostat(st0)
    osys = oracle_system(s)
    reps = [Replica(x0[k], v0[k], s['box'], vs0[k]) for k in range(K)]
    decisions = []
    with cluster_width(cl):
        for j, perm in enumerate(maps):
            e.set_replica_states(perm)
            e.propagate(SEED, it0 + j)
            dev = device_state(e)
            for k in range(K):
                l = perm[k]
                dec, U, _ = reps[k].launch(osys, SEED, it0 + j, k, n_steps, lambdas[l], KB * temps[l], pressures[l],
                                           disp[l], dt, gamma)
                assert len(dec) == 3
                decisions += dec
                assert_replica(dev, k, reps[k], U, 'launch %d' % j)
    assert np.array_equal(e.get_replica_states(), maps[-1])
    u = e.compute_energies()
    xg, bg = e.get_positions(), e.get_boxes()
    e.close()
    assert 1 in decisions and 0 in decisions, decisions
    assert_energy_matrix(u, osys, xg, bg, lambdas, temps, pressures, disp)
    # control: with the identity map's parameters the first launch ends differently for some replica
    differs = False
    for k in range(K):
        a, b = Replica(x0[k], v0[k], s['box'], vs0[k]), Replica(x0[k], v0[k], s['box'], vs0[k])
        l = maps[0][k]
        da = a.launch(osys, SEED, it0, k, n_steps, lambdas[l], KB * temps[l], pressures[l], disp[l], dt, gamma)[0]
        db = b.launch(osys, SEED, it0, k, n_steps, lambdas[k], KB * temps[k], pressures[k], disp[k], dt, gamma)[0]
        differs |= da != db or not np.array_equal(a.box, b.box)
    assert differs, 'the identity map gives the same boxes and decisions: the test cannot tell the maps apart'


# ---- 2. step-size adaptation -----------------------------------------------------------------------------------------
def fluid_states(ideal, K):
    """(lambdas, temps, pressures, dispersion): the ideal gas gets K identical states."""
    if ideal:
        return np.ones(K), np.full(K, 300.0), None, np.zeros(K)
    return (np.linspace(1.0, 0.0, K), np.linspace(300.0, 330.0, K), np.linspace(30.0, 80.0, K) * BAR,
            np.linspace(-30.0, -15.0, K))


def adaptation_run(ideal, records, n_steps, it=3):
    """K = len(records) replicas of the 512-atom fluid (epsilon = 0 for the ideal gas, so that dU = 0 and the decisions
    depend on the uniforms alone) from the given barostat records, one launch, against the oracle."""
    N, K = 512, len(records)
    s = lj_setup(N=N, n_alch=6, seed=11)
    V0 = float(np.prod(s['box']))
    lambdas, temps, pressures, disp = fluid_states(ideal, K)
    if ideal:
        pressures = np.full(K, (N + 1) * KB * 300.0 / V0)    # the box is the ideal gas's mean volume
    eps = np.zeros(N) if ideal else s['eps']
    dt, gamma = 0.002, 10.0
    e = engine(s, K, K, lambdas, temps, pressures, disp, eps=eps)
    e.set_integrator(dt, gamma, n_steps, 'V R O R V')
    x0, v0 = np.stack([s['x']] * K), start_velocities(K, N)
    e.set_positions(x0); e.set_velocities(v0)
    rec = {f: np.array([r[f] for r in records]) for f in ('volume_scale', 'step', 'n_attempted', 'n_accepted')}
    rec['volume_scale'] = rec['volume_scale'] * V0
    e.set_barostat(rec)
    e.propagate(SEED, it)
    dev = device_state(e)
    e.close()
    osys = oracle_system(dict(s, eps=eps))
    reps, decisions = [], []
    for k in range(K):
        rep = Replica(x0[k], v0[k], s['box'], rec['volume_scale'][k], rec['step'][k], rec['n_attempted'][k],
                      rec['n_accepted'][k])
        dec, U, _ = rep.launch(osys, SEED, it, k, n_steps, lambdas[k], KB * temps[k], pressures[k], disp[k], dt, gamma)
        assert_replica(dev, k, rep, U)
        reps.append(rep)
        decisions += dec
    return reps, decisions, rec['volume_scale'], V0


@pytest.mark.parametrize('ideal', [True, False], ids=['ideal-gas', 'interacting'])
def test_step_size_adaptation_at_the_tenth_attempt(ideal):
    """Records one attempt short of ten, 75 steps (three attempts, the first the tenth): 0 of 9 accepted shrinks
    volume_scale by 1.1, 9 of 9 grows it by 1.1, 9 of 9 from 0.29 V grows it to the cap 0.3 V (V before the move), 5 of
    9 keeps it and does not reset the counters."""
    records = [dict(volume_scale=0.05, step=0, n_attempted=9, n_accepted=0),
               dict(volume_scale=0.05, step=0, n_attempted=9, n_accepted=9),
               dict(volume_scale=0.29, step=0, n_attempted=9, n_accepted=9),
               dict(volume_scale=0.05, step=0, n_attempted=9, n_accepted=5)]
    reps, decisions, vs0, V0 = adaptation_run(ideal, records, 75)
    assert 1 in decisions and 0 in decisions, decisions
    shrink, grow, cap, keep = (r.st for r in reps)
    assert shrink.volume_scale == pytest.approx(vs0[0] / 1.1, rel=1e-15) and shrink.n_attempted == 2
    assert grow.volume_scale == pytest.approx(vs0[1] * 1.1, rel=1e-15) and grow.n_attempted == 2
    assert cap.volume_scale == pytest.approx(0.3 * V0, rel=1e-15) and cap.volume_scale < vs0[2] * 1.1 and cap.n_attempted == 2
    assert keep.volume_scale == vs0[3] and keep.n_attempted == 12


@pytest.mark.parametrize('ideal', [True, False], ids=['ideal-gas', 'interacting'])
def test_step_size_adaptation_inside_one_launch(ideal):
    """250 steps from fresh records are ten attempts: tiny moves (nearly all accepted) grow volume_scale and large ones
    (mostly rejected) shrink it, both at the last attempt of the launch, which resets the counters."""
    records = [dict(volume_scale=1e-4, step=0, n_attempted=0, n_accepted=0),
               dict(volume_scale=0.29, step=0, n_attempted=0, n_accepted=0),
               dict(volume_scale=2e-4, step=0, n_attempted=0, n_accepted=0),
               dict(volume_scale=0.25, step=0, n_attempted=0, n_accepted=0)]
    reps, decisions, vs0, _ = adaptation_run(ideal, records, 250, it=11)
    assert len(decisions) == 40 and 1 in decisions and 0 in decisions
    outcomes = ['grow' if r.st.volume_scale > v else 'shrink' if r.st.volume_scale < v else 'keep'
                for r, v in zip(reps, vs0)]
    assert {'grow', 'shrink'} <= set(outcomes), outcomes
    for r, o in zip(reps, outcomes):
        assert (r.st.n_attempted == 0) == (o != 'keep'), (o, r.st.n_attempted)


# ---- 3. launches that split the 25-step interval ---------------------------------------------------------------------
def test_launches_that_split_the_barostat_interval():
    """Launches of 40, 10, 1, 24 and 25 steps under consecutive iterations, replicas starting at step 0, 24, 7 and 13:
    the step counter carries over from launch to launch (exactly), the attempt counter of the Philox stream restarts in
    every launch, one replica attempts before its first step and some launch makes no attempt."""
    N, K, M = 512, 4, 5
    s = lj_setup(N=N, n_alch=6, seed=11)
    lambdas, temps = np.array([1.0, 0.7, 0.5, 0.2, 0.0]), np.array([300.0, 310.0, 320.0, 330.0, 340.0])
    pressures, disp = np.array([30.0, 45.0, 60.0, 80.0, 100.0]) * BAR, np.array([-30.0, -25.0, -20.0, -15.0, -10.0])
    perm = np.array([1, 3, 0, 4])
    dt, gamma, it0 = 0.002, 10.0, 20
    e = engine(s, K, M, lambdas, temps, pressures, disp)
    x0, v0 = np.stack([s['x']] * K), start_velocities(K, N)
    e.set_positions(x0); e.set_velocities(v0)
    e.set_replica_states(perm)
    st0 = e.get_barostat()
    st0['volume_scale'] = st0['volume_scale'] * 3.0
    st0['step'] = np.array([0, 24, 7, 13])
    e.set_barostat(st0)
    osys = oracle_system(s)
    reps = [Replica(x0[k], v0[k], s['box'], st0['volume_scale'][k], st0['step'][k]) for k in range(K)]
    decisions, counts, firsts = [], [], []
    for j, n_steps in enumerate([40, 10, 1, 24, 25]):
        e.set_integrator(dt, gamma, n_steps, 'V R O R V')
        e.propagate(SEED, it0 + j)
        dev = device_state(e)
        for k in range(K):
            l = perm[k]
            dec, U, first = reps[k].launch(osys, SEED, it0 + j, k, n_steps, lambdas[l], KB * temps[l], pressures[l],
                                           disp[l], dt, gamma)
            assert dev['baro']['step'][k] == reps[k].st.step
            assert_replica(dev, k, reps[k], U, 'launch %d' % j)
            decisions += dec
            counts.append(len(dec))
            firsts.append(first)
    e.close()
    assert 1 in decisions and 0 in decisions, decisions
    assert 0 in counts and max(counts) >= 2, counts
    assert 0 in firsts, 'no attempt before the first step of a launch'


# ---- 4. per-state moves under NPT ------------------------------------------------------------------------------------
A = (0.002, 1.0, 40, 'V R O R V', False)
B = (0.001, 5.0, 60, 'O V R V O', True)


@pytest.mark.parametrize('N,cl', [(256, None), (2048, 2), (2048, 8)])
def test_per_state_moves_under_constant_pressure(N, cl):
    """One move per state (Layout<1, true, false> at 256 atoms, the compact per-state layouts at 2048) with the barostat:
    states 0, 1 run move A (40 steps, one attempt), states 2, 3 move B (60 steps, two attempts, velocities reassigned).
    Each replica comes out bit for bit as from an engine where every state has its move -- positions, velocities, box and
    barostat record -- and one replica of each move matches the oracle."""
    K = 4
    s = lj_setup(N=N, n_alch=8, seed=61)
    lambdas, temps = np.array([1.0, 0.7, 0.3, 0.0]), np.array([300.0, 320.0, 340.0, 360.0])
    pressures, disp = np.array([20.0, 50.0, 80.0, 110.0]) * BAR, np.array([-30.0, -25.0, -20.0, -15.0])
    v0 = start_velocities(K, N, 16)
    perm = np.array([2, 0, 3, 1])
    seed, it = 77, 3

    def run(moves):
        e = engine(s, K, K, lambdas, temps, pressures, disp)
        e.set_integrator(*moves[0][:4])
        single = all(m == moves[0] for m in moves)
        if not single:
            for l, m in enumerate(moves):
                e.set_state_integrator(l, *m)
        e.set_positions(np.stack([s['x']] * K)); e.set_velocities(v0)
        e.set_replica_states(perm)
        st = e.get_barostat()
        st['volume_scale'] = st['volume_scale'] * 3.0
        e.set_barostat(st)
        with cluster_width(cl):
            e.propagate(seed, it, moves[0][4] if single else False)
        out = device_state(e)
        e.close()
        return out
    m, a, b = run([A, A, B, B]), run([A] * 4), run([B] * 4)
    for k in range(K):
        ref = a if perm[k] < 2 else b
        for f in ('x', 'v', 'box'):
            assert np.array_equal(m[f][k], ref[f][k]), (k, f)
        assert all(m['baro'][f][k] == ref['baro'][f][k] for f in m['baro']), (k, m['baro'], ref['baro'])
        assert np.isclose(m['pot'][k], ref['pot'][k], rtol=1e-12, atol=1e-9), k
    assert not np.array_equal(a['x'][0], b['x'][0])
    assert m['baro']['step'][1] == 15 and m['baro']['step'][0] == 10      # A: 40 steps, B: 60 steps from step 0
    assert m['baro']['n_attempted'][1] == 1 and m['baro']['n_attempted'][0] == 2
    osys = oracle_system(s)
    vs0 = 3.0 * 0.01 * np.prod(s['box'])
    for k in (1, 0):                      # state 0 (move A), state 2 (move B)
        l = perm[k]
        dt, gamma, n_steps, prog, reassign = A if l < 2 else B
        rep = Replica(s['x'], v0[k], s['box'], vs0)
        dec, U, _ = rep.launch(osys, seed, it, k, n_steps, lambdas[l], KB * temps[l], pressures[l], disp[l], dt, gamma,
                               prog.replace(' ', ''), s['mass'] if reassign else None)
        assert_replica(m, k, rep, U, 'move %s' % ('A' if l < 2 else 'B'))


# ---- 5. every NPT instantiation against the oracle -------------------------------------------------------------------
VARIANTS = [
    pytest.param(512, False, dict(use_switch=False), 1, id='no-switch-cl1'),
    pytest.param(512, False, dict(softcore_c=4.0), 2, id='softcore-c4-cl2'),
    pytest.param(512, False, dict(annihilate=True), 4, id='annihilate-cl4'),
    pytest.param(257, True, {}, 4, id='mixed-rect-257-cl4'),
    pytest.param(1025, False, {}, 4, id='compact-1025-cl4'),
    pytest.param(4096, False, {}, 8, id='compact-4096-cl8', marks=pytest.mark.slow),
]


@pytest.mark.parametrize('N,mixed_types,kw,cl', VARIANTS)
def test_npt_variants_match_oracle(N, mixed_types, kw, cl):
    """75 steps (three attempts) of the interacting fluid in each pair-kernel variant and layout: no switch, soft-core
    c = 4, annihilated sterics, three atom types in a rectangular box with a short last warp, a ragged compact cluster at
    1025 atoms and the only compact width at 4096; then the energy matrix at the replicas' boxes."""
    K = 4
    s = mixed(N, seed=N) if mixed_types else lj_setup(N=N, n_alch=6, seed=11)
    if kw.get('annihilate'):     # alchemical atoms close to each other, so that the A-A pairs are within the cutoff
        s['alch'][:] = 0
        d = np.linalg.norm(min_image(s['x'] - s['x'][0], s['box']), axis=1)
        s['alch'][np.argsort(d)[:8]] = 1
    lambdas, temps = np.array([1.0, 0.6, 0.3, 0.0]), np.array([300.0, 310.0, 320.0, 330.0])
    pressures, disp = np.array([30.0, 45.0, 60.0, 80.0]) * BAR, np.array([-30.0, -25.0, -20.0, -15.0])
    dt, gamma, n_steps, it = 0.002, 10.0, 75, 7
    e = engine(s, K, K, lambdas, temps, pressures, disp, **kw)
    e.set_integrator(dt, gamma, n_steps, 'V R O R V')
    x0, v0 = np.stack([s['x']] * K), start_velocities(K, N)
    e.set_positions(x0); e.set_velocities(v0)
    st0 = e.get_barostat()
    st0['volume_scale'] = st0['volume_scale'] * 3.0
    e.set_barostat(st0)
    with cluster_width(cl):
        e.propagate(SEED, it)
    dev = device_state(e)
    u = e.compute_energies()
    e.close()
    osys = oracle_system(s, annihilate=kw.get('annihilate', False), c=kw.get('softcore_c', 6.0),
                         use_switch=kw.get('use_switch', True))
    decisions = []
    for k in range(K):
        rep = Replica(x0[k], v0[k], s['box'], st0['volume_scale'][k])
        dec, U, _ = rep.launch(osys, SEED, it, k, n_steps, lambdas[k], KB * temps[k], pressures[k], disp[k], dt, gamma)
        assert len(dec) == 3
        decisions += dec
        assert_replica(dev, k, rep, U)
    assert 1 in decisions and 0 in decisions, decisions
    assert_energy_matrix(u, osys, dev['x'], dev['box'], lambdas, temps, pressures, disp)


@pytest.mark.parametrize('N', [1025, 2048])
def test_energy_matrix_of_600_states_at_per_replica_boxes(N):
    """k_energy_rows<NPT> above 1024 atoms and with more states than its 512 threads: every column of every row against
    the oracle (the 600 states share five lambdas, so the oracle's potential is taken once per lambda; the columns around
    the threads' wrap at 512 also go through the oracle's matrix whole), and unsampled states at the same boxes."""
    K, M = 4, 600
    s = lj_setup(N=N, n_alch=10, seed=5)
    scales = np.array([0.9, 1.0, 1.07, 1.15])
    xs = np.stack([(s['x'] * f).astype(np.float32).astype(np.float64) for f in scales])
    boxes = np.outer(scales, s['box'])
    lam_set = np.array([1.0, 0.75, 0.5, 0.2, 0.0])
    lambdas = lam_set[np.arange(M) % 5]
    temps = 280.0 + 0.15 * np.arange(M)
    pressures, disp = np.linspace(1.0, 120.0, M) * BAR, np.linspace(-45.0, -5.0, M)
    e = engine(s, K, M, lambdas, temps, pressures, disp)
    e.set_positions(xs)
    e.set_boxes(boxes)
    u = e.compute_energies()
    ul, ut, up, uc = np.array([0.37, 0.9, 0.05]), np.array([290.0, 350.0, 410.0]), np.array([5.0, 120.0, 60.0]) * BAR, \
        np.array([-50.0, -10.0, 0.0])
    uu = e.compute_energies_at(ut, ul, pressure=up, dispersion=uc)
    e.close()
    osys = oracle_system(s)
    U = onpt.energy_matrix(osys, xs, boxes, lam_set, np.ones(5), np.zeros(5), np.zeros(5))      # [K, 5] potentials
    V = np.prod(boxes, axis=1)[:, None]
    ref = (U[:, np.arange(M) % 5] + disp / V + pressures * V) / (KB * temps)
    assert (np.abs(u - ref) / np.maximum(1.0, np.abs(ref))).max() <= RTOL
    sel = np.array([0, 1, 4, 511, 512, 513, 517, 599])
    assert_energy_matrix(u[:, sel], osys, xs, boxes, lambdas[sel], temps[sel], pressures[sel], disp[sel])
    assert_energy_matrix(uu, osys, xs, boxes, ul, ut, up, uc)


def test_minimize_at_per_replica_boxes_above_1024_atoms():
    """k_minimize<APT = 4, NPT>: FIRE descent of 2048 atoms at each replica's own box, checked as the 512-atom test
    checks it: the oracle's forces at the returned positions and box meet the tolerance, positions are wrapped into the
    replica's box, and the boxes are left as they were."""
    N, K = 2048, 4
    s = lj_setup(N=N, n_alch=10, seed=8)
    scales = np.array([0.85, 0.95, 1.05, 1.2])
    boxes = np.outer(scales, s['box'])
    xs = np.stack([(s['x'] * f).astype(np.float32).astype(np.float64) for f in scales])
    lambdas = np.array([1.0, 0.7, 0.4, 0.0])
    rms0 = [np.sqrt((oracle_system(dict(s, box=boxes[k])).energy(xs[k], lambdas[k], forces=True)[2] ** 2).mean())
            for k in range(K)]
    tol = 0.1 * min(rms0)
    e = engine(s, K, K, lambdas, np.full(K, 300.0), np.full(K, 40.0 * BAR), np.full(K, -25.0))
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


# ---- 6. two GPUs -----------------------------------------------------------------------------------------------------
def npt_sharded_run(prefix):
    """An NPT ReplicaExchangeSampler of 8 replicas, 3 iterations, then the fused loop of a second sampler: the owned rows
    of positions, boxes and barostat records, the energy matrix and the replica->state map of both."""
    a, _, _ = npt_sampler(prefix + 'a.store', K=8, iterations=3)
    a.run()
    e = a._engine
    b = e.get_barostat()
    out = dict(k0=e.k0, x=e.get_positions(), box=e.get_boxes(), u=np.array(a._energy_thermodynamic_states),
               perm=np.array(a._replica_thermodynamic_states), **{'baro_' + f: v for f, v in b.items()})
    if a._last_npt_records is not None:     # the (K, 7) records gathered on rank 0
        out['records'] = a._last_npt_records
    d, _, _ = npt_sampler(prefix + 'd.store', K=8, iterations=3)
    d._compute_energies()
    d._engine.run_iterations(3, 'swap-all', d._seed, 1)
    e = d._engine
    b = e.get_barostat()
    out.update(fused_x=e.get_positions(), fused_box=e.get_boxes(), fused_u=e.get_energies(),
               fused_perm=e.get_replica_states(), **{'fused_baro_' + f: v for f, v in b.items()})
    return out


NPT_WORKER = r'''
import os, sys
sys.path.insert(0, %(root)r)
sys.path.insert(0, os.path.join(%(root)r, 'tests'))
import numpy as np
import torch.distributed as dist
dist.init_process_group('gloo')
from test_gpu_npt_variants import npt_sharded_run
rank = dist.get_rank()
np.savez(%(out)r + '_%%d.npz' %% rank, **npt_sharded_run(%(out)r + '_%%d_' %% rank))
dist.barrier()
'''


def test_two_gpus_reproduce_single_gpu_at_constant_pressure(tmp_path):
    """Two ranks own 4 replicas each: the boxes and barostat records are local rows, the replica->state map and the
    noise keys global.  Positions, boxes, barostat records, the energy matrix and the map equal the single-GPU run's bit
    for bit, per iteration and in the fused loop, and rank 0 gathers every replica's 7-number record."""
    from test_multi_gpu import _two_devices
    if not _two_devices():
        pytest.skip('needs 2 GPUs')
    ref = npt_sharded_run(str(tmp_path / 'one_'))
    script = tmp_path / 'npt2.py'
    out = str(tmp_path / 'two')
    script.write_text(NPT_WORKER % {'root': ROOT, 'out': out})
    r = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2',
                        '--master-addr', '127.0.0.1', '--master-port', '29537', str(script)],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    for rank in range(2):
        d = np.load(out + '_%d.npz' % rank)
        k0 = int(d['k0'])
        n = d['x'].shape[0]
        assert n == 4, n
        for key in ref:
            if key in ('k0', 'records'):
                continue
            want = ref[key] if key in ('u', 'perm', 'fused_u', 'fused_perm') else ref[key][k0:k0 + n]
            assert np.array_equal(d[key], want), (rank, key)
        if rank == 0:
            assert np.array_equal(d['records'], ref['records'])
        else:
            assert 'records' not in d.files
