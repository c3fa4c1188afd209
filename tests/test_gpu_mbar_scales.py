"""The device MBAR (rx_mbar_*) at the energy scales of real runs: states 10 to 10^4 kT apart, samples shifted by up to
10^6 kT, temperature ladders over thousands of atoms, states without samples far beyond the ends; against the 50-digit
mpmath MBAR of tests/mbar_mp.py and the log-space oracle of oracle/mbar.py.  Also the edges of the kernels' chunks and
tiles, more than 2^31 elements, and the analyzer and a live parallel-tempering run end to end."""
import ctypes as C

import numpy as np
import pytest

import mbar_mp as mm
from oracle import mbar as om
from openmmtools_b200 import _lib, multistate, states, mcmc, testsystems, unit
from openmmtools_b200._engine import Engine
from openmmtools_b200.multistate.mbar import MBAR
from test_gpu_mbar import _problem
from test_mbar_scales_host import SMALL, TABLE, check_solution

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


class _Handle:
    """rx_mbar_create on u_kn; evaluate returns every output of rx_mbar_evaluate, rx_mbar_gram and the getters."""

    def __init__(self, u, N_k):
        self.lib = _lib.load()
        self.u, self.N_k = np.ascontiguousarray(u, dtype=np.float64), np.ascontiguousarray(N_k, dtype=np.int64)
        self.h = C.c_void_p()
        assert self.lib.rx_mbar_create(self.u.shape[0], self.u.shape[1], _ptr(self.u), _ptr(self.N_k),
                                       C.byref(self.h)) == 0

    def evaluate(self, f, max_blocks=0):
        K, N = self.u.shape
        assert self.lib.rx_mbar_set_max_blocks(self.h, max_blocks) == 0
        f = np.ascontiguousarray(f, dtype=np.float64)
        s, g, H, G, w = C.c_double(), np.empty(K), np.empty((K, K)), np.empty((K, K)), np.empty(K)
        lw, logD = np.empty(K), np.empty(N)
        assert self.lib.rx_mbar_evaluate(self.h, _ptr(f), C.byref(s), _ptr(g), _ptr(H)) == 0
        assert self.lib.rx_mbar_get_log_wsum(self.h, _ptr(lw)) == 0
        assert self.lib.rx_mbar_get_logden(self.h, _ptr(logD)) == 0
        assert self.lib.rx_mbar_gram(self.h, _ptr(f), _ptr(G), _ptr(w)) == 0
        return s.value, g, H, G, w, logD, lw

    def close(self):
        self.lib.rx_mbar_destroy(self.h)


# -- 1. evaluation against mpmath ----------------------------------------------------------------------------------------
SCALES = [(spread, d) for spread in (10.0, 1.0e2, 1.0e3, 1.0e4) for d in (0.0, 1.0e6)]


@pytest.mark.parametrize('spread,d', SCALES)
def test_evaluate_matches_mpmath_at_scale(spread, d):
    """u = N(0, 1) + row offsets 0..spread + per-sample offsets d_n in [-d, d]; at f = 0 and at the solution."""
    u, N_k = mm.offsets(4, 60, spread, int(spread) + int(d), d=0.0, d_spread=d)
    ref = mm.Reference(u, N_k)
    f_mp = ref.solve()
    h = _Handle(u, N_k)
    try:
        for f in (np.zeros(4), np.array([float(x) for x in f_mp])):
            r = ref.evaluate(f)
            s, g, H, G, w, logD, lw = h.evaluate(f)
            # log D_n = (log D_n + m_n) - m_n on the shifted u: each c_k - u_kn is rounded at the size of its operands
            # and the shift adds an ulp of m_n, so a few ulp of max(|log D_n|, |c_k| + |u_kn|)
            c = np.abs(np.log(N_k) + f)[:, None] + np.abs(u)
            scale = np.maximum(np.abs(r['logD']), c.max(axis=0))
            assert np.all(np.abs(logD - r['logD']) <= 8 * EPS * scale)
            # log sum W: the shift leaves exp arguments of the size of the spread and f, so 1e-12 of max(1, |log sum|)
            assert np.all(np.isfinite(lw))
            assert np.all(np.abs(lw - r['log_wsum']) <= 1e-12 * np.maximum(1.0, np.abs(r['log_wsum'])))
            # G: 1e-12 relative where the exact value is a normal double
            normal = np.abs(r['G']) >= np.finfo(np.float64).tiny
            assert np.all(np.abs(G - r['G'])[normal] <= 1e-12 * np.abs(r['G'])[normal])
            assert np.all(np.abs(G[~normal]) <= 2 * np.finfo(np.float64).tiny)
    finally:
        h.close()


# -- 2. exact relations -------------------------------------------------------------------------------------------------
def _ladder():
    return mm.temperature_ladder(1000, 300.0, 360.0, 6, 300, 31, unsampled=50.0)


def test_row_shift_shifts_f_and_keeps_the_errors():
    u, N_k = _ladder()
    c = np.array([0.0, 3.0e3, -20.0, 1.0e2, 4.0e3, -7.0e2, 1.0e4, 5.0])
    a, b = MBAR(u, N_k), MBAR(u + c[:, None], N_k)
    assert np.all(np.abs((b.f_k - a.f_k) - (c - c[0])) <= 1e-12 * np.maximum(1.0, np.abs(c - c[0])) * 10)
    np.testing.assert_allclose(b.compute_free_energy_differences()['dDelta_f'],
                               a.compute_free_energy_differences()['dDelta_f'], rtol=1e-9, atol=1e-12)


def test_per_sample_shift_leaves_f_unchanged():
    u, N_k = _ladder()
    d = np.random.default_rng(1).uniform(-1.0e5, 1.0e5, u.shape[1])
    a, b = MBAR(u, N_k), MBAR(u + d[None, :], N_k)
    np.testing.assert_allclose(b.f_k, a.f_k, rtol=0, atol=1e-12 * np.abs(a.f_k).max() * 100)


def test_permuting_the_states_permutes_f():
    u, N_k = _ladder()
    a = MBAR(u, N_k)
    # the unsampled states move inside, and the first sampled state (the solve's gauge) is no longer state 1
    p = np.array([3, 0, 5, 7, 2, 1, 6, 4])
    b = MBAR(u[p], N_k[p])
    expect = a.f_k[p] - a.f_k[p][0]
    np.testing.assert_allclose(b.f_k, expect, rtol=0, atol=1e-11 * np.abs(expect).max())


def test_repeating_every_sample_keeps_f_and_divides_the_error():
    u, N_k = _ladder()
    a = MBAR(u, N_k)
    for m in (2, 7):
        b = MBAR(np.repeat(u, m, axis=1), N_k * m)
        np.testing.assert_allclose(b.f_k, a.f_k, rtol=0, atol=1e-11 * np.abs(a.f_k).max())
        da, db = a.compute_free_energy_differences()['dDelta_f'], b.compute_free_energy_differences()['dDelta_f']
        big = da > 1e-6 * da.max()
        np.testing.assert_allclose(db[big] * np.sqrt(m), da[big], rtol=1e-9)


# -- 3. solving at the scales of real runs ------------------------------------------------------------------------------
@pytest.mark.parametrize('name', list(SMALL))
def test_solution_matches_mpmath(name):
    u, N_k = SMALL[name]()
    ref = mm.Reference(u, N_k)
    f_mp = ref.solve()
    f_ref = np.array([float(x) for x in f_mp])
    m = MBAR(u, N_k)
    assert np.all(np.abs(m.f_k - f_ref) <= 1e-12 * np.maximum(1.0, np.abs(f_ref))), np.abs(m.f_k - f_ref).max()
    dd = ref.ddf(f_mp)
    big = dd > 1e-6 * dd.max()
    np.testing.assert_allclose(m.compute_free_energy_differences()['dDelta_f'][big], dd[big], rtol=1e-9)
    m.close()


@pytest.mark.parametrize('name', list(TABLE))
def test_solution_at_the_scales_of_real_runs(name):
    u, N_k = TABLE[name]()
    m = MBAR(u, N_k)
    check_solution(u, N_k, m.f_k, m.n_iterations)
    if N_k[0] == 0:                 # the unsampled ends are exact shifts of their neighbours by 900 kT
        assert abs(m.f_k[1] - m.f_k[0] - 900.0) <= 1e-12 * abs(m.f_k[1])
        assert abs(m.f_k[-1] - m.f_k[-2] - 900.0) <= 1e-12 * abs(m.f_k[-1])
    assert np.all(np.isfinite(m.compute_free_energy_differences()['dDelta_f']))
    m.close()


@pytest.mark.parametrize('delta', [40.0, 700.0, 1.0e4])
def test_two_state_pure_offset_gives_the_offset(delta):
    """Row 1 = row 0 + delta exactly (u on a grid of 2^-20, delta an integer), so f_1 - f_0 = delta."""
    u0 = np.round(np.random.default_rng(3).normal(0.0, 1.0, 1000) * 2.0 ** 20) / 2.0 ** 20
    m = MBAR(np.stack([u0, u0 + delta]), [500, 500])
    assert abs(m.f_k[1] - delta) <= 4 * EPS * delta
    m.close()


# -- 4. chunk and tile edges --------------------------------------------------------------------------------------------
@pytest.mark.parametrize('K', [1, 2, 65, 129])
@pytest.mark.parametrize('N', [1, 15, 16, 17, 8191, 8192, 8193, 3 * 8192 + 1, 5 * 8192 + 3])
def test_chunk_and_tile_edges_match_the_oracle(K, N):
    u, N_k, f = _problem(K, N, K * 7 + N)
    f[N_k == 0] = 0.0
    h = _Handle(u, N_k)
    try:
        runs = [h.evaluate(f, b) for b in (1, 7, 0)]
        for other in runs[1:]:
            for x, y in zip(runs[0], other):
                assert np.asarray(x).tobytes() == np.asarray(y).tobytes()
        s, g, H, G, w, logD, lw = runs[0]
        s_r, g_r, H_r, G_r, w_r, logD_r = om.evaluate(u, N_k, f)
        Nf = N_k.astype(float)
        np.testing.assert_allclose(logD, logD_r, rtol=1e-12, atol=0)
        assert abs(s - s_r) <= 1e-12 * np.abs(logD_r).sum()
        assert np.all(np.abs(g - g_r) <= 1e-12 * Nf)
        np.testing.assert_allclose(w, w_r, rtol=1e-12)
        np.testing.assert_allclose(lw, om.log_wsum(u, N_k, f), rtol=0, atol=1e-12)
        scale = np.sqrt(np.outer(np.diag(G_r), np.diag(G_r)))
        assert np.all(np.abs(G - G_r) <= 1e-11 * scale)
        assert np.all(np.abs(H - H_r) <= 1e-11 * (np.outer(Nf, Nf) * scale + np.diag(Nf * w_r)))
        assert np.array_equal(G, G.T)
    finally:
        h.close()


# -- 5. more than 2^31 elements -----------------------------------------------------------------------------------------
def test_more_than_2_31_elements_from_a_repeated_history():
    """K = 2 states, R = 64 replicas, 6 distinct iterations selected 2 796 203 times each: 2^31 + 256 elements
    (17 GB).  f is that of the 6 iterations alone, and dDelta_f shrinks by the square root of the repetition."""
    R, T, K, m = 64, 6, 2, 2796203
    rng = np.random.default_rng(5)
    u = rng.normal(0.0, 1.0, (T, R, K)) + np.array([0.0, 3.0e3])[None, None, :] - 4.0e4
    e = Engine(0, R, K)
    try:
        e.history_load(u)
        base = np.arange(T)
        cols = np.arange(K, dtype=np.int32)
        N_k = np.array([R * T // 2, R * T - R * T // 2])
        a = MBAR.from_history(e, base, cols, N_k)
        sel = np.tile(base, m)
        assert K * R * len(sel) > 2 ** 31
        try:
            b = MBAR.from_history(e, sel, cols, N_k * m)
        except NotImplementedError as err:           # the free device memory is shared: not enough now
            pytest.skip(str(err))
        np.testing.assert_allclose(b.f_k, a.f_k, rtol=0, atol=1e-9 * abs(a.f_k[1]))
        da, db = a.compute_free_energy_differences()['dDelta_f'], b.compute_free_energy_differences()['dDelta_f']
        np.testing.assert_allclose(db[0, 1] * np.sqrt(m), da[0, 1], rtol=1e-6)
        a.close(), b.close()
    finally:
        e.close()


# -- 6. end to end ------------------------------------------------------------------------------------------------------
def _write_ladder_run(path, n_atoms=4096, K=24, n_iterations=80, seed=0):
    """A stored parallel-tempering run of the temperature-ladder energy model of mbar_mp: K replicas over K
    temperatures 300..400 K with random neighbour swaps, and unsampled states 900 kT below the coldest and above the
    hottest."""
    rng = np.random.default_rng(seed)
    T = 300.0 * (400.0 / 300.0) ** (np.arange(K) / (K - 1))
    r = multistate.MultiStateReporter(str(path), open_mode='w')
    r.set_dimensions(K, K, 1)
    r.write_thermodynamic_states([], [])
    st = np.arange(K)
    for it in range(n_iterations + 1):
        if it:
            i = rng.integers(K - 1)
            a, b = np.flatnonzero(st == i)[0], np.flatnonzero(st == i + 1)[0]
            st[a], st[b] = st[b], st[a]
        t = T[st]
        E = n_atoms * (-15.0 + 1.5 * mm.KB * t) + rng.normal(0.0, mm.KB * t * np.sqrt(1.5 * n_atoms))
        u = E[:, None] / (mm.KB * T[None, :])
        un = np.stack([u[:, 0] - 900.0, u[:, -1] + 900.0], axis=1)
        r.write_energies(u, np.ones((K, K), np.int8), un, it)
        r.write_replica_thermodynamic_states(st, it)
        r.write_mixing_statistics(np.zeros((K, K)), np.zeros((K, K)), it)
        r.write_last_iteration(it)
    r.close()


def test_analyzer_on_a_stored_temperature_ladder(tmp_path):
    _write_ladder_run(tmp_path / 'run')
    a = multistate.MultiStateSamplerAnalyzer(multistate.MultiStateReporter(str(tmp_path / 'run'), open_mode='r'))
    D, dD = a.get_free_energy()
    assert np.all(np.isfinite(D)) and np.all(np.isfinite(dD))
    u_ln, N_l, _ = a._compute_mbar_decorrelated_energies()
    assert np.ptp(u_ln[1:-1].mean(axis=1)) > 1000.0           # the premise: thousands of kT across the ladder
    check_solution(u_ln, N_l, a.mbar.f_k, a.mbar.n_iterations)
    assert abs(D[0, 1] - 900.0) <= 1e-12 * abs(a.mbar.f_k[1]) + 1e-9


def test_live_parallel_tempering_run_stores_a_free_energy(tmp_path):
    fluid = testsystems.LennardJonesFluid(nparticles=512, reduced_density=0.8)
    move = mcmc.LangevinSplittingDynamicsMove(timestep=2.0 * unit.femtosecond, n_steps=50)
    s = multistate.ParallelTemperingSampler(mcmc_moves=move, number_of_iterations=40, seed=3,
                                            online_analysis_interval=20)
    box = fluid.system.getDefaultPeriodicBoxVectors()
    s.create(states.ThermodynamicState(fluid.system, 300 * unit.kelvin),
             states.SamplerState(fluid.positions, box_vectors=box),
             storage=multistate.MultiStateReporter(str(tmp_path / 'pt'), checkpoint_interval=20),
             min_temperature=300 * unit.kelvin, max_temperature=600 * unit.kelvin, n_temperatures=12)
    s.run(20)
    u = s._energy_thermodynamic_states
    spread = np.abs(u[:, -1] - u[:, 0]).min()
    assert spread > 100.0, spread                           # the premise: the end states are > 100 kT apart
    fe = multistate.MultiStateReporter(str(tmp_path / 'pt'), open_mode='r').read_online_analysis_data(
        20, 'free_energy')['free_energy']
    # the pass stored Delta_f; its error from the few decorrelated samples of 20 iterations may be +inf (NaN is stored
    # as +inf), but not negative
    assert np.isfinite(fe[0]) and fe[1] > 0, fe
