"""Device MBAR (rx_mbar_*) against the numpy/scipy MBAR of oracle/mbar.py, and MultiStateSamplerAnalyzer on stored runs."""
import ctypes as C

import numpy as np
import pytest

from oracle import mbar as om
from openmmtools_b200 import _lib, alchemy, mcmc, multistate, states, testsystems, unit
from openmmtools_b200.multistate.mbar import MBAR

pytestmark = pytest.mark.gpu


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


class _Handle:
    def __init__(self, u, N_k):
        self.lib = _lib.load()
        self.u, self.N_k = np.ascontiguousarray(u), np.ascontiguousarray(N_k, dtype=np.int64)
        self.h = C.c_void_p()
        assert self.lib.rx_mbar_create(u.shape[0], u.shape[1], _ptr(self.u), _ptr(self.N_k), C.byref(self.h)) == 0

    def evaluate(self, f, max_blocks=0):
        K, N = self.u.shape
        assert self.lib.rx_mbar_set_max_blocks(self.h, max_blocks) == 0
        f = np.ascontiguousarray(f, dtype=np.float64)
        s, g, H, G, w, logD = C.c_double(), np.empty(K), np.empty((K, K)), np.empty((K, K)), np.empty(K), np.empty(N)
        assert self.lib.rx_mbar_evaluate(self.h, _ptr(f), C.byref(s), _ptr(g), _ptr(H)) == 0
        assert self.lib.rx_mbar_get_logden(self.h, _ptr(logD)) == 0
        assert self.lib.rx_mbar_gram(self.h, _ptr(f), _ptr(G), _ptr(w)) == 0
        return s.value, g, H, G, w, logD

    def close(self):
        self.lib.rx_mbar_destroy(self.h)


def _problem(K, N, seed):
    """u_kn of K overlapping states, every fifth state (and state 1) without samples, N samples in all."""
    rng = np.random.default_rng(seed)
    N_k = np.zeros(K, np.int64)
    sampled = [k for k in range(K) if k % 5 != 1] or [0]
    N_k[sampled] = N // len(sampled)
    N_k[sampled[0]] += N - N_k.sum()
    u = rng.normal(0.0, 1.5, (K, 1)) + rng.normal(0.0, 1.0, (K, N))
    return u, N_k, rng.normal(0.0, 1.0, K)


@pytest.mark.parametrize('K,N', [(2, 1001), (3, 2003), (64, 4099), (255, 5003), (256, 4097), (1024, 3001)])
def test_evaluate_and_gram_match_the_oracle(K, N):
    u, N_k, f = _problem(K, N, K)
    h = _Handle(u, N_k)
    try:
        s, g, H, G, w, logD = h.evaluate(f)
        s_r, g_r, H_r, G_r, w_r, logD_r = om.evaluate(u, N_k, f)
        Nf = N_k.astype(float)
        np.testing.assert_allclose(logD, logD_r, rtol=1e-12, atol=0)
        assert abs(s - s_r) <= 1e-12 * np.abs(logD_r).sum()
        assert np.all(np.abs(g - g_r) <= 1e-12 * Nf)
        np.testing.assert_allclose(w, w_r, rtol=1e-12)
        scale = np.sqrt(np.outer(np.diag(G_r), np.diag(G_r)))
        assert np.all(np.abs(G - G_r) <= 1e-11 * scale)
        assert np.all(np.abs(H - H_r) <= 1e-11 * (np.outer(Nf, Nf) * scale + np.diag(Nf * w_r)))
        assert np.array_equal(G, G.T)
        assert np.all(np.isfinite(H)) and np.all(H[N_k == 0] == 0)
    finally:
        h.close()


@pytest.mark.parametrize('K,N', [(3, 20001), (256, 40000)])
def test_bit_identical_across_runs_and_grid_sizes(K, N):
    u, N_k, f = _problem(K, N, 11)
    h = _Handle(u, N_k)
    try:
        a, b, c = h.evaluate(f), h.evaluate(f), h.evaluate(f, max_blocks=5)
        for x, y, z in zip(a, b, c):
            assert np.array_equal(np.asarray(x), np.asarray(y)) and np.array_equal(np.asarray(x), np.asarray(z))
    finally:
        h.close()


@pytest.mark.parametrize('K,N', [(2, 3001), (3, 4001), (64, 20000), (255, 20000)])
def test_solution_matches_the_oracle(K, N):
    u, N_k, _ = _problem(K, N, 100 + K)
    m = MBAR(u, N_k)
    D_r, dD_r, f_r = om.free_energy_differences(u, N_k)
    np.testing.assert_allclose(m.f_k, f_r, rtol=0, atol=1e-9)
    r = m.compute_free_energy_differences()
    np.testing.assert_allclose(r['Delta_f'], D_r, rtol=0, atol=1e-9)
    np.testing.assert_allclose(r['dDelta_f'], dD_r, rtol=1e-8, atol=1e-14)
    m.close()


def test_over_large_matrix_is_refused():
    lib = _lib.load()
    K, N = 1024, 40 * 1000 * 1000          # 328 GB of u_kn: larger than any H100's memory
    N_k = np.zeros(K, np.int64)
    N_k[0] = N
    small = np.zeros(1)                    # rx_mbar_create checks the size before it reads u_kn
    h = C.c_void_p()
    assert lib.rx_mbar_create(K, N, _ptr(small), _ptr(N_k), C.byref(h)) == _lib.RX_ERR_UNSUPPORTED
    assert not h.value
    assert b'free' in lib.rx_mbar_last_error(None)


def test_parallel_tempering_harmonic_oscillator_free_energies(tmp_path):
    """16 temperatures and two unsampled ones of a 3-D harmonic oscillator: f_j - f_i = (3/2) ln(beta_j / beta_i)."""
    ho = testsystems.HarmonicOscillator()
    move = mcmc.LangevinSplittingDynamicsMove(timestep=1.0 * unit.femtosecond, n_steps=200)
    base = states.ThermodynamicState(ho.system, 300 * unit.kelvin)
    unsampled = [states.ThermodynamicState(ho.system, T * unit.kelvin) for T in (280.0, 640.0)]
    reporter = multistate.MultiStateReporter(str(tmp_path / 'pt'), checkpoint_interval=100)
    s = multistate.ParallelTemperingSampler(mcmc_moves=move, number_of_iterations=400, seed=5)
    s.create(base, states.SamplerState(ho.positions), storage=reporter, min_temperature=300 * unit.kelvin,
             max_temperature=600 * unit.kelvin, n_temperatures=16, unsampled_thermodynamic_states=unsampled)
    s.run()
    temps = [280.0] + [float(t) for t in np.logspace(np.log10(300), np.log10(600), 16)] + [640.0]
    a = multistate.ReplicaExchangeAnalyzer(multistate.MultiStateReporter(str(tmp_path / 'pt'), open_mode='r'))
    D, dD = a.get_free_energy()
    assert D.shape == (18, 18)
    assert a.mbar.N_k[0] == 0 and a.mbar.N_k[-1] == 0 and np.all(a.mbar.N_k[1:-1] > 0)
    beta = 1.0 / np.array(temps)
    exact = 1.5 * np.log(beta[None, :] / beta[:, None])
    off = ~np.eye(18, dtype=bool)
    assert np.all(np.abs(D - exact)[off] <= 4 * dD[off]), np.max((np.abs(D - exact) / np.where(off, dD, 1))[off])
    assert np.all(dD[off] > 0)


def _lj_run(path, n_iterations, K=64):
    fluid = testsystems.LennardJonesFluid(nparticles=128)
    factory = alchemy.AbsoluteAlchemicalFactory(disable_alchemical_dispersion_correction=True)
    system = factory.create_alchemical_system(fluid.system, alchemy.AlchemicalRegion(alchemical_atoms=range(10)))
    lambdas = [1.0 - l / (K - 1) for l in range(K)]
    tstates = states.create_thermodynamic_state_protocol(
        system, {'lambda_sterics': lambdas, 'lambda_electrostatics': lambdas},
        constants={'temperature': 300 * unit.kelvin}, composable_states=alchemy.AlchemicalState.from_system(system))
    sstate = states.SamplerState(fluid.positions, box_vectors=system.getDefaultPeriodicBoxVectors())
    move = mcmc.LangevinSplittingDynamicsMove(timestep=1.0 * unit.femtosecond, n_steps=50, splitting='V R O R V')
    sampler = multistate.ReplicaExchangeSampler(mcmc_moves=move, number_of_iterations=n_iterations,
                                                replica_mixing_scheme='swap-all', seed=21)
    sampler.create(tstates, [sstate], storage=multistate.MultiStateReporter(str(path), checkpoint_interval=10))
    sampler.run()


def test_alchemical_lj_fluid_free_energies_and_truncation(tmp_path):
    _lj_run(tmp_path / 'long', 60)
    _lj_run(tmp_path / 'short', 40)
    a = multistate.MultiStateSamplerAnalyzer(multistate.MultiStateReporter(str(tmp_path / 'long'), open_mode='r'))
    D, dD = a.get_free_energy()
    assert D.shape == (64, 64) and np.all(np.isfinite(D)) and np.all(np.isfinite(dD))
    np.testing.assert_array_equal(np.diag(D), 0.0)
    np.testing.assert_allclose(D, -D.T, rtol=0, atol=1e-12)
    # without the stored online f_k (the two runs store different ones) both solves start from zero: same bits
    b = multistate.MultiStateSamplerAnalyzer(multistate.MultiStateReporter(str(tmp_path / 'long'), open_mode='r'),
                                             max_n_iterations=40, use_online_data=False)
    c = multistate.MultiStateSamplerAnalyzer(multistate.MultiStateReporter(str(tmp_path / 'short'), open_mode='r'),
                                             use_online_data=False)
    Db, dDb = b.get_free_energy()
    Dc, dDc = c.get_free_energy()
    np.testing.assert_array_equal(b.mbar.u_kn, c.mbar.u_kn)
    np.testing.assert_array_equal(Db, Dc)
    np.testing.assert_array_equal(dDb, dDc)
    # the stored online estimate only changes where the solve starts
    d = multistate.MultiStateSamplerAnalyzer(multistate.MultiStateReporter(str(tmp_path / 'long'), open_mode='r'),
                                             use_online_data=False)
    np.testing.assert_allclose(d.get_free_energy()[0], D, rtol=0, atol=1e-9)
