"""MBAR and the stored-run analyzer without a GPU: the numpy/scipy MBAR of oracle/mbar.py against the MBAR equations and
against harmonic oscillators of known free energy, the timeseries statistics against an AR(1) process and a planted
transient, and the analyzer's bookkeeping on a reporter directory written here."""
import inspect
import json
import os

import numpy as np
import pytest

from oracle import mbar as om
from openmmtools_b200 import multistate
from openmmtools_b200.multistate import utils

HERE = os.path.dirname(os.path.abspath(__file__))


def _random_ukn(rng, K, N_k):
    N = int(np.sum(N_k))
    return rng.normal(0.0, 2.0, (K, 1)) + rng.normal(0.0, 1.0, (K, N))


@pytest.mark.parametrize('N_k', [[40, 60], [30, 0, 50, 20], [0, 25, 25, 0, 40, 0]])
def test_oracle_solves_the_mbar_equations(N_k):
    rng = np.random.default_rng(len(N_k))
    u = _random_ukn(rng, len(N_k), N_k)
    f = om.solve(u, N_k)
    assert f[0] == 0.0
    W = om.weights(u, N_k, f)
    sampled = np.asarray(N_k) > 0
    # sum_n W_in = 1 for the sampled states; an unsampled state's f solves the same equation
    np.testing.assert_allclose(W.sum(axis=0)[sampled], 1.0, rtol=0, atol=1e-12)
    for i in np.flatnonzero(~sampled):
        fi = -np.log(np.sum(np.exp(-u[i] - om.log_denominator(u, N_k, f))))
        assert abs(f[i] - fi) < 1e-12


def _oscillators(rng, betaK, N_k):
    """Exact samples of 3-D harmonic oscillators u_k(x) = beta_k K_k |x|^2 / 2, and u_kn."""
    x = np.concatenate([rng.normal(0.0, 1.0 / np.sqrt(b), (n, 3)) for b, n in zip(betaK, N_k)])
    return 0.5 * np.asarray(betaK)[:, None] * (x ** 2).sum(1)[None, :]


def test_oracle_recovers_harmonic_oscillator_free_energies():
    betaK = np.array([1.0, 1.6, 2.5, 4.0])
    N_k = np.array([150, 100, 200, 120])
    exact = 1.5 * np.log(betaK / betaK[0])
    deltas, errors = [], []
    for seed in range(200):
        u = _oscillators(np.random.default_rng(seed), betaK, N_k)
        D, dD, _ = om.free_energy_differences(u, N_k)
        deltas.append(D[0])
        errors.append(dD[0])
    deltas, errors = np.array(deltas), np.array(errors)
    assert np.all(np.abs(deltas[:, 1:] - exact[1:]) <= 4 * errors[:, 1:])
    spread = deltas[:, 1:].std(axis=0, ddof=1)
    np.testing.assert_allclose(errors[:, 1:].mean(axis=0), spread, rtol=0.2)


def test_statistical_inefficiency_of_ar1():
    phi, T = 0.8, 200000
    rng = np.random.default_rng(7)
    e = rng.normal(size=T)
    x = np.empty(T)
    x[0] = e[0] / np.sqrt(1 - phi ** 2)
    for t in range(1, T):
        x[t] = phi * x[t - 1] + e[t]
    g = utils.statistical_inefficiency(x)
    # (1 + phi) / (1 - phi) = 9; the estimate's relative standard error at T = 2e5 is about 2 %
    assert abs(g / ((1 + phi) / (1 - phi)) - 1) < 0.1
    assert utils.subsample_correlated_data(np.zeros(10), 2.4) == [0, 2, 5, 7]


def test_equilibration_detection_finds_a_planted_transient():
    rng = np.random.default_rng(0)
    T, phi = 5000, 0.5
    e = rng.normal(size=T)
    x = np.empty(T)
    x[0] = e[0]
    for t in range(1, T):
        x[t] = phi * x[t - 1] + e[t]
    # a transient of 30 exp(-t / 80) on an AR(1) series (g = 3): below the noise from t ~ 300 on
    i_t, g_i, n_eff = utils.get_equilibration_data_per_sample(x + 30.0 * np.exp(-np.arange(T) / 80.0), max_subset=100)
    best = np.argmax(n_eff)
    assert len(i_t) == 99 and i_t[0] == 50
    assert 200 <= i_t[best] <= 600
    assert 2.0 <= g_i[best] <= 4.5


# -- the analyzer on a stored run ------------------------------------------------------------------------------------
def _write_run(path, n_iterations=120, K=4, n_unsampled=2, locality=False, seed=0):
    """A stored replica-exchange run: K replicas over K states, random swaps, energies of a drifting model, two
    unsampled end states."""
    rng = np.random.default_rng(seed)
    r = multistate.MultiStateReporter(str(path), open_mode='w')
    r.set_dimensions(K, K, 1)
    r.write_thermodynamic_states([], [])
    states = np.arange(K)
    rows = {'u': [], 's': [], 'un': []}
    for it in range(n_iterations + 1):
        if it:
            i = rng.integers(K - 1)
            a, b = np.flatnonzero(states == i)[0], np.flatnonzero(states == i + 1)[0]
            if rng.random() < 0.6:
                states[a], states[b] = states[b], states[a]
        u = rng.normal(size=(K, K)) + np.arange(K)[None, :] + 5.0 * np.exp(-it / 8.0)
        un = rng.normal(size=(K, n_unsampled))
        nb = np.ones((K, K), np.int8)
        if locality:
            nb[0, -1] = 0
        r.write_energies(u, nb, un, it)
        r.write_replica_thermodynamic_states(states, it)
        r.write_mixing_statistics(np.zeros((K, K)), np.zeros((K, K)), it)
        r.write_last_iteration(it)
        rows['u'].append(u); rows['s'].append(states.copy()); rows['un'].append(un)
    r.close()
    return {k: np.array(v) for k, v in rows.items()}


def test_analyzer_bookkeeping(tmp_path):
    data = _write_run(tmp_path / 'run')
    reporter = multistate.MultiStateReporter(str(tmp_path / 'run'), open_mode='r')
    a = multistate.ReplicaExchangeAnalyzer(reporter, max_n_iterations=90)
    assert a.n_iterations == 120 and a.max_n_iterations == 90 and a.n_replicas == 4 and a.n_states == 4
    sampled, unsampled, nb, states = a.read_energies()
    assert sampled.shape == (4, 4, 121) and unsampled.shape == (4, 2, 121) and states.shape == (4, 121)
    # equilibration: iteration 0 always goes, the decaying transient makes the detection discard more
    assert a.n_equilibration_iterations >= 1 and a.statistical_inefficiency >= 1.0
    its = a._decorrelated_iterations
    prod = np.arange(a.n_equilibration_iterations, 91)
    np.testing.assert_array_equal(its, prod[utils.subsample_correlated_data(prod, a.statistical_inefficiency)])
    u_ln, N_l, _ = a._compute_mbar_decorrelated_energies()
    n = len(its)
    assert u_ln.shape == (6, 4 * n) and N_l.sum() == 4 * n
    assert N_l[0] == 0 and N_l[-1] == 0           # the unsampled end states take part without samples
    for k in range(4):                            # replica-major columns
        np.testing.assert_array_equal(u_ln[1:5, k * n:(k + 1) * n], data['u'][its, k, :].T)
        np.testing.assert_array_equal(u_ln[0, k * n:(k + 1) * n], data['un'][its, k, 0])
        np.testing.assert_array_equal(u_ln[5, k * n:(k + 1) * n], data['un'][its, k, 1])
    np.testing.assert_array_equal(N_l[1:5], np.bincount(data['s'][its].ravel(), minlength=4))
    # the full trajectory and an explicit equilibration
    a.use_full_trajectory = True
    np.testing.assert_array_equal(a._decorrelated_iterations, np.arange(91))
    b = multistate.MultiStateSamplerAnalyzer(reporter, n_equilibration_iterations=10, statistical_inefficiency=3.0)
    assert (b.n_equilibration_iterations, b.statistical_inefficiency) == (10, 3.0)
    assert b.effective_length == pytest.approx((120 - 10 + 1) / 3.0)
    np.testing.assert_array_equal(b._decorrelated_iterations, np.arange(10, 121, 3))


def test_analyzer_truncation_matches_a_shorter_run(tmp_path):
    _write_run(tmp_path / 'long', n_iterations=120)
    _write_run(tmp_path / 'short', n_iterations=70)
    a = multistate.MultiStateSamplerAnalyzer(multistate.MultiStateReporter(str(tmp_path / 'long')), max_n_iterations=70)
    b = multistate.MultiStateSamplerAnalyzer(multistate.MultiStateReporter(str(tmp_path / 'short')))
    ua, Na, _ = a._compute_mbar_decorrelated_energies()
    ub, Nb, _ = b._compute_mbar_decorrelated_energies()
    np.testing.assert_array_equal(ua, ub)
    np.testing.assert_array_equal(Na, Nb)


def test_analyzer_mixing_statistics(tmp_path):
    data = _write_run(tmp_path / 'run')
    a = multistate.MultiStateSamplerAnalyzer(multistate.MultiStateReporter(str(tmp_path / 'run')))
    m = a.generate_mixing_statistics(number_equilibrated=5)
    s = data['s']
    n = np.zeros((4, 4))
    for it in range(5, 120 - 1):
        for k in range(4):
            n[s[it, k], s[it + 1, k]] += 1
    t = (n + n.T) / (n.sum(1) + n.sum(0))[:, None]
    np.testing.assert_allclose(m.transition_matrix, t, rtol=1e-15)
    np.testing.assert_allclose(m.transition_matrix.sum(1), 1.0)
    assert np.all(np.diff(m.eigenvalues.real) <= 1e-12) and abs(m.eigenvalues[0] - 1) < 1e-12
    assert m.statistical_inefficiency == utils.statistical_inefficiency_multiple(s[5:120].T)


def test_analyzer_refusals(tmp_path):
    _write_run(tmp_path / 'local', locality=True)
    a = multistate.MultiStateSamplerAnalyzer(multistate.MultiStateReporter(str(tmp_path / 'local')))
    with pytest.raises(NotImplementedError, match='locality'):
        a.read_energies()
    _write_run(tmp_path / 'run')
    a = multistate.MultiStateSamplerAnalyzer(multistate.MultiStateReporter(str(tmp_path / 'run')))
    with pytest.raises(NotImplementedError, match='enthalpy'):
        a.get_enthalpy()
    with pytest.raises(NotImplementedError, match='entropy'):
        a.get_entropy()
    with pytest.raises(NotImplementedError, match='restraint'):
        a._get_radially_symmetric_restraint_data()
    with pytest.raises(NotImplementedError, match='SAMSAnalyzer'):
        multistate.SAMSAnalyzer(a.reporter)
    with pytest.raises(NotImplementedError, match='MultiPhaseAnalyzer'):
        multistate.MultiPhaseAnalyzer({'a': a})
    with pytest.raises(ValueError):
        multistate.MultiStateSamplerAnalyzer(a.reporter, statistical_inefficiency=2.0)


@pytest.mark.parametrize('key', ['multistate/multistateanalyzer.py:MultiStateSamplerAnalyzer.__init__',
                                 'multistate/replicaexchange.py:ReplicaExchangeAnalyzer.__init__'])
def test_analyzer_signature_matches_reference(key):
    gold = json.load(open(os.path.join(HERE, 'golden', 'analyzer_signatures_golden.json')))[key]
    cls = getattr(multistate, key.split(':')[1].split('.')[0])
    params = inspect.signature(cls.__init__).parameters
    positional = [p for p in params.values() if p.kind is inspect.Parameter.POSITIONAL_OR_KEYWORD][1:]
    assert [p.name for p in positional] == [n for n, _ in gold['args']]
    for p, (n, d) in zip(positional, gold['args']):
        if n == 'registry':        # the observables registry is not provided: its default is None
            assert p.default is None
        elif d is not None:
            assert p.default == eval(d), n
    kwonly = [(p.name, p.default) for p in params.values() if p.kind is inspect.Parameter.KEYWORD_ONLY]
    assert kwonly == [(n, eval(d)) for n, d in gold['kwonly']]
