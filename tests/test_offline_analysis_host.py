"""The offline free-energy pass of a running sampler, without a GPU: the completion rule, read_status, the timeseries
the pass shares with MultiStateSamplerAnalyzer, the real-time statistics file and the locality refusal."""
import os

import numpy as np
import pytest
import yaml

from openmmtools_b200 import multistate
from openmmtools_b200.multistate import multistateanalyzer as msa
from openmmtools_b200.multistate.multistatesampler import MultiStateSampler

is_completed = MultiStateSampler._is_completed_static


def test_is_completed_static():
    assert is_completed(10, 10, None, 0.0)
    assert not is_completed(10, 9, None, 0.0)
    assert not is_completed(10, 9, np.inf, 0.0)
    assert not is_completed(10, 9, 0.1, 0.0)
    assert is_completed(10, 9, 0.0, 0.0)            # a target of 0 stops only on an error of exactly 0
    assert is_completed(10, 9, 0.1, 0.1)
    assert not is_completed(10, 9, 0.11, 0.1)
    assert not is_completed(10, 9, np.nan, 0.1)
    assert not is_completed(10, 9, np.inf, 0.1)


def _storage(path, target, error, iteration=7, n_iterations=20, interval=5):
    r = multistate.MultiStateReporter(str(path), open_mode='w')
    r.set_dimensions(2, 2, 1)
    r.write_dict('options', {'number_of_iterations': n_iterations, 'online_analysis_interval': interval,
                             'online_analysis_target_error': target})
    if error is not None:
        r.write_online_data_dynamic_and_static(iteration, free_energy=np.array([1.5, error]))
    r.write_last_iteration(iteration)
    r.close()
    return str(path)


@pytest.mark.parametrize('target, error, status', [
    (0.0, 0.5, (None, False)), (0.0, 0.0, (None, False)), (0.0, np.inf, (None, False)),
    (1.0, 0.5, (1.0, True)), (1.0, 1.0, (1.0, True)), (0.2, 0.5, (0.2, False)),
    (1.0, np.inf, (1.0, False)), (1.0, np.nan, (1.0, False)), (1.0, None, (1.0, False))])
def test_read_status(tmp_path, target, error, status):
    s = MultiStateSampler.read_status(_storage(tmp_path / 'run.nc', target, error))
    assert s.iteration == 7
    assert (s.target_error, s.is_completed) == status


def test_read_status_iteration_limit(tmp_path):
    s = MultiStateSampler.read_status(_storage(tmp_path / 'run.nc', 1.0, np.inf, iteration=20))
    assert s.is_completed and s.target_error == 1.0


def test_read_status_without_online_analysis(tmp_path):
    path = _storage(tmp_path / 'run.nc', 1.0, 0.5, interval=None)
    s = MultiStateSampler.read_status(path)
    assert (s.target_error, s.is_completed) == (None, False)


def _run(path, n_iterations, K, n_unsampled, seed, log_weights):
    rng = np.random.default_rng(seed)
    r = multistate.MultiStateReporter(str(path), open_mode='w')
    r.set_dimensions(K, K, 1)
    r.write_thermodynamic_states([], [])
    states = np.arange(K)
    rows = {'u': [], 's': [], 'lw': []}
    logZ = np.zeros(K)
    for it in range(n_iterations + 1):
        if it:
            states = rng.permutation(states)
        u = rng.normal(size=(K, K)) + np.arange(K)[None, :] + 5.0 * np.exp(-it / 8.0)
        r.write_energies(u, np.ones((K, K), np.int8), rng.normal(size=(K, n_unsampled)), it)
        r.write_replica_thermodynamic_states(states, it)
        if log_weights:
            logZ = logZ + rng.normal(scale=0.1, size=K)
            lw = -np.log(K) - logZ
            r.write_online_analysis_data(it, logZ=logZ, log_weights=lw)
            rows['lw'].append(lw)
        r.write_last_iteration(it)
        rows['u'].append(u[np.arange(K), states])
        rows['s'].append(states.copy())
    r.close()
    return rows, logZ


@pytest.mark.parametrize('log_weights', [False, True])
@pytest.mark.parametrize('K', [3, 5])
def test_shared_timeseries_matches_the_analyzer(tmp_path, log_weights, K):
    """The pass keeps u[r, s_r(t)] per iteration and SAMS's log weights; from them the shared steps give the analyzer's
    effective-energy timeseries, equilibration and decorrelated iterations bit for bit."""
    rows, logZ = _run(tmp_path / 'run.nc', 90, K, 2, K, log_weights)
    a = multistate.MultiStateSamplerAnalyzer(multistate.MultiStateReporter(str(tmp_path / 'run.nc')))
    assert a.has_log_weights == log_weights
    states = np.stack(rows['s'], axis=1)
    lw = np.stack(rows['lw'], axis=1) if log_weights else None
    u_n = msa.effective_energy_timeseries(np.stack(rows['u'], axis=1), states, lw, -logZ if log_weights else None)
    ref = a.get_effective_energy_timeseries()
    assert u_n.tobytes() == ref.tobytes()
    n_eq, g, n_eff = msa.equilibration_data(u_n, 1, 100)
    assert (n_eq, g, n_eff) == (a.n_equilibration_iterations, a.statistical_inefficiency, a.effective_length)
    np.testing.assert_array_equal(msa.decorrelated_iterations(n_eq, g, 90), a._decorrelated_iterations)


def test_real_time_statistics_round_trip(tmp_path):
    r = multistate.MultiStateReporter(str(tmp_path / 'complex.nc'), open_mode='w')
    entries = []
    for it in (10, 20):
        data = {'iteration': it, 'percent_complete': it * 100 / 40,
                'mbar_analysis': {'free_energy_in_kT': -1.25 * it, 'standard_error_in_kT': np.inf if it == 10 else 0.5,
                                  'number_of_uncorrelated_samples': np.float32(12.5),
                                  'n_equilibrium_iterations': np.int64(3), 'statistical_inefficiency': 2.0},
                'timing_data': {'iteration_seconds': 0.01, 'ns_per_day': None, 'device_phase_ms': np.array([1.0, 2.0])}}
        r.write_current_statistics(data)
        entries.append(data)
    path = tmp_path / 'complex_real_time_analysis.yaml'
    assert r.real_time_statistics_path == str(path)
    loaded = yaml.safe_load(open(path))
    assert [e['iteration'] for e in loaded] == [10, 20]
    assert list(loaded[0]) == ['iteration', 'percent_complete', 'mbar_analysis', 'timing_data']
    assert list(loaded[0]['mbar_analysis']) == ['free_energy_in_kT', 'standard_error_in_kT',
                                               'number_of_uncorrelated_samples', 'n_equilibrium_iterations',
                                               'statistical_inefficiency']
    assert loaded[0]['mbar_analysis']['standard_error_in_kT'] == np.inf
    assert loaded[1]['mbar_analysis'] == {'free_energy_in_kT': -25.0, 'standard_error_in_kT': 0.5,
                                          'number_of_uncorrelated_samples': 12.5, 'n_equilibrium_iterations': 3,
                                          'statistical_inefficiency': 2.0}
    assert loaded[1]['timing_data']['device_phase_ms'] == [1.0, 2.0]
    # a resumed session appends; a fresh run starts over
    r2 = multistate.MultiStateReporter(str(tmp_path / 'complex.nc'), open_mode='a')
    r2.write_current_statistics({'iteration': 30})
    assert [e['iteration'] for e in yaml.safe_load(open(path))] == [10, 20, 30]
    r3 = multistate.MultiStateReporter(str(tmp_path / 'complex.nc'), open_mode='w')
    r3.write_current_statistics({'iteration': 5})
    assert yaml.safe_load(open(path)) == [{'iteration': 5}]


def test_locality_sampler_never_runs_the_pass(tmp_path):
    s = MultiStateSampler(locality=1, online_analysis_interval=2)
    s._reporter = multistate.MultiStateReporter(str(tmp_path / 'run.nc'), open_mode='w')
    s._iteration = 4
    s._online_analysis = lambda: np.inf

    def fail():
        raise AssertionError('the offline pass ran')
    s._offline_analysis = fail
    s._record_offline_inputs()          # keeps nothing (it would need an engine otherwise)
    assert s._offline_inputs is None
    s._offline_inputs = {'u': [], 'states': [], 'log_weights': None}    # (what would make a global run's pass run)
    s._update_analysis()
    assert s._last_err_free_energy == np.inf
    s.locality = None
    with pytest.raises(AssertionError, match='the offline pass ran'):
        s._update_analysis()
