"""The offline MBAR pass of a running sampler: the engine's device energy history, u_kn gathered from it, parity of the
stored free energies with MultiStateSamplerAnalyzer, stopping at online_analysis_target_error, and resume."""
import os
import subprocess
import sys

import numpy as np
import pytest

from openmmtools_b200 import _lib, alchemy, mcmc, multistate, states, testsystems, unit
from openmmtools_b200._engine import Engine, EngineError
from openmmtools_b200.multistate.mbar import MBAR

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# -- gather ------------------------------------------------------------------------------------------------------------
def _history(R, M, U, T, seed):
    rng = np.random.default_rng(seed)
    u = rng.normal(0.0, 1.0, (T, R, M)) + 0.3 * np.arange(M)[None, None, :]
    uu = rng.normal(0.0, 1.0, (T, R, U)) + np.array([-0.5, 0.3 * M])[None, None, :U]
    st = np.array([rng.permutation(M)[:R] for _ in range(T)])
    return u, uu, st


def _host_ukn(u, uu, st, selected):
    """MultiStateSamplerAnalyzer's layout: unsampled states first and last, replica-major samples."""
    T, R, M = u.shape
    U = uu.shape[2]
    first = U // 2
    samp = np.moveaxis(u[selected], 0, -1)       # [replica, state, iteration]
    uns = np.moveaxis(uu[selected], 0, -1)
    u_ln = np.zeros((M + U, R * len(selected)))
    u_ln[first:first + M] = multistate.MultiStateSamplerAnalyzer.reformat_energies_for_mbar(samp)
    if U:
        u_ln[[0, -1]] = multistate.MultiStateSamplerAnalyzer.reformat_energies_for_mbar(uns)
    N_l = np.zeros(M + U, np.int64)
    v, c = np.unique(st[selected], return_counts=True)
    N_l[first + v] = c
    columns = np.zeros(M + U, np.int32)
    columns[first:first + M] = np.arange(M)
    if U:
        columns[[0, -1]] = (M, M + U - 1)
    return u_ln, N_l, columns


@pytest.mark.parametrize('R,M,U,T,n_sel', [(7, 11, 2, 60, 37), (33, 70, 2, 150, 101), (5, 9, 0, 40, 33)])
def test_gathered_u_kn_gives_the_host_bits(R, M, U, T, n_sel):
    u, uu, st = _history(R, M, U, T, R)
    e = Engine(0, R, M)
    try:
        e.history_load(u, uu if U else None)
        assert e.history_length() == (T, U)
        selected = np.sort(np.random.default_rng(M).choice(np.arange(1, T), n_sel, replace=False))
        u_ln, N_l, columns = _host_ukn(u, uu, st, selected)
        host = MBAR(u_ln, N_l)
        dev = MBAR.from_history(e, selected, columns, N_l)
        assert dev.u_kn is None
        np.testing.assert_array_equal(dev.f_k, host.f_k)
        a, b = host.compute_free_energy_differences(), dev.compute_free_energy_differences()
        np.testing.assert_array_equal(a['Delta_f'], b['Delta_f'])
        np.testing.assert_array_equal(a['dDelta_f'], b['dDelta_f'])
        lib = _lib.load()
        for blocks in (1, 3, 0):
            for m in (host, dev):
                assert lib.rx_mbar_set_max_blocks(m._h, blocks) == 0
            for x, y in zip(host._evaluate(host.f_k, True), dev._evaluate(host.f_k, True)):
                assert np.array_equal(x, y)
            logD = [np.empty(R * n_sel), np.empty(R * n_sel)]
            for m, out in zip((host, dev), logD):
                assert lib.rx_mbar_get_logden(m._h, out.ctypes.data_as(__import__('ctypes').c_void_p)) == 0
            assert logD[0].tobytes() == logD[1].tobytes()
        host.close(), dev.close()
    finally:
        e.close()


def test_gather_refuses_non_finite_energies_and_bad_indices():
    R, M, U, T = 7, 11, 2, 30
    u, uu, st = _history(R, M, U, T, 1)
    u[17, 3, 5] = np.nan
    e = Engine(0, R, M)
    try:
        e.history_load(u, uu)
        _, N_l, columns = _host_ukn(u, uu, st, np.arange(20))
        with pytest.raises(ValueError, match='finite'):
            MBAR.from_history(e, np.arange(20), columns, N_l)
        _, N_l, columns = _host_ukn(u, uu, st, np.arange(17))       # iteration 17 not selected: fine
        MBAR.from_history(e, np.arange(17), columns, N_l).close()
        uu[3, 0, 1] = np.inf                                        # an unsampled column
        e.history_load(u, uu)
        with pytest.raises(ValueError, match='finite'):
            MBAR.from_history(e, np.arange(5), columns, _host_ukn(u, uu, st, np.arange(5))[1])
        e.history_truncate(9)
        assert e.history_length() == (10, U)
        with pytest.raises(ValueError, match='not in the history'):
            MBAR.from_history(e, np.arange(11), columns, _host_ukn(u, uu, st, np.arange(11))[1])
        bad = columns.copy()
        bad[1] = M + U
        with pytest.raises(ValueError, match='column'):
            MBAR.from_history(e, np.arange(5), bad, _host_ukn(u, uu, st, np.arange(5))[1])
    finally:
        e.close()


def test_history_growth_beyond_free_memory_is_refused_and_the_run_goes_on(tmp_path):
    s = _ho_pt(tmp_path / 'run', 60, interval=20)
    s.run(30)
    n, U = s._engine.history_length()
    assert (n, U) == (31, 2)
    with pytest.raises(EngineError) as err:
        s._engine.history_reserve(10 ** 9, 2)         # 10^9 x 8 x 9 x 8 bytes: far beyond the device
    assert err.value.code == _lib.RX_ERR_UNSUPPORTED and 'free' in err.value.message
    assert s._engine.history_length() == (31, 2)
    s.run()
    assert s._engine.history_length() == (61, 2)
    r = multistate.MultiStateReporter(str(tmp_path / 'run'), open_mode='r')
    assert np.isfinite(r.read_online_analysis_data(60, 'free_energy')['free_energy']).all()


# -- samplers ----------------------------------------------------------------------------------------------------------
def _ho_pt(path, n_iterations, interval=50, checkpoint_interval=25, seed=11, target=0.0):
    ho = testsystems.HarmonicOscillator()
    move = mcmc.LangevinSplittingDynamicsMove(timestep=1.0 * unit.femtosecond, n_steps=100)
    base = states.ThermodynamicState(ho.system, 300 * unit.kelvin)
    unsampled = [states.ThermodynamicState(ho.system, T * unit.kelvin) for T in (290.0, 520.0)]
    s = multistate.ParallelTemperingSampler(mcmc_moves=move, number_of_iterations=n_iterations, seed=seed,
                                            online_analysis_interval=interval, online_analysis_target_error=target)
    s.create(base, states.SamplerState(ho.positions),
             storage=multistate.MultiStateReporter(str(path), checkpoint_interval=checkpoint_interval),
             min_temperature=300 * unit.kelvin, max_temperature=500 * unit.kelvin, n_temperatures=7,
             unsampled_thermodynamic_states=unsampled)
    return s


def _ho_sams(path, n_iterations, interval=50):
    ho = testsystems.HarmonicOscillator()
    move = mcmc.LangevinSplittingDynamicsMove(timestep=1.0 * unit.femtosecond, n_steps=100)
    ts = [states.ThermodynamicState(ho.system, T * unit.kelvin) for T in np.linspace(300.0, 450.0, 6)]
    s = multistate.SAMSSampler(mcmc_moves=move, number_of_iterations=n_iterations, seed=3,
                               online_analysis_interval=interval, flatness_criteria='minimum-visits')
    s.create(ts, [states.SamplerState(ho.positions)] * 4,
             storage=multistate.MultiStateReporter(str(path), checkpoint_interval=25))
    return s


def _lj_re(path, n_iterations, interval=50, K=64):
    fluid = testsystems.LennardJonesFluid(nparticles=128)
    factory = alchemy.AbsoluteAlchemicalFactory(disable_alchemical_dispersion_correction=True)
    system = factory.create_alchemical_system(fluid.system, alchemy.AlchemicalRegion(alchemical_atoms=range(10)))
    lambdas = [1.0 - l / (K - 1) for l in range(K)]
    tstates = states.create_thermodynamic_state_protocol(
        system, {'lambda_sterics': lambdas, 'lambda_electrostatics': lambdas},
        constants={'temperature': 300 * unit.kelvin}, composable_states=alchemy.AlchemicalState.from_system(system))
    sstate = states.SamplerState(fluid.positions, box_vectors=system.getDefaultPeriodicBoxVectors())
    move = mcmc.LangevinSplittingDynamicsMove(timestep=1.0 * unit.femtosecond, n_steps=50, splitting='V R O R V')
    s = multistate.ReplicaExchangeSampler(mcmc_moves=move, number_of_iterations=n_iterations,
                                          replica_mixing_scheme='swap-all', seed=21, online_analysis_interval=interval)
    s.create(tstates, [sstate], storage=multistate.MultiStateReporter(str(path), checkpoint_interval=25))
    return s


def _stored(path, t):
    r = multistate.MultiStateReporter(str(path), open_mode='r')
    d = r.read_online_analysis_data(t, 'free_energy', 'f_k_offline')
    return d['free_energy'], d['f_k_offline']


def _check_parity(s, path, n_iterations, interval):
    """At every interval iteration t the stored free energy is the analyzer's on iterations 0..t, started from the
    previous pass's f_k, bit for bit."""
    n_states = s.n_states + len(s._unsampled_states)
    prev, passes = np.zeros(n_states), 0
    while s.iteration < n_iterations:
        s.run(interval)
        t = s.iteration
        a = multistate.MultiStateSamplerAnalyzer(multistate.MultiStateReporter(str(path), open_mode='r'),
                                                 max_n_iterations=t, analysis_kwargs={'initial_f_k': prev})
        D, dD = a.get_free_energy()
        fe, f_k = _stored(path, t)
        err = np.inf if np.isnan(dD[0, -1]) else dD[0, -1]
        assert fe[0] == D[0, -1] and fe[1] == err, (t, fe, D[0, -1], dD[0, -1])
        assert f_k.tobytes() == a.mbar.f_k.tobytes()
        assert np.isfinite(fe[1])
        prev = a.mbar.f_k
        passes += 1
    assert passes == n_iterations // interval
    return prev


def test_parallel_tempering_parity(tmp_path):
    s = _ho_pt(tmp_path / 'pt', 300)
    _check_parity(s, tmp_path / 'pt', 300, 50)
    entries = __import__('yaml').safe_load(open(tmp_path / 'pt_real_time_analysis.yaml'))
    assert [e['iteration'] for e in entries] == [50, 100, 150, 200, 250, 300]
    fe, _ = _stored(tmp_path / 'pt', 300)
    assert entries[-1]['mbar_analysis']['free_energy_in_kT'] == fe[0]
    assert entries[-1]['mbar_analysis']['standard_error_in_kT'] == fe[1]


def test_sams_parity(tmp_path):
    s = _ho_sams(tmp_path / 'sams', 300)
    _check_parity(s, tmp_path / 'sams', 300, 50)


def test_alchemical_lj_replica_exchange_parity(tmp_path):
    s = _lj_re(tmp_path / 'lj', 100, interval=25)
    _check_parity(s, tmp_path / 'lj', 100, 25)


def _errors(path, n_iterations, interval):
    return {t: _stored(path, t)[0][1] for t in range(interval, n_iterations + 1, interval)}


def test_target_error_stops_the_run(tmp_path):
    full = _ho_pt(tmp_path / 'full', 300)
    full.run()
    assert full.iteration == 300              # a target of 0 runs to number_of_iterations
    errors = _errors(tmp_path / 'full', 300, 50)
    # the last interval iteration before the end whose error is below every earlier one
    t_star = max(t for t in errors if t < 300 and all(errors[t] < errors[q] for q in errors if q < t))
    target = float(np.nextafter(errors[t_star], np.inf))
    s = _ho_pt(tmp_path / 'stop', 300, target=target)
    s.run()
    assert s.iteration == t_star and s.is_completed
    status = multistate.ParallelTemperingSampler.read_status(str(tmp_path / 'stop'))
    assert status.iteration == t_star and status.target_error == target and status.is_completed
    assert _stored(tmp_path / 'stop', t_star)[0].tobytes() == _stored(tmp_path / 'full', t_star)[0].tobytes()
    resumed = multistate.ParallelTemperingSampler.from_storage(str(tmp_path / 'stop'))
    resumed.run()
    assert resumed.iteration == t_star
    assert multistate.MultiStateReporter(str(tmp_path / 'stop'), open_mode='r').read_last_iteration(False) == t_star


def test_resumed_run_stores_the_same_free_energies(tmp_path):
    full = _ho_pt(tmp_path / 'full', 300)
    full.run()
    part = _ho_pt(tmp_path / 'part', 300)
    part.run(160)
    del part
    resumed = multistate.ParallelTemperingSampler.from_storage(str(tmp_path / 'part'))
    assert resumed.iteration == 150
    assert resumed._engine.history_length() == (151, 2)
    resumed.run()
    for t in range(50, 301, 50):
        a, b = _stored(tmp_path / 'full', t), _stored(tmp_path / 'part', t)
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes(), t


def test_resumed_sams_run_stores_the_same_free_energies(tmp_path):
    full = _ho_sams(tmp_path / 'full', 200)
    full.run()
    part = _ho_sams(tmp_path / 'part', 200)
    part.run(130)
    del part
    resumed = multistate.SAMSSampler.from_storage(str(tmp_path / 'part'))
    assert resumed.iteration == 125
    resumed.run()
    for t in range(50, 201, 50):
        a, b = _stored(tmp_path / 'full', t), _stored(tmp_path / 'part', t)
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes(), t


# -- two ranks ---------------------------------------------------------------------------------------------------------
WORKER = r'''
import os, sys
sys.path.insert(0, %(root)r)
sys.path.insert(0, os.path.join(%(root)r, 'tests'))
import numpy as np
import torch.distributed as dist
dist.init_process_group('gloo')
from openmmtools_b200._dist import TorchCommunicator
from openmmtools_b200 import multistate, mcmc, states, testsystems, unit
ho = testsystems.HarmonicOscillator()
move = mcmc.LangevinSplittingDynamicsMove(timestep=1.0 * unit.femtosecond, n_steps=100)
base = states.ThermodynamicState(ho.system, 300 * unit.kelvin)
unsampled = [states.ThermodynamicState(ho.system, T * unit.kelvin) for T in (290.0, 520.0)]
s = multistate.ParallelTemperingSampler(mcmc_moves=move, number_of_iterations=300, seed=11, online_analysis_interval=50,
                                        online_analysis_target_error=%(target)r, communicator=TorchCommunicator())
s.create(base, states.SamplerState(ho.positions),
         storage=multistate.MultiStateReporter(%(path)r, checkpoint_interval=25),
         min_temperature=300 * unit.kelvin, max_temperature=500 * unit.kelvin, n_temperatures=7,
         unsampled_thermodynamic_states=unsampled)
s.run()
print('stopped', dist.get_rank(), s.iteration, flush=True)
dist.barrier()
'''


def _two_devices():
    import ctypes
    try:
        cuda = ctypes.CDLL('libcudart.so.12')
    except OSError:
        cuda = ctypes.CDLL('libcudart.so')
    n = ctypes.c_int()
    cuda.cudaGetDeviceCount(ctypes.byref(n))
    return n.value >= 2


def test_two_ranks_stop_together(tmp_path):
    if not _two_devices():
        pytest.skip('needs 2 GPUs')
    one = _ho_pt(tmp_path / 'one', 300)
    one.run()
    errors = _errors(tmp_path / 'one', 300, 50)
    t_star = max(t for t in errors if t < 300 and all(errors[t] < errors[q] for q in errors if q < t))
    target = float(np.nextafter(errors[t_star], np.inf))
    script = tmp_path / 'w.py'
    script.write_text(WORKER % {'root': ROOT, 'path': str(tmp_path / 'two'), 'target': target})
    r = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2',
                        '--master-addr', '127.0.0.1', '--master-port', '29547', str(script)],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert sorted(l for l in r.stdout.splitlines() if l.startswith('stopped')) == \
        ['stopped 0 %d' % t_star, 'stopped 1 %d' % t_star]
    for t in range(50, t_star + 1, 50):
        a, b = _stored(tmp_path / 'one', t), _stored(tmp_path / 'two', t)
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes(), t
