"""Free energies of stored multistate runs: MultiStateSamplerAnalyzer and ReplicaExchangeAnalyzer
(openmmtools/multistate/multistateanalyzer.py:446-1135, :1137-2221, replicaexchange.py:427-439).

The analyzer reads a MultiStateReporter directory, detects equilibration on the effective energy timeseries
(:1414-1477, :2026-2093), subsamples the production iterations by their statistical inefficiency, lays the decorrelated
energies out as MBAR's u_kn with the unsampled end states as states without samples (:994-1036, :1479-1554), and solves
MBAR on the GPU (multistate.mbar.MBAR).  Free energies are in kT.

Not provided, each raising NotImplementedError: enthalpy and entropy (MBAR expectations of the reduced potential),
restraint unbiasing (no radially symmetric restraint force exists in this package, so ``unbias_restraint`` has nothing
to unbias, as in the reference for a system without one), SAMSAnalyzer, MultiPhaseAnalyzer and the observables registry.
"""
from typing import NamedTuple

import numpy as np
from scipy.special import logsumexp

from . import utils
from .mbar import MBAR
from .multistatereporter import MultiStateReporter


class MixingStatistics(NamedTuple):
    transition_matrix: np.ndarray
    eigenvalues: np.ndarray
    statistical_inefficiency: float


# The analysis steps below are shared by MultiStateSamplerAnalyzer, which reads a stored run, and the sampler's periodic
# offline pass (MultiStateSampler._offline_analysis), which keeps the same inputs in memory: the same operations in the
# same order give both the same bits.
def effective_energy_timeseries(u_kt, replica_state_indices=None, log_weights=None, f_l=None):
    """u_n = sum over replicas of u_kt [replica, iteration], each replica's reduced potential in the state it visits; with
    the [state, iteration] log weights of a SAMS run and its latest f_l = -logZ, corrected for the changing weights
    (:1414-1477)."""
    u_n = np.ascontiguousarray(u_kt, dtype=np.float64).sum(0)
    if log_weights is not None:
        for it in range(len(u_n)):
            st = replica_state_indices[:, it]
            u_n[it] += -np.sum(log_weights[st, it]) + logsumexp(-f_l + log_weights[:, it])
    return u_n


def equilibration_data(u_n, t0, max_subset):
    """(iterations discarded to equilibration, statistical inefficiency, effective samples) of the timeseries u_n, with
    the origins from t0 on (:2026-2093)."""
    i_t, g_i, n_effective_i = utils.get_equilibration_data_per_sample(u_n[t0:], max_subset=max_subset)
    i_max = n_effective_i.argmax()
    return i_t[i_max] + t0, g_i[i_max], n_effective_i.max()


def decorrelated_iterations(n_equilibration, statistical_inefficiency, max_n_iterations):
    """The production iterations n_equilibration..max_n_iterations, subsampled by the statistical inefficiency
    (:2211-2219)."""
    production = np.arange(n_equilibration, max_n_iterations + 1)
    return production[utils.subsample_correlated_data(production, statistical_inefficiency)]


class MultiStateSamplerAnalyzer:
    """MBAR analysis of a run stored by a MultiStateReporter.

    Parameters follow the reference: ``reporter, name, reference_states, max_n_iterations, analysis_kwargs,
    use_online_data, use_full_trajectory`` (PhaseAnalyzer) and then ``unbias_restraint, restraint_energy_cutoff,
    restraint_distance_cutoff, n_equilibration_iterations, statistical_inefficiency, max_subset``.  ``analysis_kwargs``
    go to MBAR (``initial_f_k``, ``maximum_iterations``, ``relative_tolerance``); with ``use_online_data`` the stored
    online f_k is the solver's starting point.  ``registry`` (the observables registry) is not provided.
    """

    def __init__(self, reporter, name=None, reference_states=(0, -1), max_n_iterations=None, analysis_kwargs=None,
                 registry=None, use_online_data=True, use_full_trajectory=False, *, unbias_restraint=True,
                 restraint_energy_cutoff='auto', restraint_distance_cutoff='auto', n_equilibration_iterations=None,
                 statistical_inefficiency=None, max_subset=100):
        if not isinstance(reporter, MultiStateReporter):
            raise ValueError('reporter must be a MultiStateReporter instance')
        if registry is not None:
            raise NotImplementedError('the observables registry (multistateanalyzer.py:106-355) is not provided')
        if analysis_kwargs is None:
            analysis_kwargs = {}
        elif not isinstance(analysis_kwargs, dict):
            raise ValueError('analysis_kwargs must be either None or a dictionary')
        if statistical_inefficiency and n_equilibration_iterations is None:
            raise ValueError('statistical_inefficiency needs n_equilibration_iterations: without it the equilibration '
                             'iterations cannot be found for the given statistical inefficiency')
        if not reporter.is_open():
            reporter.open(mode='r')
        self._reporter = reporter
        self.name = name
        self.reference_states = reference_states
        self._user_analysis_kwargs = dict(analysis_kwargs)
        self._use_online_data = use_online_data
        self.unbias_restraint = unbias_restraint
        self.restraint_energy_cutoff = restraint_energy_cutoff
        self.restraint_distance_cutoff = restraint_distance_cutoff
        self._n_equilibration_iterations = n_equilibration_iterations
        self._statistical_inefficiency = statistical_inefficiency
        self._max_subset = max_subset
        self._cache = {}
        self._max_n_iterations = None
        self.max_n_iterations = max_n_iterations
        self.use_full_trajectory = use_full_trajectory

    # -- properties of the reference
    @property
    def reporter(self):
        return self._reporter

    @property
    def reference_states(self):
        """(i, j): the states whose free energy difference a multi-phase analysis would combine."""
        return self._reference_states

    @reference_states.setter
    def reference_states(self, value):
        i, j = value[0], value[1]
        if type(i) is not int or type(j) is not int:
            raise ValueError('reference_states must be a length 2 iterable of ints')
        self._reference_states = (i, j)

    @property
    def n_iterations(self):
        """The last stored iteration (iteration 0 is the one before the first propagation)."""
        return self._reporter.read_last_iteration(last_checkpoint=False)

    @property
    def n_replicas(self):
        return len(self._reporter.read_replica_thermodynamic_states(iteration=0))

    @property
    def n_states(self):
        return self._reporter.read_energies(iteration=0)[0].shape[-1]

    @property
    def max_n_iterations(self):
        return self._max_n_iterations

    @max_n_iterations.setter
    def max_n_iterations(self, value):
        if value is None or value > self.n_iterations:
            value = self.n_iterations
        if value != self._max_n_iterations:
            self._cache.clear()
        self._max_n_iterations = value

    @property
    def use_full_trajectory(self):
        return self._use_full_trajectory

    @use_full_trajectory.setter
    def use_full_trajectory(self, value):
        if type(value) is not bool:
            raise ValueError('use_full_trajectory must be a boolean!')
        self._cache.pop('decorrelated', None)
        self._cache.pop('mbar', None)
        self._cache.pop('free_energy', None)
        self._use_full_trajectory = value

    @property
    def use_online_data(self):
        return self._use_online_data

    @use_online_data.setter
    def use_online_data(self, value):
        self._use_online_data = value
        self._cache.pop('mbar', None)
        self._cache.pop('free_energy', None)

    def clear(self):
        """Forget everything read or computed, for a reporter whose data changed."""
        self._cache.clear()
        self.max_n_iterations = None

    # -- data
    def read_energies(self):
        """(sampled [replica, state, iteration], unsampled [replica, unsampled state, iteration],
        neighborhoods [replica, state, iteration], replica_state_indices [replica, iteration]) of every stored
        iteration (:831-850)."""
        return self._read_energies(truncate_max_n_iterations=False)

    def _read_energies(self, truncate_max_n_iterations=False):
        sampled, neighborhoods, unsampled = self._reporter.read_energies()
        data = [sampled, unsampled, neighborhoods, self._reporter.read_replica_thermodynamic_states()]
        if truncate_max_n_iterations:
            data = [d[:self.max_n_iterations + 1] for d in data]
        data = [np.moveaxis(np.asarray(d), 0, -1) for d in data]
        if np.any(data[2] == 0):
            # a run stored with `locality` evaluated each replica in its neighbourhood of states only (:892)
            raise NotImplementedError('MBAR of a run stored with locality (neighbourhoods that are not all states) is '
                                      'not implemented')
        return tuple(data)

    @property
    def has_log_weights(self):
        """True when the storage holds the per-iteration log weights and logZ of a SAMS run."""
        try:
            self._reporter.read_online_analysis_data(0, 'log_weights', 'logZ')
            return True
        except (KeyError, OSError, IndexError, ValueError):
            return False

    def get_effective_energy_timeseries(self, energies=None, neighborhoods=None, replica_state_indices=None):
        """u_n = sum over replicas of the reduced potential in the state each replica visits at iteration n, corrected
        for changing log weights (:1414-1477)."""
        if energies is None and replica_state_indices is None:
            energies, _, neighborhoods, replica_state_indices = self._read_energies(truncate_max_n_iterations=True)
        elif (energies is None) != (replica_state_indices is None):
            raise ValueError('energies and replica_state_indices must be given together')
        n_replicas, _, n_iterations = energies.shape
        u_kt = energies[np.arange(n_replicas)[:, None], replica_state_indices, np.arange(n_iterations)[None, :]]
        log_weights = f_l = None
        if self.has_log_weights:
            data = self._reporter.read_online_analysis_data(slice(None), 'log_weights', 'logZ')
            log_weights = np.moveaxis(np.asarray(data['log_weights']), 0, -1)
            f_l = -np.asarray(data['logZ'])[-1]
        return effective_energy_timeseries(u_kt, replica_state_indices, log_weights, f_l)

    def _get_equilibration_data(self, energies=None, neighborhoods=None, replica_state_indices=None):
        """(iterations discarded to equilibration, statistical inefficiency, effective samples) (:2026-2093)."""
        if self._n_equilibration_iterations is not None and self._statistical_inefficiency is not None:
            n_equilibration = self._n_equilibration_iterations
            g_t = self._statistical_inefficiency
            n_effective_max = (self.max_n_iterations - n_equilibration + 1) / g_t
        else:
            u_n = self.get_effective_energy_timeseries(energies=energies, neighborhoods=neighborhoods,
                                                       replica_state_indices=replica_state_indices)
            # iteration 0 (right after minimisation) is always discarded; SAMS's second stage start t0 when stored
            t0 = self._n_equilibration_iterations if self._n_equilibration_iterations is not None else 1
            try:
                t0 = max(t0, int(np.asarray(self._reporter.read_online_analysis_data(None, 't0')['t0']).ravel()[0]))
            except (KeyError, OSError, IndexError, ValueError):
                pass
            n_equilibration, g_t, n_effective_max = equilibration_data(u_n, t0, self._max_subset)
            if self._statistical_inefficiency is not None:
                g_t = self._statistical_inefficiency
        return n_equilibration, g_t, n_effective_max

    @property
    def _equilibration_data(self):
        if 'equilibration' not in self._cache:
            self._cache['equilibration'] = self._get_equilibration_data()
        return self._cache['equilibration']

    @property
    def n_equilibration_iterations(self):
        """int: iterations discarded to equilibration."""
        return self._equilibration_data[0]

    @property
    def statistical_inefficiency(self):
        """float: statistical inefficiency of the production iterations."""
        return self._equilibration_data[1]

    @property
    def effective_length(self):
        """float: the production data as a number of uncorrelated samples."""
        return self._equilibration_data[2]

    @property
    def _decorrelated_iterations(self):
        """Indices of the iterations MBAR uses, up to max_n_iterations (:2211-2219)."""
        if self.use_full_trajectory:
            return np.arange(self.max_n_iterations + 1, dtype=int)
        return decorrelated_iterations(self.n_equilibration_iterations, self.statistical_inefficiency, self.max_n_iterations)

    @staticmethod
    def reformat_energies_for_mbar(u_kln, n_k=None):
        """[replica, state, iteration] -> [state, replica-major sample] (:994-1036); ``n_k`` limits each replica's
        iterations."""
        k, l, n = u_kln.shape
        if n_k is None:
            n_k = np.full(k, n, dtype=np.int64)
        return np.concatenate([u_kln[i, :, :n_k[i]] for i in range(k)], axis=1) if k else np.zeros((l, 0))

    def _compute_mbar_decorrelated_energies(self):
        """(u_ln, N_l): the decorrelated energies after equilibration, with the unsampled states first and last and
        without samples of their own (:1479-1554)."""
        data = list(self._read_energies(truncate_max_n_iterations=True))
        sampled, unsampled, neighborhoods, states = data
        if 'equilibration' not in self._cache:
            self._cache['equilibration'] = self._get_equilibration_data(sampled, neighborhoods, states)
        n_equilibration, g_t, _ = self._cache['equilibration']
        if not self.use_full_trajectory:
            data = [utils.subsample_data_along_axis(utils.remove_unequilibrated_data(d, n_equilibration, -1), g_t, -1)
                    for d in data]
        sampled, unsampled, _, states = data
        n_replicas, n_sampled, n_iterations = sampled.shape
        n_unsampled = unsampled.shape[1]
        n_total = n_sampled + n_unsampled
        u_ln = np.zeros((n_total, n_iterations * n_replicas))
        N_l = np.zeros(n_total, dtype=np.int64)
        first = n_unsampled // 2           # the unsampled states sit at both ends of the protocol
        u_ln[first:first + n_sampled] = self.reformat_energies_for_mbar(sampled)
        visited, counts = np.unique(states, return_counts=True)
        N_l[first + visited] = counts
        if n_unsampled > 0:
            u_ln[[0, -1]] = self.reformat_energies_for_mbar(unsampled)
        kwargs = dict(self._user_analysis_kwargs)
        if self.use_online_data and 'initial_f_k' not in kwargs:
            try:
                online_f_k = np.asarray(self._reporter.read_online_analysis_data(None, 'f_k')['f_k'], np.float64)
            except (KeyError, OSError, IndexError, ValueError):
                online_f_k = None
            if online_f_k is not None and online_f_k.shape == (n_sampled,):
                f = np.zeros(n_total)
                f[first:first + n_sampled] = online_f_k
                kwargs['initial_f_k'] = f
        return u_ln, N_l, kwargs

    @property
    def _decorrelated(self):
        if 'decorrelated' not in self._cache:
            self._cache['decorrelated'] = self._compute_mbar_decorrelated_energies()
        return self._cache['decorrelated']

    def _get_radially_symmetric_restraint_data(self):
        raise NotImplementedError('restraint unbiasing needs a radially symmetric restraint force '
                                  '(forces.RadiallySymmetricRestraintForce), which this package does not provide')

    @property
    def mbar(self):
        """multistate.mbar.MBAR of the decorrelated energies (states with no samples included)."""
        if 'mbar' not in self._cache:
            u_ln, N_l, kwargs = self._decorrelated
            self._cache['mbar'] = MBAR(u_ln, N_l, **kwargs)
        return self._cache['mbar']

    def get_free_energy(self):
        """(Delta_f_ij, dDelta_f_ij) in kT over every state, unsampled ones included (:1958-1974)."""
        if 'free_energy' not in self._cache:
            r = self.mbar.compute_free_energy_differences()
            self._cache['free_energy'] = (r['Delta_f'], r['dDelta_f'])
        return self._cache['free_energy']

    def get_enthalpy(self):
        raise NotImplementedError('enthalpy differences need MBAR expectations of the reduced potential, which '
                                  'multistate.mbar.MBAR does not compute')

    def get_entropy(self):
        raise NotImplementedError('entropy differences need MBAR expectations of the reduced potential, which '
                                  'multistate.mbar.MBAR does not compute')

    def generate_mixing_statistics(self, number_equilibrated=None):
        """Symmetrised state transition matrix of the replicas, its eigenvalues in descending order and the
        statistical inefficiency of the replicas' state indices, from ``number_equilibrated`` on (:1243-1303)."""
        if number_equilibrated is None:
            number_equilibrated = self.n_equilibration_iterations
        states = self._reporter.read_replica_thermodynamic_states()
        n_states = self.n_states
        n_ij = np.zeros((n_states, n_states), np.int64)
        for it in range(number_equilibrated, self.max_n_iterations - 1):
            np.add.at(n_ij, (states[it], states[it + 1]), 1)
        t_ij = np.zeros((n_states, n_states))
        for i in range(n_states):
            den = float(n_ij[i, :].sum() + n_ij[:, i].sum())
            if den > 0:
                t_ij[i, :] = (n_ij[i, :] + n_ij[:, i]) / den
            else:
                t_ij[i, i] = 1.0
        mu = np.linalg.eigvals(t_ij)
        mu = -np.sort(-mu)
        g = utils.statistical_inefficiency_multiple(np.transpose(states[number_equilibrated:self.max_n_iterations]))
        return MixingStatistics(transition_matrix=t_ij, eigenvalues=mu, statistical_inefficiency=g)


class ReplicaExchangeAnalyzer(MultiStateSamplerAnalyzer):
    """The analyzer of a ReplicaExchangeSampler or ParallelTemperingSampler run (replicaexchange.py:427-439)."""
    pass


class SAMSAnalyzer:
    """Not provided (sams.py:694-): raises NotImplementedError."""

    def __init__(self, *args, **kwargs):
        raise NotImplementedError('SAMSAnalyzer is not provided: its weighted MBAR over the SAMS log weights is not '
                                  'implemented')


class MultiPhaseAnalyzer:
    """Not provided (multistateanalyzer.py:2224-): raises NotImplementedError."""

    def __init__(self, phases):
        raise NotImplementedError('MultiPhaseAnalyzer is not provided: combine the free energies of the phases\' '
                                  'get_free_energy() by hand')


class ObservablesRegistry:
    """Not provided (multistateanalyzer.py:106-355): raises NotImplementedError."""

    def __init__(self):
        raise NotImplementedError('the observables registry is not provided; MultiStateSamplerAnalyzer computes the '
                                  'free energy only')
