"""SAMSSampler: self-adjusted mixture sampling (expanded ensembles with on-the-fly weights) on the GPU engine.

Mirrors /root/reference/openmmtools/multistate/sams.py: options and validators (:196-289), ``_pre_write_create``
(:297-368), ``_mix_replicas`` (:395-437) with the ``global-jump`` scheme (:477-501; the only scheme the reference
currently allows, :246), the two-stage logZ update (:606-681), ``_update_stage`` (:564-604), ``_update_log_weights``
(:683-691), the state histogram bookkeeping (:385-393) and resume (:370-383).

Split of work: propagation and the K x M energy matrix run on the GPU (one launch each for all replicas; K replicas do
not have to equal M states here).  The jump itself and the weight update are O(K M) host arithmetic on the matrix the
reporter needs on the host anyway; they restate the reference line by line with numpy's legacy ``RandomState`` (the
reference uses numpy's global generator, seeded or not), and are pinned to golden vectors lifted from the reference
(tests/golden/make_sams_golden.py).

``device_weight_update=True`` moves the jump and the weight update onto the GPU as well (``rx_sams_step``, csrc/rx_sams.cuh:
one kernel on the resident energy matrix; logZ, weights, histogram, stage and t0 stay on the device), drawing the same
uniforms from the engine's copy of the MT19937 stream; the host generator is advanced in lockstep, so checkpoints and a later
switch back to the host path see the same stream.  The device arithmetic uses CUDA's exp/log, so logZ agrees with the host
path to ~1e-13, not bitwise (tests/test_gpu_sams.py); ``run_fused(n)`` runs n whole iterations without a host round trip.
"""
import numpy as np
from scipy.special import logsumexp
from .multistatesampler import MultiStateSampler


class SAMSSampler(MultiStateSampler):
    _TITLE_TEMPLATE = ('Self-adjusted mixture sampling (SAMS) simulation using SAMSSampler '
                       'class of openmmtools_b200.multistate on {}')
    _STORED_OPTIONS = MultiStateSampler._STORED_OPTIONS + (
        'state_update_scheme', 'update_stages', 'flatness_criteria', 'flatness_threshold', 'weight_update_method',
        'adapt_target_probabilities', 'gamma0', 'log_target_probabilities', 'device_weight_update')   # (a _StoredProperty in the reference, sams.py:281)

    def __init__(self, number_of_iterations=1, log_target_probabilities=None, state_update_scheme='global-jump',
                 locality=5, update_stages='two-stage', flatness_criteria='logZ-flatness', flatness_threshold=0.2,
                 weight_update_method='rao-blackwellized', adapt_target_probabilities=False, gamma0=1.0,
                 logZ_guess=None, device_weight_update=False, **kwargs):
        super().__init__(number_of_iterations=number_of_iterations, **kwargs)
        self.device_weight_update = bool(device_weight_update)
        self._sams_on_device = False
        self._sams_draws = 0          # uniforms drawn for jumps so far (either path): positions the device's stream copy
        self.log_target_probabilities = log_target_probabilities
        self.state_update_scheme = self._validate('state_update_scheme', state_update_scheme, ['global-jump'])
        self.locality = locality
        self.update_stages = self._validate('update_stages', update_stages, ['one-stage', 'two-stage'])
        self.flatness_criteria = self._validate('flatness_criteria', flatness_criteria,
                                                ['minimum-visits', 'logZ-flatness', 'histogram-flatness'])
        self.flatness_threshold = flatness_threshold
        self.weight_update_method = self._validate('weight_update_method', weight_update_method,
                                                   ['optimal', 'rao-blackwellized'])
        self.adapt_target_probabilities = self._validate('adapt_target_probabilities', adapt_target_probabilities, [False])
        self.gamma0 = gamma0
        self.logZ_guess = logZ_guess
        self._replica_neighbors = None
        self._cached_state_histogram = None
        self._rng = None

    @staticmethod
    def _validate(name, value, supported):
        if value not in supported:      # sams.py:243-279
            raise ValueError("Unknown update scheme '{}'. Supported values are {}.".format(value, supported))
        return value

    # ------------------------------------------------------------------ create
    def _initialize_stage(self):
        self._t0 = 0
        self._stage = 1 if self.update_stages == 'one-stage' else 0

    def _pre_write_create(self, thermodynamic_states, sampler_states, **kwargs):
        super()._pre_write_create(thermodynamic_states, sampler_states, **kwargs)
        if self.state_update_scheme == 'global-jump':
            self.locality = None           # sams.py:336-337: global jumps see every state
        self._initialize_stage()
        if self.log_target_probabilities is None:
            self.log_target_probabilities = np.zeros([self.n_states], np.float64) - np.log(self.n_states)
        else:
            self.log_target_probabilities = np.array(self.log_target_probabilities, np.float64)
        self._logZ = np.zeros([self.n_states], np.float64)
        if self.logZ_guess is not None:
            if len(self.logZ_guess) != self.n_states:
                raise Exception('Initial logZ_guess (dim {}) must have same number of states as n_states ({})'.format(
                    len(self.logZ_guess), self.n_states))
            self._logZ = np.array(self.logZ_guess, np.float64)
        self._update_log_weights()
        self._cached_state_histogram = np.zeros(self.n_states, dtype=int)
        self._last_gamma = None
        self._rng = np.random.RandomState((self._seed >> 8) & 0xFFFFFFFF)

    # ------------------------------------------------------------------ mixing = state jumps + weight update
    def _neighborhood(self, state_index=None):
        if self.locality is None or state_index is None:
            return list(range(0, self.n_states))
        return list(range(max(0, state_index - self.locality), min(self.n_states, state_index + self.locality + 1)))

    def _seed_mixing_streams(self):
        super()._seed_mixing_streams()
        from .. import _lib
        # the engine's numpy-RandomState stream is a copy of self._rng's (same seed): rx_sams_step draws the jumps from it
        self._engine.mix_seed((self._seed >> 8) & 0xFFFFFFFF, _lib.RX_STREAM_NUMPY)
        self._sams_on_device = False

    def _sams_device_init(self):
        """Hand the host's SAMS state to the device (first device step, after a restore, after host-path iterations)."""
        if self._sams_on_device:
            return
        from .. import _lib
        e = self._engine
        pos = e.mix_stream_position(_lib.RX_STREAM_NUMPY)
        if pos > 2 * self._sams_draws:
            raise RuntimeError('the device copy of the SAMS random stream is ahead of the host generator')
        if pos < 2 * self._sams_draws:
            e.mix_skip(2 * self._sams_draws - pos, _lib.RX_STREAM_NUMPY)
        e.set_energies(self._energy_thermodynamic_states)
        e.set_replica_states(self._replica_thermodynamic_states)
        e.sams_set(self.log_target_probabilities, self._logZ, histogram=self._cached_state_histogram, gamma0=self.gamma0,
                   flatness_threshold=self.flatness_threshold, weight_update_method=self.weight_update_method,
                   update_stages=self.update_stages, flatness_criteria=self.flatness_criteria, stage=self._stage, t0=self._t0)
        self._sams_on_device = True

    def _mix_replicas_device(self):
        """sams.py:395-437 in one kernel (rx_sams_step): jump of every replica, stage schedule, logZ and weight update."""
        e = self._engine
        K = self.n_replicas
        self._sams_device_init()
        update = self._iteration > 0          # not during equilibration (sams.py:429-435)
        e.sams_step(self._iteration, update_weights=update, histogram=self._cached_state_histogram)
        r = e.sams_get()
        self._n_accepted_matrix[:, :] = 0
        self._n_proposed_matrix[:, :] = 0
        for cur, new in zip(r['previous_states'], r['states']):
            self._n_proposed_matrix[cur, :] += 1
            self._n_accepted_matrix[cur, new] += 1
        self._replica_thermodynamic_states[:] = r['states']
        if update:
            self._logZ = r['logZ']
            self.log_weights = r['log_weights']
            self._stage, self._t0, self._last_gamma = int(r['stage']), int(r['t0']), float(r['gamma'])
        self._rng.random_sample(K)            # the host generator stays in lockstep (checkpoints, switching paths)
        self._sams_draws += K
        return self._replica_thermodynamic_states

    def run_fused(self, n_iterations):
        """n whole SAMS iterations (jump + weight update -> propagate -> energies) on the device without a host round trip
        (rx_sams_run_iterations); nothing is reported for them.  The sampler's host mirrors are refreshed at the end."""
        e = self._engine
        K = self.n_replicas
        if not self.device_weight_update:
            raise RuntimeError('run_fused needs device_weight_update=True')
        self._sams_device_init()
        e.sams_run_iterations(n_iterations, self._seed, self._iteration + 1)
        self._iteration += n_iterations
        r = e.sams_get()
        self._replica_thermodynamic_states[:] = r['states']
        self._logZ, self.log_weights = r['logZ'], r['log_weights']
        self._stage, self._t0, self._last_gamma = int(r['stage']), int(r['t0']), float(r['gamma'])
        self._cached_state_histogram[:] = r['histogram']
        self._rng.random_sample(K * n_iterations)
        self._sams_draws += K * n_iterations
        self._energy_thermodynamic_states[:] = e.get_energies()
        self._states_stale = True

    def _mix_replicas(self):
        if self.device_weight_update and self._engine is not None:
            return self._mix_replicas_device()
        self._sams_on_device = False
        self._sams_draws += self.n_replicas
        self._n_accepted_matrix[:, :] = 0
        self._n_proposed_matrix[:, :] = 0
        replicas_log_P_k = np.zeros([self.n_replicas, self.n_states], np.float64)
        self._global_jump(replicas_log_P_k)
        if self._iteration > 0:            # not during equilibration (sams.py:429-435)
            self._update_logZ_estimates(replicas_log_P_k)
            self._update_log_weights()
        if self._engine is not None:
            self._engine.set_replica_states(self._replica_thermodynamic_states)
        return self._replica_thermodynamic_states

    def _global_jump(self, replicas_log_P_k):
        """sams.py:477-501"""
        n_states = self.n_states
        for replica_index, current_state_index in enumerate(self._replica_thermodynamic_states):
            neighborhood = self._neighborhood(current_state_index)
            log_P_k = np.zeros([n_states], np.float64)
            u_k = self._energy_thermodynamic_states[replica_index, :]
            for state_index in neighborhood:
                log_P_k[state_index] = - u_k[state_index] + self.log_weights[state_index]
            log_P_k -= logsumexp(log_P_k)
            P_k = np.exp(log_P_k[neighborhood])
            new_state_index = self._rng.choice(neighborhood, p=P_k)
            self._replica_thermodynamic_states[replica_index] = new_state_index
            replicas_log_P_k[replica_index, :] = log_P_k[:]
            self._n_proposed_matrix[current_state_index, neighborhood] += 1
            self._n_accepted_matrix[current_state_index, new_state_index] += 1

    @property
    def _state_histogram(self):
        return self._cached_state_histogram

    def _update_stage(self):
        """sams.py:564-604"""
        minimum_visits = 1
        N_k = self._state_histogram
        if (self.update_stages == 'two-stage') and (self._stage == 0):
            advance = False
            if N_k.sum() == 0:
                return
            if self.flatness_criteria == 'minimum-visits':
                if np.all(N_k >= minimum_visits):
                    advance = True
            elif self.flatness_criteria == 'histogram-flatness':
                empirical_pi_k = N_k[:] / N_k.sum()
                pi_k = np.exp(self.log_target_probabilities)
                relative_error_k = np.abs(pi_k - empirical_pi_k) / pi_k
                if np.all(relative_error_k < self.flatness_threshold):
                    advance = True
            elif self.flatness_criteria == 'logZ-flatness':
                criteria = abs(self._logZ / self.gamma0) > self.flatness_threshold
                if np.all(criteria):
                    advance = True
            if advance or ((self._t0 > 0) and (self._iteration > self._t0)):
                self._stage = 1
                self._t0 = self._iteration - 1

    def _update_logZ_estimates(self, replicas_log_P_k):
        """sams.py:606-681"""
        log_pi_k = self.log_target_probabilities
        pi_k = np.exp(self.log_target_probabilities)
        self._update_stage()
        gamma = None
        for (replica_index, state_index) in enumerate(self._replica_thermodynamic_states):
            beta_factor = 0.8
            pi_star = pi_k.min()
            t = float(self._iteration)
            if self._stage == 0:
                gamma = self.gamma0 * min(pi_star, t ** (-beta_factor))
            elif self._stage == 1:
                gamma = self.gamma0 * min(pi_star, (t - self._t0 + self._t0 ** beta_factor) ** (-1))
            else:
                raise Exception(f'stage {self._stage} unknown')
            if self.weight_update_method == 'optimal':
                self._logZ[state_index] += gamma * np.exp(-log_pi_k[state_index])
            else:   # rao-blackwellized
                log_P_k = replicas_log_P_k[replica_index, :]
                neighborhood = np.where(self._neighborhoods[replica_index, :])[0]
                self._logZ[neighborhood] += gamma * np.exp(log_P_k[neighborhood] - log_pi_k[neighborhood])
        if self._stage == 1:
            self._logZ[:] -= self._logZ[0]
        self._last_gamma = gamma

    def _update_log_weights(self):
        self.log_weights = self.log_target_probabilities[:] - self._logZ[:]

    # ------------------------------------------------------------------ reporting / resume
    def _report_iteration_items(self):
        """Runs inside ``_report_iteration`` BEFORE the commit marker, so that an iteration the marker points at always has
        its logZ / stage / t0 / histogram record (a crash in between leaves the previous iteration as the last one)."""
        # state histogram exactly as the reference accumulates it (sams.py:385-393)
        st, cnt = np.unique(self._replica_thermodynamic_states, return_counts=True)
        self._cached_state_histogram[st] += cnt
        if self._reporter is not None and self._rank == 0:
            self._reporter.write_online_analysis_data(self._iteration, logZ=self._logZ, log_weights=self.log_weights,
                                                      stage=np.array([self._stage]), t0=np.array([self._t0]),
                                                      histogram=self._cached_state_histogram)

    def _log_weights_and_logZ(self):
        return self.log_weights, self._logZ

    def _checkpoint_extra(self):
        e = super()._checkpoint_extra()
        st = self._rng.get_state()
        e['sams_rng'] = [st[0], [int(x) for x in st[1]], int(st[2]), int(st[3]), float(st[4])]
        e['sams_draws'] = int(self._sams_draws)
        return e

    def _restore_sampler_from_reporter(self, reporter):
        super()._restore_sampler_from_reporter(reporter)
        if self.state_update_scheme == 'global-jump':
            self.locality = None
        data = reporter.read_online_analysis_data(self._iteration, 'logZ', 'stage', 't0', 'histogram')
        self.log_target_probabilities = np.zeros([self.n_states], np.float64) - np.log(self.n_states) \
            if self.log_target_probabilities is None else np.array(self.log_target_probabilities, np.float64)
        self._logZ = np.array(data['logZ'], np.float64)
        self._stage = int(data['stage'][0])
        self._t0 = int(data['t0'][0])
        self._cached_state_histogram = np.array(data['histogram'], dtype=int)
        self._update_log_weights()
        self._last_gamma = None
        extra = reporter.read_checkpoint_extra(self._iteration)
        self._rng = np.random.RandomState(0)
        r = extra['sams_rng']
        self._rng.set_state((r[0], np.array(r[1], dtype=np.uint32), r[2], r[3], r[4]))
        self._sams_draws = int(extra.get('sams_draws', int(extra.get('mt_numpy_words', 0)) // 2))
        self._sams_on_device = False
