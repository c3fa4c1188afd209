"""MultiStateSampler: K replicas x M thermodynamic states on one (or several) H100s.

Mirrors /root/reference/openmmtools/multistate/multistatesampler.py for the hot path: ``create`` (:537-609,
836-926), ``run`` (:724-804), ``extend`` (:806), ``equilibrate`` (:649-720) and the three hooks
``_mix_replicas`` (:1500-1517), ``_propagate_replicas`` (:1287-1337), ``_compute_energies`` (:1436-1494).

What is different by design: the replicas are resident on the GPU (float4 positions/velocities for all K
replicas, the K x M energy matrix, the replica->state map, the swap statistics), the three phases are three
kernel launches, and ``sampler_states`` are materialised on the host only when asked for (or every iteration with
``host_resident_states=True``, which reproduces the reference's per-iteration host round trip).  Storage goes
through :class:`MultiStateReporter` (a netCDF4-free container with the reference's variable names; checkpoints also
carry the RNG positions, so a resumed run is bit-identical to an uninterrupted one).  Minimisation is outside the hot
path (SURVEY.md section 8f).  The periodic offline MBAR pass of a run with storage reads the energy matrices from a
history the engine keeps on the device (DESIGN §4.8), not from storage.

Multi-GPU: one process per GPU (torchrun style: RANK / WORLD_SIZE / LOCAL_RANK); replicas are sharded in contiguous
blocks, energy rows are all-gathered with NCCL, mixing is replicated from identical generator state.
"""
import collections
import copy
import logging
import os
import struct
import time
import numpy as np
from .. import unit, mcmc, states, _backend, _lib
from .._engine import EngineError, scale_mask
from ..cache import ContextCache
from .utils import SimulationNaNError
from .multistatereporter import MultiStateReporter
from .mbar import MBAR, MBARConvergenceError
from .multistateanalyzer import effective_energy_timeseries, equilibration_data, decorrelated_iterations

logger = logging.getLogger(__name__)


class MultiStateSampler:
    """Base class for samplers of multiple thermodynamic states (multistatesampler.py:63)."""

    _TITLE_TEMPLATE = ('Multi-state sampler simulation created using MultiStateSampler class '
                       'of openmmtools_b200.multistate on {}')
    Status = collections.namedtuple('Status', ['iteration', 'target_error', 'is_completed'])
    _global_citation_silence = False

    def __init__(self, mcmc_moves=None, number_of_iterations=1, online_analysis_interval=200,
                 online_analysis_target_error=0.0, online_analysis_minimum_iterations=200, locality=None,
                 host_resident_states=False, seed=None, communicator=None):
        if locality is not None and (not isinstance(locality, (int, np.integer)) or locality < 1):
            raise ValueError('locality must be a positive integer or None')     # multistatesampler.py:505-508
        # default move as the reference (multistatesampler.py:222-227)
        if mcmc_moves is None:
            self._mcmc_moves = mcmc.LangevinDynamicsMove(timestep=2.0 * unit.femtosecond,
                                                         collision_rate=5.0 / unit.picosecond, n_steps=500,
                                                         reassign_velocities=True, n_restart_attempts=6)
        else:
            self._mcmc_moves = copy.deepcopy(mcmc_moves)
        self._thermodynamic_states = None
        self._unsampled_states = None
        self._sampler_states = None
        self._replica_thermodynamic_states = None
        self._iteration = None
        self._energy_thermodynamic_states = None
        self._neighborhoods = None
        self._energy_unsampled_states = None
        self._n_accepted_matrix = None
        self._n_proposed_matrix = None
        self._metadata = None
        self._timing_data = dict()
        self._have_displayed_citations_before = False
        self.number_of_iterations = number_of_iterations
        self.online_analysis_interval = online_analysis_interval
        self.online_analysis_target_error = online_analysis_target_error
        self.online_analysis_minimum_iterations = online_analysis_minimum_iterations
        self.locality = locality
        self._last_mbar_f_k = None
        self._last_err_free_energy = None
        self._last_mbar_f_k_offline = None
        self._offline_inputs = None        # rank 0: the host inputs of the offline pass, one entry per iteration
        self._offline_stopped = False      # the energy history could not grow: no more offline passes in this run
        self.host_resident_states = host_resident_states
        self.energy_context_cache = ContextCache()
        self.sampler_context_cache = ContextCache()
        self._reporter = None
        self._want_async_reporting = False
        self._unsampled_table = None
        self._engine = None
        self._mc_moves = None          # per state, the Metropolized moves the engine runs (None: no state has one)
        self._states_stale = False     # host copies of sampler states are behind the device
        self._host_x = self._host_v = None   # page-locked backing store of the owned sampler states
        self._host_store = None
        self._seed = seed
        self._communicator = communicator
        self._rank = int(os.environ.get('RANK', '0')) if communicator is None else communicator.rank
        self._world_size = int(os.environ.get('WORLD_SIZE', '1')) if communicator is None else communicator.world_size

    # ------------------------------------------------------------------ properties (multistatesampler.py:365-535)
    @property
    def n_states(self):
        return None if self._thermodynamic_states is None else len(self._thermodynamic_states)

    @property
    def n_replicas(self):
        return None if self._sampler_states is None else len(self._sampler_states)

    @property
    def iteration(self):
        return self._iteration

    @property
    def mcmc_moves(self):
        return copy.deepcopy(self._mcmc_moves)

    @mcmc_moves.setter
    def mcmc_moves(self, new_value):
        if self._thermodynamic_states is not None:
            raise RuntimeError('Cannot modify MCMC move after initialization (create()).')
        self._mcmc_moves = copy.deepcopy(new_value)

    @property
    def sampler_states(self):
        """Deep copies of the sampler states (multistatesampler.py:410-429); pulls them from the GPU if needed."""
        self._sync_sampler_states()
        return copy.deepcopy(self._sampler_states)

    @sampler_states.setter
    def sampler_states(self, value):
        if self._iteration != 0:
            raise RuntimeError('Sampler states can be assigned only between create() and run().')
        if len(value) != self.n_replicas:
            raise ValueError('Passed {} sampler states for {} replicas'.format(len(value), self.n_replicas))
        self._sampler_states = copy.deepcopy(value)
        self._upload_sampler_states()

    @property
    def is_periodic(self):
        if self._thermodynamic_states is None:
            return None
        return self._thermodynamic_states[0].is_periodic

    @property
    def metadata(self):
        return copy.deepcopy(self._metadata)

    @property
    def is_completed(self):
        return self._is_completed()

    @classmethod
    def default_options(cls):
        import inspect
        opts = {}
        for c in reversed(cls.__mro__):
            if c is object:
                continue
            for n, p in inspect.signature(c.__init__).parameters.items():
                if p.default is not inspect.Parameter.empty and p.kind is not inspect.Parameter.VAR_KEYWORD:
                    opts[n] = p.default
        return opts

    @property
    def options(self):
        return {n: getattr(self, n, getattr(self, '_' + n, None)) for n in self.default_options()}

    # options that are stored with the data and restored by from_storage (the reference stores every __init__ kwarg
    # through _StoredProperty, multistatesampler.py:438-518)
    _STORED_OPTIONS = ('number_of_iterations', 'online_analysis_interval', 'online_analysis_target_error',
                       'online_analysis_minimum_iterations', 'locality', 'host_resident_states', 'replica_mixing_scheme')

    @classmethod
    def from_storage(cls, storage, communicator=None):
        """Restore a sampler from disk and prepare it to resume (multistatesampler.py:264-300, 956-1047): the most
        recent checkpoint is loaded (positions, velocities, states, energies of that iteration) and -- unlike the
        reference, whose generators are not stored -- the RNG streams are put back where they were, so the continuation
        is bit-identical to an uninterrupted run."""
        reporter = storage if isinstance(storage, MultiStateReporter) else MultiStateReporter(storage)
        if not reporter.is_open():
            reporter.open('a')
        options = reporter.read_dict('options') or {}
        kwargs = {k: v for k, v in options.items() if k in cls._STORED_OPTIONS and k in cls.default_options()}
        if kwargs.get('number_of_iterations') == 'inf':
            kwargs['number_of_iterations'] = np.inf
        sampler = cls(mcmc_moves=reporter.read_mcmc_moves(), seed=options.get('seed'), communicator=communicator, **kwargs)
        sampler._restore_sampler_from_reporter(reporter)
        return sampler

    @classmethod
    def read_status(cls, storage):
        """Iteration, target error and completion state of a stored run (multistatesampler.py:308-360)."""
        reporter = storage if isinstance(storage, MultiStateReporter) else MultiStateReporter(storage)
        was_open = reporter.is_open()
        if not was_open:
            reporter.open('r')
        options = reporter.read_dict('options') or {}
        iteration = reporter.read_last_iteration(last_checkpoint=False)
        n_it = options.get('number_of_iterations')
        n_it = np.inf if n_it == 'inf' else n_it
        target = options.get('online_analysis_target_error', 0.0)
        target_error = last_err = None
        # the error of the last offline pass counts only when online analysis runs and the target is a stopping condition
        if options.get('online_analysis_interval') is not None and target != 0.0:
            target_error = target
            try:
                last_err = float(reporter.read_online_analysis_data(None, 'free_energy')['free_energy'][1])
            except (KeyError, OSError, IndexError, ValueError):
                last_err = np.inf
        if not was_open:
            reporter.close()
        is_completed = n_it is not None and cls._is_completed_static(n_it, iteration, last_err, target)
        return cls.Status(iteration=iteration, target_error=target_error, is_completed=is_completed)

    def _restore_sampler_from_reporter(self, reporter):
        metadata = reporter.read_dict('metadata')
        thermodynamic_states, unsampled_states = reporter.read_thermodynamic_states()
        last = reporter.read_last_iteration(last_checkpoint=False)
        checkpoints = [c for c in reporter.read_checkpoint_iterations() if c <= last]
        if not checkpoints:
            raise RuntimeError('Attempting to restore from any checkpoint failed.')
        checkpoint = checkpoints[-1]
        self._iteration = int(checkpoint)
        self._thermodynamic_states = thermodynamic_states
        self._unsampled_states = unsampled_states or []
        self._sampler_states = reporter.read_sampler_states(iteration=checkpoint)
        self._replica_thermodynamic_states = np.array(reporter.read_replica_thermodynamic_states(iteration=checkpoint), dtype=np.int64)
        e, nb, _ = reporter.read_energies(iteration=checkpoint)
        self._energy_thermodynamic_states = np.array(e, dtype=np.float64)
        self._neighborhoods = np.array(nb, dtype=np.int8)
        _un = reporter.read_unsampled_energies(checkpoint)
        self._energy_unsampled_states = np.zeros((len(self._sampler_states), len(self._unsampled_states))) if _un is None else np.array(_un)
        na, npr = reporter.read_mixing_statistics(iteration=checkpoint)
        self._n_accepted_matrix = np.array(na, dtype=np.int64)
        self._n_proposed_matrix = np.array(npr, dtype=np.int64)
        self._metadata = metadata
        self._timing_data = dict()
        try:  # the online free-energy estimate of the checkpoint iteration (multistatesampler.py:1697-1718)
            self._last_mbar_f_k = np.array(reporter.read_online_analysis_data(int(checkpoint), 'f_k')['f_k'])
        except (KeyError, IndexError, FileNotFoundError):
            self._last_mbar_f_k = None
        if isinstance(self._mcmc_moves, mcmc.MCMCMove):
            self._mcmc_moves = [copy.deepcopy(self._mcmc_moves) for _ in thermodynamic_states]
        self._reporter = reporter
        self._wrap_reporter()
        extra = reporter.read_checkpoint_extra(checkpoint)
        if self._seed is None:
            self._seed = extra.get('seed')
        self._create_engine()
        if 'mc_accepted' in extra and self._mc_moves:   # the move counts of the checkpoint (the moves may be stored later)
            self._mc_counts_to_moves(self._mc_moves, np.array(extra['mc_accepted']), np.array(extra['mc_proposed']))
            self._push_mc_statistics()
        if 'barostat' in extra:     # the NPT run continues with the barostat state it had at the checkpoint
            self._engine.set_barostat({k: np.asarray(v)[self._engine.k0:self._engine.k1] for k, v in extra['barostat'].items()},
                                      first=self._engine.k0)
        if 'barostat_anisotropic' in extra:     # ... and the per-axis state of an anisotropic one
            k0, k1 = self._engine.k0, self._engine.k1
            a = {k: np.asarray(v)[k0:k1] for k, v in extra['barostat_anisotropic'].items()}
            a['step'] = np.asarray(extra['barostat']['step'])[k0:k1]
            a['scale_mask'] = np.full(k1 - k0, scale_mask(_backend.barostat_scale(self._thermodynamic_states)))
            self._engine.set_barostat_anisotropic(a, first=k0)
        # energies of the checkpoint iteration are what the next mixing uses
        self._engine.set_energies(self._energy_thermodynamic_states)
        # put the two MT19937 streams back where they were
        for stream, key in ((_lib.RX_STREAM_NUMBA, 'mt_numba_words'), (_lib.RX_STREAM_NUMPY, 'mt_numpy_words')):
            n = int(extra.get(key, 0))
            if n:
                self._engine.mix_skip(n, stream)
        self._equil_counter = int(extra.get('equil_counter', 0))
        self._restore_offline_analysis(reporter, int(checkpoint))

    def _restore_offline_analysis(self, reporter, checkpoint):
        """The offline pass of the checkpoint iteration's state: its error and the last f_k_offline up to the checkpoint
        (where the reference restarts from zeros; these keep the stored free energies of a resumed run bit-identical to an
        uninterrupted run's), and on rank 0 its inputs: the stored energies of iterations 0..checkpoint, read once."""
        try:
            self._last_err_free_energy = float(reporter.read_online_analysis_data(checkpoint, 'free_energy')['free_energy'][1])
        except (KeyError, IndexError, OSError):
            self._last_err_free_energy = None
        try:
            f = np.asarray(reporter.read_online_analysis_data(slice(0, checkpoint + 1), 'f_k_offline')['f_k_offline'])
            done = np.flatnonzero(np.any(f != 0, axis=1))      # (iterations without a pass hold zeros)
            self._last_mbar_f_k_offline = f[done[-1]].copy() if len(done) else None
        except (KeyError, OSError):
            self._last_mbar_f_k_offline = None
        if not self._keeps_offline_inputs:
            return
        e, _, unsampled = reporter.read_energies(slice(0, checkpoint + 1))
        st = reporter.read_replica_thermodynamic_states(slice(0, checkpoint + 1))
        try:
            lw = np.asarray(reporter.read_online_analysis_data(slice(0, checkpoint + 1), 'log_weights')['log_weights'])
        except (KeyError, OSError):
            lw = None
        try:
            self._engine.history_load(e, unsampled if unsampled.shape[-1] else None)
        except EngineError as err:
            self._stop_offline_analysis(err)
            return
        diag = e[np.arange(len(e))[:, None], np.arange(e.shape[1])[None, :], st]
        self._offline_inputs = {'u': list(diag), 'states': list(st), 'log_weights': None if lw is None else list(lw)}

    # ------------------------------------------------------------------ create (multistatesampler.py:537-609)
    def create(self, thermodynamic_states, sampler_states, storage=None, initial_thermodynamic_states=None,
               unsampled_thermodynamic_states=None, metadata=None):
        if storage is not None:
            self._reporter = storage if isinstance(storage, MultiStateReporter) else MultiStateReporter(storage)
            self._wrap_reporter()
        if self._thermodynamic_states is not None:
            raise RuntimeError('Cannot initialize the same sampler twice (create() was already called).')
        # multistatesampler.py:586-589: an existing storage is never overwritten
        if self._reporter is not None and self._reporter.storage_exists():
            raise RuntimeError('Storage file {} already exists; cowardly refusing to overwrite.'.format(
                self._reporter.filepath))
        if isinstance(sampler_states, states.SamplerState):
            sampler_states = [sampler_states]
        self._pre_write_create(list(thermodynamic_states), list(sampler_states),
                               initial_thermodynamic_states=initial_thermodynamic_states,
                               unsampled_thermodynamic_states=unsampled_thermodynamic_states, metadata=metadata)
        self._initialize_reporter()

    def _pre_write_create(self, thermodynamic_states, sampler_states, initial_thermodynamic_states=None,
                          unsampled_thermodynamic_states=None, metadata=None):
        # checks of multistatesampler.py:850-869
        n_particles = thermodynamic_states[0].n_particles
        for s in thermodynamic_states:
            if s.is_periodic != thermodynamic_states[0].is_periodic:
                raise Exception('Thermodynamic states contain a mixture of systems with and without periodic boundary conditions.')
            if s.n_particles != n_particles:
                raise ValueError('All ThermodynamicStates must have the same number of particles')
        for ss in sampler_states:
            if ss.n_particles != n_particles:
                raise ValueError('All SamplerStates must have the same number of particles')
            if thermodynamic_states[0].is_periodic and ss.box_vectors is None:
                raise Exception('All sampler states must have box_vectors defined if the system is periodic.')
        self._metadata = metadata
        self._thermodynamic_states = [copy.deepcopy(s) for s in thermodynamic_states]
        self._unsampled_states = [copy.deepcopy(s) for s in (unsampled_thermodynamic_states or [])]
        for s in self._unsampled_states:
            if s.n_particles != n_particles:
                raise ValueError('All ThermodynamicStates must have the same number of particles')
        self._sampler_states = [copy.deepcopy(s) for s in sampler_states]
        K, M = len(self._sampler_states), len(self._thermodynamic_states)
        # initial assignment (multistatesampler.py:892-895, 1118-1143)
        if initial_thermodynamic_states is None:
            self._replica_thermodynamic_states = self._default_initial_thermodynamic_states(
                self._thermodynamic_states, self._sampler_states)
        else:
            init = np.array(initial_thermodynamic_states, dtype=np.int64)
            if len(init) != K or init.min() < 0 or init.max() >= M:
                raise ValueError('initial_thermodynamic_states must hold one valid state index per replica')
            self._replica_thermodynamic_states = init
        # one (deep-copied) move per state (multistatesampler.py:906-910)
        if isinstance(self._mcmc_moves, mcmc.MCMCMove):
            self._mcmc_moves = [copy.deepcopy(self._mcmc_moves) for _ in range(M)]
        elif len(self._mcmc_moves) != M:
            raise RuntimeError('The number of MCMCMoves ({}) and ThermodynamicStates ({}) must be the same.'.format(
                len(self._mcmc_moves), M))
        # (moves that differ between states are handed to the engine one by one: _apply_moves)
        self._n_accepted_matrix = np.zeros([M, M], np.int64)
        self._n_proposed_matrix = np.zeros([M, M], np.int64)
        self._energy_thermodynamic_states = np.zeros([K, M], np.float64)
        self._neighborhoods = np.ones([K, M], np.int8)
        self._energy_unsampled_states = np.zeros([K, len(self._unsampled_states)], np.float64)
        self._iteration = 0
        self._create_engine()

    @staticmethod
    def _default_initial_thermodynamic_states(thermodynamic_states, sampler_states):
        """multistatesampler.py:1118-1143: one-to-one when the counts match, otherwise whole loops over the states and the
        remainder spread evenly from the first to the last state."""
        n_thermo, n_sampler = len(thermodynamic_states), len(sampler_states)
        thermo_indices = np.arange(n_thermo, dtype=int)
        initial = np.zeros(n_sampler, dtype=int)
        loops = n_sampler // n_thermo
        n_looped = n_thermo * loops
        initial[:n_looped] = np.tile(thermo_indices, loops)
        initial[n_looped:] = np.linspace(0, n_thermo - 1, n_sampler - n_looped, dtype=int)
        return initial.astype(np.int64)

    # ------------------------------------------------------------------ engine plumbing
    def _create_engine(self):
        K = len(self._sampler_states)
        device = _backend.default_device(self.sampler_context_cache)
        self._engine = _backend.build_engine(self._thermodynamic_states, K, device=device, rank=self._rank,
                                             world_size=self._world_size)
        if self._world_size > 1:
            self._init_communicator()
        self._apply_moves()
        if self._seed is None:
            self._seed = int(np.random.SeedSequence().entropy & 0x7FFFFFFFFFFFFFFF)
            if self._world_size > 1:
                self._seed = self._bcast_int(self._seed)
        self._engine.set_replica_states(self._replica_thermodynamic_states)
        self._seed_mixing_streams()
        self._upload_sampler_states()
        self._pin_result_arrays()

    def _pin_result_arrays(self):
        """The matrices the engine writes every iteration (energies, swap statistics, permutation) move into page-locked
        memory, so that the engine's results land in them by direct DMA (no staging, no intermediate arrays)."""
        e = self._engine
        for name in ('_energy_thermodynamic_states', '_n_accepted_matrix', '_n_proposed_matrix'):
            a = getattr(self, name)
            b = e.pinned_array(a.shape, a.dtype)
            b[...] = a
            setattr(self, name, b)
        st = np.asarray(self._replica_thermodynamic_states, dtype=np.int64)
        self._replica_thermodynamic_states = e.pinned_array(st.shape, np.int64)
        self._replica_thermodynamic_states[...] = st

    def _apply_moves(self, moves=None):
        """The moves (default: the sampler's) go to the engine: one for all states, or -- when the states carry different moves
        (multistatesampler.py:906-910) -- one per state; a replica is propagated with the move of the state it is in
        (multistatesampler.py:1311-1322), inside the same fused launch.  The Metropolized moves of a move
        (mcmc.split_move) run before the dynamics, per state, with the counts the move objects hold."""
        own = moves is None
        moves = self._mcmc_moves if own else moves
        integrators = [mcmc.integrator_part(mv) for mv in moves]
        mcmc.check_hmc(integrators, self._thermodynamic_states[0].pressure)
        mv0 = integrators[0]
        mv0._set_on_engine(self._engine)
        self._reassign = bool(mv0.reassign_velocities)
        if own:
            self._n_restart = mv0.n_restart_attempts
        if any(not mcmc.same_integrator(mv, mv0) for mv in integrators[1:]):
            for l, mv in enumerate(integrators):
                mv._set_on_engine(self._engine, l)
        mc = [mcmc.split_move(mv)[0] for mv in moves]
        if any(mc) or self._mc_moves is not None:
            n = self._thermodynamic_states[0].n_particles
            self._engine.set_mc_moves([[m._engine_move(n) for m in ms] for ms in mc])
            self._mc_moves = mc if any(mc) else None
            if self._mc_moves:
                self._push_mc_statistics()

    # Monte Carlo move counts: the device keeps them per state and move slot, summed over the replicas a rank owns; the move
    # objects get the totals over every rank.  A move object that several states share (equilibrate with one move) gets the
    # sum over them.
    @staticmethod
    def _mc_counts_to_moves(mc, accepted, proposed):
        totals = {}
        for l, ms in enumerate(mc):
            for j, m in enumerate(ms):
                a, p = totals.get(id(m), (0, 0))
                totals[id(m)] = (a + int(accepted[l, j]), p + int(proposed[l, j]))
        for ms in mc:
            for m in ms:
                m.n_accepted, m.n_proposed = totals[id(m)]

    def _push_mc_statistics(self):
        """The counts of the move objects go to the device: all of them to rank 0, so that the ranks' sums are the totals."""
        acc = np.zeros((self.n_states, mcmc.RX_MAX_MC_MOVES), np.int64)
        prop = np.zeros_like(acc)
        seen = set()
        for l, ms in enumerate(self._mc_moves):
            for j, m in enumerate(ms):
                if id(m) not in seen and self._rank == 0:
                    acc[l, j], prop[l, j] = m.n_accepted, m.n_proposed
                seen.add(id(m))
        self._engine.set_mc_statistics(acc, prop)
        self._mc_last = (acc, prop)

    def _pull_mc_statistics(self):
        """The device counts, summed over the ranks (every rank takes part), into the move objects on rank 0."""
        acc, prop = self._engine.get_mc_statistics()
        if self._world_size > 1:
            from .._dist import default_communicator, sum_counts
            comm = self._communicator
            if comm is None:
                comm = self._communicator = default_communicator()
            both = sum_counts(comm, np.stack([acc, prop]))
            if self._rank != 0:
                return
            acc, prop = both
        self._mc_counts_to_moves(self._mc_moves, acc, prop)
        self._mc_last = (acc, prop)

    def _seed_mixing_streams(self):
        # the reference never seeds numba's / numpy's generators (os.urandom); a user seed makes runs reproducible
        self._engine.mix_seed(self._seed & 0xFFFFFFFF, _lib.RX_STREAM_NUMBA)
        self._engine.mix_seed((self._seed >> 16) & 0xFFFFFFFF, _lib.RX_STREAM_NUMPY)

    def _init_communicator(self):
        """Distribute an NCCL unique id (rank 0 creates it) and initialise the engine's communicator."""
        comm = self._communicator
        if comm is None:
            from .._dist import default_communicator
            comm = self._communicator = default_communicator()
        uid = self._engine.comm_unique_id() if self._rank == 0 else None
        uid = comm.bcast_bytes(uid, 128)
        self._engine.comm_init(uid)

    def _bcast_int(self, v):
        comm = self._communicator
        if comm is None:
            from .._dist import default_communicator
            comm = self._communicator = default_communicator()
        return int.from_bytes(comm.bcast_bytes(int(v).to_bytes(8, 'little') if self._rank == 0 else None, 8), 'little')

    @property
    def asynchronous_reporting(self):
        """True: the records of an iteration are written to storage by a writer thread while the next iteration runs
        (multistate/_async_writer.py); run() returns with everything on storage.  Default False (the reference's behaviour)."""
        return self._want_async_reporting

    @asynchronous_reporting.setter
    def asynchronous_reporting(self, on):
        self._want_async_reporting = bool(on)
        self._wrap_reporter()

    def _wrap_reporter(self):
        from ._async_writer import AsyncReporter
        r = self._reporter
        if r is None:
            return
        if self._want_async_reporting and not isinstance(r, AsyncReporter):
            self._reporter = AsyncReporter(r)
        elif not self._want_async_reporting and isinstance(r, AsyncReporter):
            r.shutdown()
            self._reporter = r._reporter

    class _HostStore:
        """Page-locked backing store of the owned SamplerStates: positions, velocities (K_loc, N, 3) and the energies the
        engine reported last; `dirty` is set by a SamplerState whose arrays were replaced (states.py)."""

        def __init__(self, x, v):
            self.x, self.v = x, v
            self.pot = np.zeros(len(x))
            self.kin = np.zeros(len(x))
            self.dirty = True   # states not attached yet

    def _attach_host_store(self):
        """One page-locked (K_loc, N, 3) pair is the backing store of the owned SamplerStates: their position / velocity
        arrays are views into it and their energies are read from it, so that the per-iteration exchange with the device
        is one copy each way and NO per-replica work on the host (the loops below only run when a caller assigned new
        arrays to a state)."""
        e = self._engine
        n = e.k1 - e.k0
        if n == 0 or self._host_x is not None:
            return
        N = self._sampler_states[0].n_particles
        self._host_x = e.pinned_array((n, N, 3))
        self._host_v = e.pinned_array((n, N, 3))
        self._host_v[:] = 0.0
        self._host_store = self._HostStore(self._host_x, self._host_v)
        for r, k in enumerate(range(e.k0, e.k1)):
            s = self._sampler_states[k]
            self._host_x[r] = s._positions
            s._positions = self._host_x[r]
            if s._velocities is not None:
                self._host_v[r] = s._velocities
                s._velocities = self._host_v[r]
            s._store, s._store_index = self._host_store, r

    def _collect_host_store(self):
        """Positions / velocities a caller replaced on a SamplerState go back into the backing store."""
        e = self._engine
        st = self._host_store
        if st is None or not st.dirty:
            return
        for r, k in enumerate(range(e.k0, e.k1)):
            s = self._sampler_states[k]
            if s._store is not st:
                s._store, s._store_index = st, r
            if s._positions.base is not self._host_x.base:
                self._host_x[r] = s._positions
                s._positions = self._host_x[r]
            if s._velocities is None:
                raise RuntimeError('host-resident sampler state %d has no velocities' % k)
            if s._velocities.base is not self._host_v.base:
                self._host_v[r] = s._velocities
                s._velocities = self._host_v[r]
        # (the dirty flag is cleared by _sync_sampler_states, which also re-attaches the energies)

    @property
    def _npt(self):
        return self._thermodynamic_states[0].pressure is not None

    @property
    def _anisotropic(self):
        return self._npt and _backend.barostat_scale(self._thermodynamic_states) is not None

    def _upload_sampler_states(self):
        e = self._engine
        K = len(self._sampler_states)
        x = np.stack([s._positions for s in self._sampler_states])
        e.set_positions(x)
        if self._npt:     # each replica propagates in its own box
            e.set_boxes(_backend.box_edges(self._sampler_states))
        have_v = [s._velocities is not None for s in self._sampler_states]
        if all(have_v):
            e.set_velocities(np.stack([s._velocities for s in self._sampler_states]))
        else:
            # replicas without velocities get Maxwell-Boltzmann ones (what BaseIntegratorMove.apply would do through
            # a fresh Context, mcmc.py:709-711)
            e.randomize_velocities(self._seed, 0)
            if any(have_v):
                for k, hv in enumerate(have_v):
                    if hv:
                        e.set_velocities(self._sampler_states[k]._velocities[None], first=k)
        # velocities drawn on the device are not on the host yet
        self._states_stale = not all(have_v)
        if self.host_resident_states:
            self._sync_sampler_states()

    def _sync_sampler_states(self):
        """Pull positions/velocities/energies of the owned replicas back into the host SamplerStates."""
        if self._engine is None or not self._states_stale:
            return
        e = self._engine
        self._attach_host_store()
        if e.k1 > e.k0:
            e.get_positions(out=self._host_x)
            e.get_velocities(out=self._host_v)
        pot, kin = e.get_replica_energies()
        if self._npt and e.k1 > e.k0:     # the barostat's boxes go back into the SamplerStates like the positions
            for r, edges in enumerate(e.get_boxes()):
                self._sampler_states[e.k0 + r]._box_vectors = np.diag(edges)
        st = self._host_store
        if st is not None:
            st.pot[:] = pot[e.k0:e.k1]
            st.kin[:] = kin[e.k0:e.k1]
        if st is not None and st.dirty:
            from ..states import _FROM_STORE
            hx, hv = self._host_x, self._host_v
            for r, k in enumerate(range(e.k0, e.k1)):
                s = self._sampler_states[k]
                s._store, s._store_index = st, r
                if s._positions.base is not hx.base:
                    s._positions = hx[r]
                if s._velocities is None or s._velocities.base is not hv.base:
                    s._velocities = hv[r]
                s._potential_energy = _FROM_STORE
                s._kinetic_energy = _FROM_STORE
            st.dirty = False
        self._states_stale = False

    # ------------------------------------------------------------------ run (multistatesampler.py:724-804)
    def run(self, n_iterations=None):
        if self._engine is None:
            raise RuntimeError('Cannot run a sampler that has not been created (call create()).')
        if self._is_completed():
            return
        if self._iteration == 0:
            self._compute_energies()
            if self._reporter is not None and self._rank == 0:      # multistatesampler.py:741-746
                self._reporter.write_energies(self._energy_thermodynamic_states, self._neighborhoods,
                                              self._energy_unsampled_states, 0)
            self._record_offline_inputs()
            self._check_nan_energy()
        iteration_limit = self.number_of_iterations if n_iterations is None else \
            min(self._iteration + n_iterations, self.number_of_iterations)
        timer_start = time.time()
        run_initial_iteration = self._iteration
        while not self._is_completed(iteration_limit):
            self._iteration += 1
            t0 = time.time()
            self._replica_thermodynamic_states = self._mix_replicas()
            t1 = time.time()
            self._propagate_replicas()
            t2 = time.time()
            self._compute_energies()
            t3 = time.time()
            self._report_iteration()
            self._record_offline_inputs()
            self._update_analysis()
            self._update_timing(t3 - t0, time.time() - timer_start, run_initial_iteration, iteration_limit,
                                phases=(t1 - t0, t2 - t1, t3 - t2))
            self._check_nan_energy()
        if self._want_async_reporting and self._reporter is not None:
            self._reporter.drain()     # run() returns with every record on storage

    def extend(self, n_iterations):
        if self._iteration + n_iterations > self.number_of_iterations:
            self.number_of_iterations = self._iteration + n_iterations
        self.run(n_iterations)

    def equilibrate(self, n_iterations, mcmc_moves=None):
        """propagate -> energies -> mix without advancing the iteration counter (multistatesampler.py:649-720)."""
        if self._engine is None:
            raise RuntimeError('Cannot equilibrate a sampler that has not been created.')
        if mcmc_moves is not None:
            mv = mcmc_moves if isinstance(mcmc_moves, mcmc.MCMCMove) else mcmc_moves[0]
            if self._mc_moves:     # the sampler's own moves keep their counts
                self._pull_mc_statistics()
            self._apply_moves([mv] * self.n_states)
        reassign = self._reassign
        self._equil_counter = getattr(self, '_equil_counter', 0)
        for _ in range(n_iterations):
            self._equil_counter += 1
            self._propagate_replicas(iteration=(1 << 40) + self._equil_counter, reassign=reassign)
            self._compute_energies()
            self._replica_thermodynamic_states = self._mix_replicas()
        if mcmc_moves is not None:
            if self._mc_moves:
                self._pull_mc_statistics()
            self._apply_moves()

    def minimize(self, tolerance=1.0 * unit.kilojoules_per_mole / unit.nanometers, max_iterations=0):
        """Minimize all replicas, each in its current thermodynamic state (multistatesampler.py:611-647).

        One fused FIRE launch (``rx_minimize``) in place of the per-replica FIRE -> L-BFGS of
        ``_minimize_replica`` (multistatesampler.py:1339-1402); ``tolerance`` bounds the RMS force component.
        Minimized positions are stored at the end, velocities are left as they are.
        """
        if self._engine is None or self.n_replicas == 0:
            raise RuntimeError('Cannot minimize replicas. The simulation must be created first.')
        tol = float(unit.to_md(tolerance, unit.kilojoules_per_mole / unit.nanometers, 'tolerance'))
        e = self._engine
        self._sync_sampler_states()
        rms, n_it = e.minimize(tol, max_iterations)
        x = e.get_positions()
        for r, k in enumerate(range(e.k0, e.k1)):
            self._sampler_states[k].positions = unit.Quantity(x[r], unit.nanometer)
        self._last_minimization = {'rms_force': rms[e.k0:e.k1].copy(), 'iterations': n_it[e.k0:e.k1].copy()}
        if self._reporter is not None:
            if self._world_size > 1:
                self._gather_sampler_states()
                if self._npt:
                    self._last_npt_records = self._gather_npt_records()
                if self._anisotropic:
                    self._last_aniso_records = self._gather_aniso_records()
            if self._rank == 0:
                self._reporter.write_sampler_states(self._sampler_states, self._iteration, extra=self._checkpoint_extra())

    # ------------------------------------------------------------------ the three hooks
    def _mix_replicas(self):
        """Base class: no swaps (multistatesampler.py:1500-1517)."""
        self._n_accepted_matrix[:, :] = 0
        self._n_proposed_matrix[:, :] = 0
        return self._replica_thermodynamic_states

    def _propagate_replicas(self, iteration=None, reassign=None):
        """One fused launch propagates every owned replica in its current state (multistatesampler.py:1287-1337)."""
        e = self._engine
        if self.host_resident_states:
            # reference semantics: sampler states live on the host and are pushed to the device every iteration
            # (SamplerState.apply_to_context, mcmc.py:709)
            self._sync_sampler_states()
            self._attach_host_store()
            if e.k1 > e.k0:
                self._collect_host_store()
                e.set_positions(self._host_x, first=e.k0)
                e.set_velocities(self._host_v, first=e.k0)
        it = self._iteration if iteration is None else iteration
        n_restart = self._n_restart
        re = self._reassign if reassign is None else reassign
        for attempt in range(n_restart + 1):
            try:
                if attempt == 0:
                    e.propagate(self._seed, it, re)
                else:
                    # restart policy of mcmc.py:706-759: ONLY the replicas that failed go back to the state they had at
                    # the start of this iteration (a device-side snapshot taken by rx_propagate) and run again with
                    # other noise; the replicas that came through keep their result
                    e.propagate_retry(self._seed + attempt * 0x9E3779B9, it, re)
                break
            except EngineError as err:
                if err.code != _lib.RX_ERR_NAN:
                    raise
                if attempt == n_restart:
                    bad = np.nonzero(err.nan_flags)[0]
                    raise SimulationNaNError('Propagating replica {} at state {} resulted in a NaN!'.format(
                        bad[0], self._replica_thermodynamic_states[bad[0]]))
        self._states_stale = True
        if self.host_resident_states:
            self._sync_sampler_states()

    def _compute_energies(self):
        """u[k, l] for all replicas and states in one launch (+ NCCL all-gather) (multistatesampler.py:1436-1494)."""
        if self.locality is None:
            self._engine.compute_energies(out=self._energy_thermodynamic_states)
            self._neighborhoods[:, :] = 1
            u = self._energy_thermodynamic_states
        else:
            u = self._engine.compute_energies()
            # only the states within `locality` of each replica's current state are (re)written, the rest keeps its old
            # value exactly as in the reference (multistatesampler.py:1263-1281,1441-1456); the device matrix is complete,
            # and swap-neighbors (forced by locality, replicaexchange.py:228-230) only reads entries inside the band
            M = self.n_states
            self._neighborhoods[:, :] = 0
            for k, st in enumerate(self._replica_thermodynamic_states):
                lo, hi = max(0, st - self.locality), min(M, st + self.locality + 1)
                self._neighborhoods[k, lo:hi] = 1
                self._energy_thermodynamic_states[k, lo:hi] = u[k, lo:hi]
        if self._unsampled_states:
            # energies at states that are evaluated but never sampled (multistatesampler.py:1452-1456,1489-1494)
            if self._unsampled_table is None:
                both = list(self._thermodynamic_states[:1]) + list(self._unsampled_states)
                _, self._unsampled_table = _backend.engine_tables(both)
                self._unsampled_table = {k: v[1:] for k, v in self._unsampled_table.items()}
                npt = _backend.pressure_tables(both)
                if npt is not None:     # (the dispersion corrections go to the engine as c_l / V)
                    self._unsampled_table.update(energy_offset=np.zeros(len(self._unsampled_states)), pressure=npt[0][1:],
                                                 dispersion=npt[1][1:])
            self._energy_unsampled_states[:, :] = self._engine.compute_energies_at(**self._unsampled_table)

    # ------------------------------------------------------------------ bookkeeping
    def _initialize_reporter(self):
        """Write everything that identifies the run plus iteration 0 (multistatesampler.py:1169-1187); rank 0 only."""
        if self._reporter is None or self._rank != 0:
            return
        r = self._reporter
        if r.is_open():
            r.close()
        r.open('w')
        r.set_dimensions(self.n_replicas, self.n_states, self._thermodynamic_states[0].n_particles)
        r.write_thermodynamic_states(self._thermodynamic_states, self._unsampled_states)
        r.write_mcmc_moves(self._mcmc_moves)
        opts = {k: getattr(self, k, None) for k in self._STORED_OPTIONS if hasattr(self, k)}
        if opts.get('number_of_iterations') == np.inf:
            opts['number_of_iterations'] = 'inf'
        opts['seed'] = self._seed
        r.write_dict('options', opts)
        r.write_dict('metadata', self._metadata)
        self._report_iteration()

    def _checkpoint_extra(self):
        e = self._engine
        extra = dict(seed=int(self._seed), iteration=int(self._iteration),
                     mt_numba_words=int(e.mix_stream_position(_lib.RX_STREAM_NUMBA)),
                     mt_numpy_words=int(e.mix_stream_position(_lib.RX_STREAM_NUMPY)),
                     equil_counter=int(getattr(self, '_equil_counter', 0)))
        if self._mc_moves:        # the move counts as of the last report (rank 0: the totals over the ranks)
            extra['mc_accepted'], extra['mc_proposed'] = (a.tolist() for a in self._mc_last)
        if self._npt:     # (rank 0: the records gathered for this iteration's report)
            rec = self._last_npt_records if self._world_size > 1 else self._local_npt_records()
            extra['barostat'] = dict(volume_scale=rec[:, 3].tolist(),
                                     **{f: [int(q) for q in rec[:, c]] for c, f in ((4, 'step'), (5, 'n_attempted'), (6, 'n_accepted'))})
        if self._anisotropic:
            rec = self._last_aniso_records if self._world_size > 1 else self._local_aniso_records()
            extra['barostat_anisotropic'] = dict(volume_scale=rec[:, 0].tolist(),
                                                 **{f: [[int(q) for q in row] for row in rec[:, c]]
                                                    for c, f in ((1, 'n_attempted'), (2, 'n_accepted'))})
        return extra

    def _report_iteration(self):
        """multistatesampler.py:1191-1207: states, checkpointed positions, mixing statistics, energies, commit marker."""
        if self._reporter is None:
            self._report_iteration_items()
            return
        it = self._iteration
        checkpoint = (it % self._reporter.checkpoint_interval == 0)
        analysis = self._reporter.wants_analysis_states(it)   # per-iteration streams of the analysis particles
        if checkpoint or analysis:
            self._sync_sampler_states()
            if self._world_size > 1:
                self._gather_sampler_states()
        npt = self._last_npt_records = self._gather_npt_records() if self._npt else None
        self._last_aniso_records = self._gather_aniso_records() if self._anisotropic else None
        if self._mc_moves:
            self._pull_mc_statistics()
        if self._rank != 0:
            self._report_iteration_items()
            return
        r = self._reporter
        r.write_replica_thermodynamic_states(self._replica_thermodynamic_states, it)
        if npt is not None:      # the reference's per-iteration 'volumes' (multistatereporter.py:1640-1651)
            r.write_volumes(np.prod(npt[:, :3], axis=1), it)
        if checkpoint or analysis:
            r.write_sampler_states(self._sampler_states, it, extra=self._checkpoint_extra())
        r.write_mixing_statistics(self._n_accepted_matrix, self._n_proposed_matrix, it)
        if self._mc_moves:        # the moves with their counts, at every reported iteration (multistatesampler.py:1219)
            r.write_mcmc_moves(self._mcmc_moves)
        r.write_energies(self._energy_thermodynamic_states, self._neighborhoods, self._energy_unsampled_states, it)
        self._report_iteration_items()      # subclass records (SAMS) go in before the commit marker
        r.write_last_iteration(it)

    def _report_iteration_items(self):
        """Hook: per-iteration records of a subclass, written before the commit marker."""

    def _gather_sampler_states(self):
        """Multi-GPU checkpoint: every rank sends its shard of positions/velocities/energies to rank 0 (the role of
        mpiplus.distribute(..., send_results_to=0), multistatesampler.py:1296-1302)."""
        e = self._engine
        comm = self._communicator
        if comm is None:
            from .._dist import default_communicator
            comm = self._communicator = default_communicator()
        npt = self._local_npt_records() if self._npt else None
        shard = [(k, s._positions, s._velocities) + s._energies_md() + (None if npt is None else npt[r],)
                 for r, (k, s) in enumerate(zip(range(e.k0, e.k1), self._sampler_states[e.k0:e.k1]))]
        gathered = comm.gather_object(shard)
        if self._rank == 0:
            for part in gathered:
                for k, x, v, pe, ke, rec in part:
                    if not (e.k0 <= k < e.k1):   # (this rank's own states are already current)
                        self._sampler_states[k]._update(x, v, pe, ke)
                        if rec is not None:
                            self._sampler_states[k]._box_vectors = np.diag(rec[:3])

    def _local_npt_records(self):
        """(K_loc, 7): box edges and barostat state (volume_scale, step, n_attempted, n_accepted) of the owned replicas."""
        e = self._engine
        if e.k1 == e.k0:
            return np.zeros((0, 7))
        b = e.get_barostat()
        return np.column_stack([e.get_boxes(), b['volume_scale'], b['step'], b['n_attempted'], b['n_accepted']])

    def _gather_npt_records(self):
        """(K, 7) records of every replica on rank 0 (None elsewhere); every rank takes part."""
        rec = self._local_npt_records()
        if self._world_size == 1:
            return rec
        e = self._engine
        comm = self._communicator
        if comm is None:
            from .._dist import default_communicator
            comm = self._communicator = default_communicator()
        shard = [(k, np.zeros((0, 3)), None, None, None, rec[r]) for r, k in enumerate(range(e.k0, e.k1))]
        gathered = comm.gather_object(shard)
        if self._rank != 0:
            return None
        out = np.zeros((self.n_replicas, 7))
        for part in gathered:
            for item in part:
                out[item[0]] = item[5]
        return out

    def _local_aniso_records(self):
        """(K_loc, 3, 3): per-axis volume_scale, n_attempted and n_accepted of the owned replicas' anisotropic barostat."""
        e = self._engine
        if e.k1 == e.k0:
            return np.zeros((0, 3, 3))
        a = e.get_barostat_anisotropic()
        return np.stack([a['volume_scale'], a['n_attempted'], a['n_accepted']], axis=1).astype(np.float64)

    def _gather_aniso_records(self):
        """(K, 3, 3) records of every replica on rank 0 (None elsewhere), carried as the position rows of a shard;
        every rank takes part."""
        rec = self._local_aniso_records()
        if self._world_size == 1:
            return rec
        e = self._engine
        comm = self._communicator
        if comm is None:
            from .._dist import default_communicator
            comm = self._communicator = default_communicator()
        gathered = comm.gather_object([(k, rec[r], None, None, None) for r, k in enumerate(range(e.k0, e.k1))])
        if self._rank != 0:
            return None
        out = np.zeros((self.n_replicas, 3, 3))
        for part in gathered:
            for item in part:
                out[item[0]] = item[1]
        return out

    # ------------------------------------------------------------------ online analysis (multistatesampler.py:1625-1695)
    @staticmethod
    def _online_f_k_update(f_k, u, replica_states, locality, iteration, gamma0=1.0):
        """One stochastic-approximation step of the online free-energy estimate (multistatesampler.py:1625-1664):
        every replica adds gamma * P(l | x_k) over its neighbourhood to logZ_l, gamma = gamma0 / (iteration + 1), then
        logZ is shifted so that logZ_0 = 0.  Returns the new f_k = -logZ."""
        u = np.asarray(u, dtype=np.float64)
        K, M = u.shape
        st = np.asarray(replica_states)
        logZ = -np.asarray(f_k, dtype=np.float64)
        if locality is None:
            log_p = -u                      # (every state is in every replica's neighbourhood: no mask to build)
        else:
            l = np.arange(M)[None, :]
            mask = (l >= st[:, None] - locality) & (l <= st[:, None] + locality)
            log_p = np.where(mask, -u, -np.inf)
        top = log_p.max(axis=1, keepdims=True)
        p = log_p - top
        np.exp(p, out=p)
        p /= p.sum(axis=1, keepdims=True)
        logZ = logZ + (gamma0 / float(iteration + 1)) * p.sum(axis=0)
        return -(logZ - logZ[0])

    def _online_analysis(self, gamma0=1.0):
        if self._last_mbar_f_k is None:
            self._last_mbar_f_k = np.zeros(self.n_states)
        self._last_mbar_f_k = self._online_f_k_update(self._last_mbar_f_k, self._energy_thermodynamic_states,
                                                      self._replica_thermodynamic_states, self.locality,
                                                      self._iteration, gamma0)
        self._last_err_free_energy = np.inf
        if self._reporter is not None and self._rank == 0:
            free_energy = self._last_mbar_f_k[-1] - self._last_mbar_f_k[0]
            self._reporter.write_online_data_dynamic_and_static(
                self._iteration, f_k=self._last_mbar_f_k, free_energy=np.array([free_energy, self._last_err_free_energy]))
        return self._last_err_free_energy

    def _update_analysis(self):
        """multistatesampler.py:1676-1695.  The online estimate runs every iteration and sets the error to +inf; every
        ``online_analysis_interval`` iterations of a run with storage, the offline MBAR pass sets it to the standard error
        of the free energy between the end states, so a run can stop only at those iterations.  Rank 0 runs the pass and
        every rank gets its error, so that all stop at the same iteration.  Runs with ``locality`` have no pass (MBAR of
        them is not implemented)."""
        if self.online_analysis_interval is None:
            return
        self._last_err_free_energy = self._online_analysis()
        if self._iteration % self.online_analysis_interval != 0 or self._reporter is None or self.locality is not None:
            return
        err = self._offline_analysis() if self._rank == 0 and self._offline_inputs is not None else None
        if self._world_size > 1:
            err = self._bcast_error(err)
        if err is not None:
            self._last_err_free_energy = err

    @property
    def _keeps_offline_inputs(self):
        return (self._rank == 0 and self._reporter is not None and self.locality is None
                and self.online_analysis_interval is not None and not self._offline_stopped)

    def _log_weights_and_logZ(self):
        """Hook: (log weights, logZ) of a sampler whose state weights change during the run (SAMS), else None."""
        return None

    def _stop_offline_analysis(self, err):
        if err.code != _lib.RX_ERR_UNSUPPORTED:
            raise err
        logger.warning('offline free-energy analysis stops for the rest of this run: %s', err.message)
        self._offline_stopped = True
        self._offline_inputs = None

    def _record_offline_inputs(self):
        """What the offline pass needs of the iteration just reported (rank 0 of a run with storage): the energy matrices
        go to the engine's device history; the host keeps u[r, s_r(t)] of the K replicas, their states and, for SAMS, the
        log weights."""
        if not self._keeps_offline_inputs:
            return
        it = self._iteration
        rec = self._offline_inputs
        if it == 0 or rec is None:
            rec = self._offline_inputs = {'u': [], 'states': [], 'log_weights': None}
        if it > len(rec['u']):
            # iterations ran without reports (run_fused): the history has a gap the analyzer of the storage would not see
            logger.warning('offline free-energy analysis stops for the rest of this run: iterations %d..%d were not '
                           'reported', len(rec['u']), it - 1)
            self._offline_stopped = True
            self._offline_inputs = None
            return
        try:
            self._engine.history_append(it, len(self._unsampled_states))
        except EngineError as err:
            self._stop_offline_analysis(err)
            return
        st = np.array(self._replica_thermodynamic_states, dtype=np.int64)
        del rec['u'][it:], rec['states'][it:]
        rec['u'].append(self._energy_thermodynamic_states[np.arange(len(st)), st])
        rec['states'].append(st)
        lw = self._log_weights_and_logZ()
        if lw is not None:
            if rec['log_weights'] is None:
                rec['log_weights'] = []
            del rec['log_weights'][it:]
            rec['log_weights'].append(np.array(lw[0], dtype=np.float64))

    def _offline_analysis(self):
        """The reference's offline pass (multistatesampler.py:1526-1620): the decisions of MultiStateSamplerAnalyzer
        (effective-energy timeseries, equilibration, subsampling, initial_f_k = the previous pass's f_k) on iterations
        0..t, from the inputs kept in memory; MBAR's u_kn is gathered on the device from the engine's energy history.
        Returns the standard error of Delta f between the end states (NaN becomes +inf), or None when MBAR fails (then
        nothing is written and the previous error stands)."""
        rec = self._offline_inputs
        it = self._iteration
        M, U = self.n_states, len(self._unsampled_states)
        if self._last_mbar_f_k_offline is None:
            self._last_mbar_f_k_offline = np.zeros(M + U)
        try:
            states = np.stack(rec['states'], axis=1)
            log_weights, f_l = None, None
            lw = self._log_weights_and_logZ()
            if lw is not None:
                log_weights, f_l = np.stack(rec['log_weights'], axis=1), -np.asarray(lw[1], dtype=np.float64)
            u_n = effective_energy_timeseries(np.stack(rec['u'], axis=1), states, log_weights, f_l)
            # t0 = 1: iteration 0 is discarded.  SAMS stores its t0 per iteration, not as the static record the analyzer
            # looks for, so the analyzer starts at 1 as well.
            n_equilibration, g_t, n_effective = equilibration_data(u_n, 1, 100)
            selected = decorrelated_iterations(n_equilibration, g_t, it)
            first = U // 2          # the unsampled states at both ends, as MultiStateSamplerAnalyzer lays out u_kn
            columns = np.zeros(M + U, dtype=np.int32)
            columns[first:first + M] = np.arange(M)
            if U > 0:
                columns[[0, -1]] = (M, M + U - 1)
            N_k = np.zeros(M + U, dtype=np.int64)
            visited, counts = np.unique(states[:, selected], return_counts=True)
            N_k[first + visited] = counts
            mbar = MBAR.from_history(self._engine, selected, columns, N_k, initial_f_k=self._last_mbar_f_k_offline)
            try:
                r = mbar.compute_free_energy_differences()
            finally:
                mbar.close()
        except (MBARConvergenceError, ValueError) as err:
            logger.debug('offline free-energy analysis at iteration %d failed: %s', it, err)
            return None
        self._last_mbar_f_k_offline = mbar.f_k
        free_energy, err = float(r['Delta_f'][0, -1]), float(r['dDelta_f'][0, -1])
        if np.isnan(err):
            err = np.inf
        self._reporter.write_online_data_dynamic_and_static(it, f_k_offline=self._last_mbar_f_k_offline,
                                                            free_energy=np.array([free_energy, err]))
        self._reporter.write_current_statistics({
            'iteration': it, 'percent_complete': it * 100 / self.number_of_iterations,
            'mbar_analysis': {'free_energy_in_kT': free_energy, 'standard_error_in_kT': err,
                              'number_of_uncorrelated_samples': float(n_effective),
                              'n_equilibrium_iterations': int(n_equilibration),
                              'statistical_inefficiency': float(g_t)},
            'timing_data': self._timing_data})
        return err

    def _bcast_error(self, err):
        comm = self._communicator
        if comm is None:
            from .._dist import default_communicator
            comm = self._communicator = default_communicator()
        data = struct.pack('<d', np.nan if err is None else err) if self._rank == 0 else None
        v = struct.unpack('<d', comm.bcast_bytes(data, 8))[0]
        return None if np.isnan(v) else v

    def _is_completed(self, iteration_limit=None):
        if iteration_limit is None:
            iteration_limit = self.number_of_iterations
        return self._iteration is not None and self._is_completed_static(
            iteration_limit, self._iteration, self._last_err_free_energy, self.online_analysis_target_error)

    @staticmethod
    def _is_completed_static(iteration_limit, iteration, last_err_free_energy, online_analysis_target_error):
        """multistatesampler.py:1722-1739: the iteration limit is reached, or the last error is at or below the target."""
        return iteration >= iteration_limit or (
            last_err_free_energy is not None and last_err_free_energy <= online_analysis_target_error)

    def _check_nan_energy(self):
        """multistatesampler.py:1049-1081"""
        diag = self._energy_thermodynamic_states[np.arange(self.n_replicas), self._replica_thermodynamic_states]
        if np.any(np.isnan(diag)):
            bad = np.nonzero(np.isnan(diag))[0]
            raise SimulationNaNError('NaN encountered in energies for replicas {}'.format(bad.tolist()))

    def _update_timing(self, iteration_time, partial_total_time, run_initial_iteration, iteration_limit, phases=None):
        """Timing dictionary with the reference's keys (multistatesampler.py:1766-1803)."""
        t = self._timing_data
        t['iteration_seconds'] = iteration_time
        t['average_seconds_per_iteration'] = partial_total_time / max(self._iteration - run_initial_iteration, 1)
        t['estimated_time_remaining'] = t['average_seconds_per_iteration'] * (iteration_limit - self._iteration)
        t['estimated_total_time'] = t['average_seconds_per_iteration'] * self.number_of_iterations \
            if np.isfinite(self.number_of_iterations) else np.inf
        mv = mcmc.integrator_part(self._mcmc_moves[0])
        try:
            dt_ns = unit.to_md(mv.timestep) * mv.n_steps * 1e-3
            t['ns_per_day'] = dt_ns / (t['average_seconds_per_iteration'] / 86400.0)
        except Exception:
            t['ns_per_day'] = None
        if phases is not None:
            t['mixing_seconds'], t['propagation_seconds'], t['energy_seconds'] = phases
        t['device_phase_ms'] = self._engine.phase_times()

    def __del__(self):
        try:
            if self._engine is not None:
                self._engine.close()
        except Exception:
            pass
