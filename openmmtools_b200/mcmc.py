"""MCMC moves of the replica-exchange path: Langevin splitting dynamics and Monte Carlo rigid-body moves on the CUDA engine.

Mirrors /root/reference/openmmtools/mcmc.py: ``LangevinSplittingDynamicsMove`` (:1175-1316),
``LangevinDynamicsMove`` (:1023-1172), ``BaseIntegratorMove.apply`` (:668-776) and ``IntegratorMoveError``
(:538-600).  The splitting grammar and its validation follow ``integrators.LangevinIntegrator``
(/root/reference/openmmtools/integrators.py:1319-1363,1474-1537): tokens R, V, O; force groups (``V0``),
Metropolization (``{ }``), shadow-work and heat bookkeeping need per-substep energy sums and are not provided.

``MetropolizedMove`` (:810-970), ``MCDisplacementMove`` (:1704-1770), ``MCRotationMove`` (:1777-1911) and
``SequenceMove`` (:350-437) run as launches before the Langevin kernels (rx_set_state_mc_moves): a move is one
Metropolized move, one Langevin move, or a ``SequenceMove`` of up to ``RX_MAX_MC_MOVES`` = 4 Metropolized moves followed
by at most one Langevin move (none: the replicas take no dynamics steps).  On a periodic box a rotation makes its subset
whole by minimum image from the subset's first atom and rejects a proposal that would put a rotated atom half a box edge
or more from that atom.

``HMCMove`` (:1493-1594, ``integrators.HMCIntegrator`` :885-1012) runs inside the same fused propagation kernels
(rx_set_hmc_integrator) on the LJ fluid, the harmonic oscillator and molecules (constrained); it takes the place of the
Langevin move, alone or after the Metropolized moves of a ``SequenceMove``.  GHMC/barostat/weighted moves are other kernels and out of scope.
"""
import copy
import numpy as np
from . import unit
from . import _backend
from ._engine import EngineError
from . import _lib


class IntegratorMoveError(Exception):
    """The integrator produced NaN (mcmc.py:538-600)."""

    def __init__(self, message, move, context=None):
        super().__init__(message)
        self.move = move
        self.context = context

    def serialize_error(self, path_files_prefix):
        """Dump what is available for post-mortem (the reference writes system/integrator/state XML)."""
        import json
        with open(path_files_prefix + '-move.json', 'w') as f:
            json.dump({k: str(v) for k, v in self.move.__getstate__().items()}, f)


def parse_splitting(splitting):
    """Validate a splitting string, returning it without spaces (integrators.py:1319-1402; behaviour per string pinned
    by tests/golden/splitting_golden.json).  ``V0`` is the plain ``V`` of a system whose forces all sit in group 0."""
    tokens = splitting.split()
    steps = []
    groups = set()
    for step in tokens:
        if step in ('{', '}'):
            raise NotImplementedError('Metropolized splittings ({ }) are not provided on the GPU path')
        if step[0] == 'V' and len(step) > 1:
            try:
                group = int(step[1:])
            except ValueError:
                raise ValueError('You must use an integer force group')
            if group > 31:
                raise ValueError('OpenMM only allows up to 32 force groups')
            groups.add(group)
            steps.append('V')
            continue
        if step not in ('R', 'V', 'O'):
            raise ValueError("Invalid step name '{}' used; valid step names are R, V, O".format(step))
        steps.append(step)
    if groups - {0}:
        raise NotImplementedError('multiple-time-step splittings (V<group>) are not provided on the GPU path')
    joined = ''.join(steps)
    for need in 'RVO':
        assert need in joined, 'splitting must contain R, V and O steps'
    return joined


class MCMCMove:
    """Interface: ``apply(thermodynamic_state, sampler_state, context_cache=None)`` mutates the sampler state
    (mcmc.py:143-175)."""

    def apply(self, thermodynamic_state, sampler_state, context_cache=None):
        raise NotImplementedError


class BaseIntegratorMove(MCMCMove):
    def __init__(self, n_steps, reassign_velocities=False, n_restart_attempts=4, context_cache=None):
        self.n_steps = n_steps
        self.reassign_velocities = reassign_velocities
        self.n_restart_attempts = n_restart_attempts
        self.context_cache = context_cache
        self._seed_counter = 0

    # engine-facing description: (timestep ps, collision rate 1/ps, n_steps, splitting)
    def _integrator_parameters(self):
        raise NotImplementedError

    def _set_on_engine(self, engine, state=None):
        """This move as the engine's move for every state (state None) or for one state."""
        dt, gamma, n_steps, splitting = self._integrator_parameters()
        if state is None:
            engine.set_integrator(dt, gamma, n_steps, splitting)
        else:
            engine.set_state_integrator(state, dt, gamma, n_steps, splitting, bool(self.reassign_velocities))

    def apply(self, thermodynamic_state, sampler_state, context_cache=None):
        """Propagate one replica (mcmc.py:668-776): builds a single-replica engine, steps, updates the state.
        NaN -> retry up to n_restart_attempts times, then IntegratorMoveError (mcmc.py:706-759)."""
        _apply_one_replica(self, [], self, thermodynamic_state, sampler_state, context_cache)

    def __getstate__(self):
        return dict(n_steps=self.n_steps, reassign_velocities=self.reassign_velocities,
                    n_restart_attempts=self.n_restart_attempts)

    def __setstate__(self, s):
        self.n_steps = s['n_steps']
        self.reassign_velocities = s['reassign_velocities']
        self.n_restart_attempts = s['n_restart_attempts']
        self.context_cache = None
        self._seed_counter = 0


class LangevinSplittingDynamicsMove(BaseIntegratorMove):
    """Langevin dynamics with an arbitrary R/V/O splitting (mcmc.py:1175-1316); default "V R O R V" (BAOAB)."""

    def __init__(self, timestep=1.0 * unit.femtosecond, collision_rate=10.0 / unit.picoseconds, n_steps=1000,
                 reassign_velocities=False, splitting="V R O R V", constraint_tolerance=1.0e-8,
                 measure_shadow_work=False, measure_heat=False, **kwargs):
        super().__init__(n_steps=n_steps, reassign_velocities=reassign_velocities, **kwargs)
        if measure_shadow_work or measure_heat:
            raise NotImplementedError('shadow-work / heat bookkeeping is not provided on the GPU path')
        parse_splitting(splitting)
        self.timestep = timestep
        self.collision_rate = collision_rate
        self.splitting = splitting
        self.constraint_tolerance = constraint_tolerance
        self.measure_shadow_work = measure_shadow_work
        self.measure_heat = measure_heat

    def _integrator_parameters(self):
        return (float(unit.to_md(self.timestep, unit.picosecond, 'timestep')),
                float(unit.to_md(self.collision_rate, unit.picosecond ** -1, 'collision_rate')),
                int(self.n_steps), parse_splitting(self.splitting))

    def __getstate__(self):
        s = super().__getstate__()
        s.update(timestep=self.timestep, collision_rate=self.collision_rate, splitting=self.splitting,
                 constraint_tolerance=self.constraint_tolerance, measure_shadow_work=self.measure_shadow_work,
                 measure_heat=self.measure_heat)
        return s

    def __setstate__(self, s):
        super().__setstate__(s)
        for k in ('timestep', 'collision_rate', 'splitting', 'constraint_tolerance', 'measure_shadow_work', 'measure_heat'):
            setattr(self, k, s[k])


class LangevinDynamicsMove(BaseIntegratorMove):
    """Langevin dynamics with OpenMM's LangevinMiddleIntegrator discretisation (mcmc.py:1023-1172): per step
    v += dt f/m ; x += dt/2 v ; v = a v + b sqrt(kT/m) xi ; x += dt/2 v, i.e. the splitting "V R O R"."""

    def __init__(self, timestep=1.0 * unit.femtosecond, collision_rate=10.0 / unit.picoseconds, n_steps=1000,
                 reassign_velocities=False, constraint_tolerance=1e-8, **kwargs):
        super().__init__(n_steps=n_steps, reassign_velocities=reassign_velocities, **kwargs)
        self.timestep = timestep
        self.collision_rate = collision_rate
        self.constraint_tolerance = constraint_tolerance

    def _integrator_parameters(self):
        return (float(unit.to_md(self.timestep, unit.picosecond, 'timestep')),
                float(unit.to_md(self.collision_rate, unit.picosecond ** -1, 'collision_rate')),
                int(self.n_steps), 'VROR')

    def __getstate__(self):
        s = super().__getstate__()
        s.update(timestep=self.timestep, collision_rate=self.collision_rate, constraint_tolerance=self.constraint_tolerance)
        return s

    def __setstate__(self, s):
        super().__setstate__(s)
        for k in ('timestep', 'collision_rate', 'constraint_tolerance'):
            setattr(self, k, s[k])


class HMCMove(BaseIntegratorMove):
    """Hybrid Monte Carlo (mcmc.py:1493-1594 -> integrators.HMCIntegrator, integrators.py:885-1012).

    One trial draws the velocities from the Maxwell-Boltzmann distribution, takes ``n_steps`` velocity-Verlet steps of
    ``timestep`` and keeps the new positions with probability min(1, exp(-(Enew - Eold)/kT)), E = kinetic + potential;
    a rejected trial restores the positions and keeps the velocities the trajectory ended with.  As in the reference,
    ``apply`` runs ``n_steps`` such trials (``BaseIntegratorMove.apply`` calls ``integrator.step(n_steps)`` and one step of
    ``HMCIntegrator(nsteps=n_steps)`` is a whole trial): n_steps**2 force evaluations, 10**6 at the default n_steps=1000.

    Runs on the LJ fluid, the harmonic oscillator and molecules (positions and velocities constrained as in the reference's
    program) at constant volume; constant pressure and samplers whose states mix HMC and Langevin moves raise
    NotImplementedError.  The engine counts accepted and attempted trials per replica (``Engine.get_hmc_statistics``)."""

    def __init__(self, timestep=1.0 * unit.femtosecond, n_steps=1000, **kwargs):
        super().__init__(n_steps=n_steps, **kwargs)
        self.timestep = timestep

    def _integrator_parameters(self):
        return float(unit.to_md(self.timestep, unit.picosecond, 'timestep')), 0.0, int(self.n_steps), 'HMC'

    def _set_on_engine(self, engine, state=None):
        dt, _, n_steps, _ = self._integrator_parameters()
        if state is None:
            engine.set_hmc_integrator(dt, n_steps)
        else:
            engine.set_state_hmc_integrator(state, dt, n_steps)

    def __getstate__(self):
        serialization = super().__getstate__()
        serialization['timestep'] = self.timestep
        return serialization

    def __setstate__(self, serialization):
        super().__setstate__(serialization)
        self.timestep = serialization['timestep']


def check_hmc(integrators, pressure=None):
    """NotImplementedError for what the HMC kernels do not run: HMC under a barostat, or states that mix HMC and Langevin
    moves (one fused launch runs one kind of move)."""
    hmc = [isinstance(m, HMCMove) for m in integrators]
    if not any(hmc):
        return
    if not all(hmc):
        raise NotImplementedError('the states mix HMCMove and Langevin moves; one launch runs one kind of move: give every '
                                  'state an HMCMove (timesteps and n_steps may differ) or none')
    if pressure is not None:
        raise NotImplementedError('HMCMove at constant pressure (MonteCarloBarostat / MonteCarloAnisotropicBarostat) is '
                                  'not provided: HMCMove runs at constant volume')


def _apply_one_replica(owner, mc_moves, integrator, thermodynamic_state, sampler_state, context_cache):
    """`mc_moves` then `integrator` (None: no dynamics) on one replica in a single-replica engine, as one rx_propagate.
    A NaN retry reruns the dynamics only, from the state the Monte Carlo moves left (the restart loop of the Langevin move
    inside SequenceMove.apply, mcmc.py:420-424, 706-759).  `owner` carries the seed counter."""
    dyn = integrator if integrator is not None else _NO_DYNAMICS
    check_hmc([dyn], thermodynamic_state.pressure)
    device = _backend.default_device(context_cache or getattr(owner, 'context_cache', None))
    eng = _backend.build_engine([thermodynamic_state], 1, device=device)
    try:
        dyn._set_on_engine(eng)
        if mc_moves:
            eng.set_mc_moves([[m._engine_move(sampler_state.n_particles) for m in mc_moves]])
        has_v = sampler_state._velocities is not None
        reassign = integrator is not None and (integrator.reassign_velocities or not has_v)
        attempts = 0
        seed0 = getattr(owner, 'seed', None)
        if seed0 is None:
            seed0 = int(np.random.SeedSequence().entropy & 0xFFFFFFFFFFFFFFFF)
        while True:
            if attempts == 0 or not mc_moves:
                eng.set_positions(sampler_state._positions[None])
                if has_v:
                    eng.set_velocities(sampler_state._velocities[None])
            try:
                if attempts > 0 and mc_moves:
                    eng.propagate_retry(seed0 + attempts, owner._seed_counter, reassign_velocities=reassign)
                else:
                    eng.propagate(seed0 + attempts, owner._seed_counter, reassign_velocities=reassign)
                break
            except EngineError as e:
                if e.code != _lib.RX_ERR_NAN:
                    raise
                attempts += 1
                if attempts > dyn.n_restart_attempts:
                    raise IntegratorMoveError('Potential energy is NaN after {} attempts of integration '
                                              'with move {}'.format(attempts, owner.__class__.__name__), owner)
        owner._seed_counter += 1
        pot, kin = eng.get_replica_energies()
        if mc_moves:
            acc, prop = eng.get_mc_statistics()
            for j, m in enumerate(mc_moves):
                m.n_accepted += int(acc[0, j])
                m.n_proposed += int(prop[0, j])
        if integrator is None:    # Monte Carlo moves alone leave the velocities as they were
            sampler_state._update(eng.get_positions()[0], sampler_state._velocities, pot[0], None)
        else:
            sampler_state._update(eng.get_positions()[0], eng.get_velocities()[0], pot[0], kin[0])
    finally:
        eng.close()


class _NoDynamics(BaseIntegratorMove):
    """The integrator of a SequenceMove without a Langevin move: zero steps (the engine always runs one program)."""

    def __init__(self):
        super().__init__(n_steps=0, n_restart_attempts=0)

    def _integrator_parameters(self):
        return 0.001, 1.0, 0, 'VRO'


_NO_DYNAMICS = _NoDynamics()


# ---- Monte Carlo moves (mcmc.py:350-437, 810-970, 1704-1911) -------------------------------------------------------------
RX_MAX_MC_MOVES = _lib.RX_MAX_MC_MOVES


class MetropolizedMove(MCMCMove):
    """A rigid move of ``atom_subset`` accepted with the Metropolis criterion (mcmc.py:810-970).

    ``atom_subset``: None (every atom), a slice, or a list of atom indices.  ``n_accepted`` / ``n_proposed`` count the
    proposals.  In a sampler the proposals run on the device before each replica's Langevin steps; the counts are brought
    back into the move when the sampler writes its moves to storage."""

    def __init__(self, atom_subset=None, **kwargs):
        self.context_cache = kwargs.pop('context_cache', None)
        if kwargs:
            raise TypeError('unexpected arguments %s' % sorted(kwargs))
        self.n_accepted = 0
        self.n_proposed = 0
        self.atom_subset = atom_subset
        self._seed_counter = 0

    @property
    def statistics(self):
        """The acceptance statistics as a dictionary."""
        return dict(n_accepted=self.n_accepted, n_proposed=self.n_proposed)

    @statistics.setter
    def statistics(self, value):
        self.n_accepted = value['n_accepted']
        self.n_proposed = value['n_proposed']

    def apply(self, thermodynamic_state, sampler_state, context_cache=None):
        """One proposal on one replica; the statistics are updated (mcmc.py:869-941)."""
        _apply_one_replica(self, [self], None, thermodynamic_state, sampler_state, context_cache)

    def subset_indices(self, n_particles):
        """The indices of ``atom_subset`` in a system of n_particles atoms (mcmc.py:903-910), checked: in range, each
        once, at least one."""
        if self.atom_subset is None:
            idx = np.arange(n_particles)
        elif isinstance(self.atom_subset, slice):
            idx = np.arange(n_particles)[self.atom_subset]
        else:
            idx = np.asarray(self.atom_subset)
            if idx.ndim != 1 or not (np.issubdtype(idx.dtype, np.integer) or idx.size == 0):
                raise ValueError('atom_subset must be None, a slice or a list of atom indices')
            idx = idx.astype(np.int64)
        if idx.size == 0:
            raise ValueError('atom_subset selects no atom')
        if idx.min() < 0 or idx.max() >= n_particles:
            raise ValueError('atom_subset holds an index outside 0..%d' % (n_particles - 1))
        if len(np.unique(idx)) != idx.size:
            raise ValueError('atom_subset lists an atom twice')
        return idx

    def _engine_move(self, n_particles):
        raise NotImplementedError

    def __getstate__(self):
        serialization = dict(atom_subset=self.atom_subset)
        serialization.update(self.statistics)
        return serialization

    def __setstate__(self, serialization):
        self.atom_subset = serialization['atom_subset']
        self.statistics = serialization
        self.context_cache = None
        self._seed_counter = 0


class MCDisplacementMove(MetropolizedMove):
    """Displace the subset by a normal vector of standard deviation ``displacement_sigma`` per component
    (mcmc.py:1704-1770)."""

    def __init__(self, displacement_sigma=1.0 * unit.nanometer, **kwargs):
        super().__init__(**kwargs)
        self.displacement_sigma = displacement_sigma

    @staticmethod
    def displace_positions(positions, displacement_sigma=1.0 * unit.nanometer):
        """The positions after a random displacement (numpy's global generator, as the reference)."""
        positions_unit = positions.unit
        unitless_displacement_sigma = displacement_sigma / positions_unit
        displacement_vector = unit.Quantity(np.random.randn(3) * unitless_displacement_sigma, positions_unit)
        return positions + displacement_vector

    def _engine_move(self, n_particles):
        sigma = float(unit.to_md(self.displacement_sigma, unit.nanometer, 'displacement_sigma'))
        if not (np.isfinite(sigma) and sigma >= 0.0):
            raise ValueError('displacement_sigma must be finite and >= 0')
        return _lib.RX_MC_DISPLACEMENT, sigma, self.subset_indices(n_particles)

    def __getstate__(self):
        serialization = super().__getstate__()
        serialization['displacement_sigma'] = self.displacement_sigma
        return serialization

    def __setstate__(self, serialization):
        super().__setstate__(serialization)
        self.displacement_sigma = serialization['displacement_sigma']


class MCRotationMove(MetropolizedMove):
    """Rotate the subset about its geometric centre by a uniformly distributed rotation (mcmc.py:1777-1911)."""

    def __init__(self, **kwargs):
        super().__init__(**kwargs)

    @classmethod
    def rotate_positions(cls, positions):
        """The positions after a random rotation about their centre of geometry."""
        positions_unit = positions.unit
        x_initial = np.asarray(positions / positions_unit, np.float64)
        x_initial_mean = x_initial.mean(0)
        rotation_matrix = cls.generate_random_rotation_matrix()
        x_proposed = (rotation_matrix @ (x_initial - x_initial_mean).T).T + x_initial_mean
        return unit.Quantity(x_proposed, positions_unit)

    @classmethod
    def generate_random_rotation_matrix(cls):
        """A random 3x3 rotation matrix, uniform over rotations."""
        return cls._rotation_matrix_from_quaternion(cls._generate_uniform_quaternion())

    @staticmethod
    def _rotation_matrix_from_quaternion(q):
        """The rotation matrix of the quaternion (w, x, y, z); q need not be normalised (zero norm: the identity)."""
        w, x, y, z = q
        Nq = (np.asarray(q) ** 2).sum()
        s = 2.0 / Nq if Nq > 0.0 else 0.0
        X = x * s; Y = y * s; Z = z * s
        wX = w * X; wY = w * Y; wZ = w * Z
        xX = x * X; xY = x * Y; xZ = x * Z
        yY = y * Y; yZ = y * Z; zZ = z * Z
        return np.array([[1.0 - (yY + zZ), xY - wZ, xZ + wY],
                         [xY + wZ, 1.0 - (xX + zZ), yZ - wX],
                         [xZ - wY, yZ + wX, 1.0 - (xX + yY)]])

    @staticmethod
    def _generate_uniform_quaternion():
        """A uniform unit quaternion (Shoemake, Graphics Gems III, 124-132 (1992))."""
        u = np.random.rand(3)
        return np.array([np.sqrt(1 - u[0]) * np.sin(2 * np.pi * u[1]), np.sqrt(1 - u[0]) * np.cos(2 * np.pi * u[1]),
                         np.sqrt(u[0]) * np.sin(2 * np.pi * u[2]), np.sqrt(u[0]) * np.cos(2 * np.pi * u[2])])

    def _engine_move(self, n_particles):
        return _lib.RX_MC_ROTATION, 0.0, self.subset_indices(n_particles)


class SequenceMove(MCMCMove):
    """A sequence of moves applied in order (mcmc.py:350-437).  Provided shapes: up to RX_MAX_MC_MOVES Metropolized moves
    followed by at most one Langevin move."""

    def __init__(self, move_list, **kwargs):
        self.context_cache = kwargs.pop('context_cache', None)
        if kwargs:
            raise TypeError('unexpected arguments %s' % sorted(kwargs))
        self.move_list = list(move_list)
        self._seed_counter = 0

    @property
    def statistics(self):
        """The statistics of every move, {} for a move without statistics."""
        return [getattr(move, 'statistics', {}) for move in self.move_list]

    @statistics.setter
    def statistics(self, value):
        for i, move in enumerate(self.move_list):
            if hasattr(move, 'statistics'):
                move.statistics = value[i]

    def apply(self, thermodynamic_state, sampler_state, context_cache=None):
        """The moves in order on one replica, in one single-replica engine."""
        mc, integrator = split_move(self)
        _apply_one_replica(self, mc, integrator, thermodynamic_state, sampler_state, context_cache)

    def __str__(self):
        return str(self.move_list)

    def __iter__(self):
        return iter(self.move_list)

    def __getstate__(self):
        return dict(move_list=[copy.deepcopy(move) for move in self.move_list])

    def __setstate__(self, serialization):
        self.move_list = list(serialization['move_list'])
        self.context_cache = None
        self._seed_counter = 0


_SEQUENCE_RULE = ('a move must be a Metropolized move, a Langevin move, an HMCMove, or a SequenceMove of up to %d '
                  'Metropolized moves followed by at most one Langevin move or HMCMove' % RX_MAX_MC_MOVES)


def split_move(move):
    """(Metropolized moves, integrator move -- Langevin or HMC -- or None) of a move; NotImplementedError for the shapes the
    engine does not run."""
    if isinstance(move, MetropolizedMove):
        return [move], None
    if isinstance(move, BaseIntegratorMove):
        return [], move
    if not isinstance(move, SequenceMove):
        raise NotImplementedError('%s is not provided on the GPU path: %s' % (type(move).__name__, _SEQUENCE_RULE))
    mc, integrator = [], None
    for m in move.move_list:
        if isinstance(m, MetropolizedMove):
            if integrator is not None:
                raise NotImplementedError('a Monte Carlo move after the dynamics: ' + _SEQUENCE_RULE)
            mc.append(m)
        elif isinstance(m, BaseIntegratorMove):
            if integrator is not None:
                raise NotImplementedError('two integrator moves in one sequence: ' + _SEQUENCE_RULE)
            integrator = m
        else:
            raise NotImplementedError('%s inside a SequenceMove: %s' % (type(m).__name__, _SEQUENCE_RULE))
    if len(mc) > RX_MAX_MC_MOVES:
        raise NotImplementedError('%d Monte Carlo moves in one sequence: %s' % (len(mc), _SEQUENCE_RULE))
    return mc, integrator


def integrator_part(move):
    """The integrator move a move runs (split_move), or the zero-step stand-in of a move without dynamics."""
    integrator = split_move(move)[1]
    return _NO_DYNAMICS if integrator is None else integrator


def same_integrator(a, b):
    return type(a) is type(b) and a._integrator_parameters() == b._integrator_parameters() and \
        a.reassign_velocities == b.reassign_velocities
