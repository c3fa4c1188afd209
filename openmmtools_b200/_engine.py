"""Thin Python handle over the C-ABI engine (one engine = one GPU = one shard of the replicas).

This is the binding the reference-side hooks call:
  ReplicaExchangeSampler._mix_replicas       -> Engine.mix_swap_all / mix_swap_neighbors
  MultiStateSampler._propagate_replicas      -> Engine.propagate
  MultiStateSampler._compute_energies        -> Engine.compute_energies
(/root/reference/openmmtools/multistate/multistatesampler.py:1287,1436; replicaexchange.py:255)
"""
import ctypes as C
import numpy as np
from . import _lib


class EngineError(RuntimeError):
    def __init__(self, code, message):
        super().__init__('[rx %d] %s' % (code, message))
        self.code = code
        self.message = message


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _c64(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.float64)
    if shape is not None and tuple(a.shape) != tuple(shape):
        raise ValueError('expected array of shape %s, got %s' % (shape, a.shape))
    return a


def scale_mask(scale):
    """(scale_x, scale_y, scale_z) flags -> the barostat's axis mask (bit d: axis d is scaled)."""
    if len(scale) != 3:
        raise ValueError('scale needs three flags (x, y, z), got %r' % (scale,))
    return sum(1 << d for d, f in enumerate(scale) if f)


class Engine:
    def __init__(self, system_kind, n_replicas, n_states, n_atoms=0, device=0, rank=0, world_size=1,
                 box=(1.0, 1.0, 1.0), r_cutoff=0.0, r_switch=0.0, use_switch=False, annihilate_sterics=False,
                 softcore_alpha=0.5, softcore_a=1.0, softcore_b=1.0, softcore_c=6.0):
        self._lib = _lib.load()
        self._h = C.c_void_p()
        self.K, self.M, self.N = int(n_replicas), int(n_states), int(n_atoms)
        self.rank, self.world_size = int(rank), int(world_size)
        cfg = _lib.RxConfig(_lib.RX_ABI_VERSION, system_kind, self.K, self.M, self.N, device, rank, world_size,
                            (C.c_double * 3)(*[float(b) for b in box]), float(r_cutoff), float(r_switch),
                            int(bool(use_switch)), int(bool(annihilate_sterics)), float(softcore_alpha),
                            float(softcore_a), float(softcore_b), float(softcore_c))
        rc = self._lib.rx_create(C.byref(cfg), C.byref(self._h))
        if rc != 0:
            msg = self._lib.rx_last_error(None).decode()
            self._h = None
            raise EngineError(rc, msg)
        self.k0 = (self.rank * self.K) // self.world_size
        self.k1 = ((self.rank + 1) * self.K) // self.world_size

    # -- plumbing
    def _check(self, rc):
        if rc != 0:
            raise EngineError(rc, self._lib.rx_last_error(self._h).decode())

    def close(self):
        if getattr(self, '_h', None):
            self._lib.rx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- tables
    def set_particles(self, sigma, epsilon, mass, alchemical_mask=None):
        mass = _c64(mass, (self.N,))
        sigma = None if sigma is None else _c64(sigma, (self.N,))
        epsilon = None if epsilon is None else _c64(epsilon, (self.N,))
        mask = None if alchemical_mask is None else np.ascontiguousarray(alchemical_mask, dtype=np.uint8)
        self._check(self._lib.rx_set_particles(self._h, _ptr(sigma), _ptr(epsilon), _ptr(mass), _ptr(mask)))
        self._two_regions = False

    @staticmethod
    def _state_table(temperature, lambda_sterics=None, energy_offset=None, ho_K=None, ho_x0=None, lambda_electrostatics=None):
        M = len(temperature)
        arr = (_lib.RxStateParams * M)()
        for l in range(M):
            arr[l].temperature = float(temperature[l])
            arr[l].lambda_sterics = 1.0 if lambda_sterics is None else float(lambda_sterics[l])
            arr[l].energy_offset = 0.0 if energy_offset is None else float(energy_offset[l])
            arr[l].ho_K = 0.0 if ho_K is None else float(ho_K[l])
            arr[l].lambda_electrostatics = 1.0 if lambda_electrostatics is None else float(lambda_electrostatics[l])
            x0 = (0.0, 0.0, 0.0) if ho_x0 is None else ho_x0[l]
            for q in range(3):
                arr[l].ho_x0[q] = float(x0[q])
        return arr

    def set_states(self, temperature, lambda_sterics=None, energy_offset=None, ho_K=None, ho_x0=None, lambda_sterics_2=None,
                   lambda_electrostatics=None):
        """lambda_sterics_2: the second alchemical region's lambda of every state (rx_set_states_region2);
        lambda_electrostatics: read for alchemical molecules only."""
        if len(temperature) != self.M:
            raise ValueError('expected %d states' % self.M)
        self._check_region2(lambda_sterics_2)
        arr = self._state_table(temperature, lambda_sterics, energy_offset, ho_K, ho_x0, lambda_electrostatics)
        self._check(self._lib.rx_set_states(self._h, C.cast(arr, C.c_void_p)))
        if lambda_sterics_2 is not None:
            self._check(self._lib.rx_set_states_region2(self._h, _ptr(_c64(lambda_sterics_2, (self.M,)))))

    def _check_region2(self, lambda_sterics_2):
        # a two-region engine takes the second region's lambdas with every state table (the C layer would take 1)
        two = getattr(self, '_two_regions', False)
        if two and lambda_sterics_2 is None:
            raise ValueError('a two-region engine needs lambda_sterics_2 with every state table')
        if not two and lambda_sterics_2 is not None:
            raise ValueError('lambda_sterics_2 needs an engine with two alchemical regions (set_alchemical_regions)')

    def set_alchemical_regions(self, region, annihilate_1, annihilate_2):
        """Two alchemical regions: region[i] = 0 (environment), 1 or 2, and each region's annihilate_sterics
        (rx_set_alchemical_regions; after set_particles)."""
        r = np.ascontiguousarray(region, dtype=np.uint8)
        if r.shape != (self.N,):
            raise ValueError('expected %d region ids' % self.N)
        self._check(self._lib.rx_set_alchemical_regions(self._h, _ptr(r), int(bool(annihilate_1)), int(bool(annihilate_2))))
        self._two_regions = True

    def compute_energies_at(self, temperature, lambda_sterics=None, energy_offset=None, ho_K=None, ho_x0=None, pressure=None,
                            dispersion=None, lambda_sterics_2=None, lambda_electrostatics=None):
        """u[K][n] of every replica at n other states (unsampled states); the resident matrix is untouched.  An NPT engine
        takes those states' pressures (kJ/mol/nm^3) and dispersion coefficients (kJ/mol nm^3) as well; a two-region engine
        their second-region lambdas."""
        self._check_region2(lambda_sterics_2)
        arr = self._state_table(temperature, lambda_sterics, energy_offset, ho_K, ho_x0, lambda_electrostatics)
        n = len(temperature)
        out = np.zeros((self.K, n))
        if lambda_sterics_2 is not None:
            l2 = _c64(lambda_sterics_2, (n,))
            p, c = (None, None) if pressure is None else (_c64(pressure, (n,)), _c64(dispersion, (n,)))
            self._check(self._lib.rx_compute_energies_at_region2(self._h, C.cast(arr, C.c_void_p), _ptr(l2), _ptr(p), _ptr(c), n,
                                                                 _ptr(out)))
        elif pressure is None:
            self._check(self._lib.rx_compute_energies_at(self._h, C.cast(arr, C.c_void_p), n, _ptr(out)))
        else:
            p, c = _c64(pressure, (n,)), _c64(dispersion, (n,))
            self._check(self._lib.rx_compute_energies_at_npt(self._h, C.cast(arr, C.c_void_p), _ptr(p), _ptr(c), n, _ptr(out)))
        return out

    def set_integrator(self, timestep, collision_rate, n_steps, splitting='V R O R V'):
        self._check(self._lib.rx_set_integrator(self._h, float(timestep), float(collision_rate), int(n_steps),
                                                splitting.replace(' ', '').encode()))

    def set_molecule(self, system, constraint_tolerance=1e-8):
        """Particles and force field of a RX_SYSTEM_MOLECULE engine from a system.System of kind 'molecule'."""
        f = lambda a, w: np.ascontiguousarray(np.asarray(a if a is not None else np.zeros((0, w)), np.float64).reshape(-1, w))
        arrs = dict(mass=np.ascontiguousarray(system.masses, np.float64), charge=np.ascontiguousarray(system.charge, np.float64),
                    sigma=np.ascontiguousarray(system.sigma, np.float64), epsilon=np.ascontiguousarray(system.epsilon, np.float64),
                    bonds=f(system.bonds, 4), angles=f(system.angles, 5), torsions=f(system.torsions, 7),
                    exclusions=np.ascontiguousarray(np.asarray(system.exclusions if system.exclusions is not None else np.zeros((0, 2)), np.int64).reshape(-1, 2)),
                    exceptions=f(system.exceptions, 5), constraints=f(system.constraints, 3))
        m = _lib.RxMolecule(len(arrs['bonds']), len(arrs['angles']), len(arrs['torsions']), len(arrs['exclusions']),
                            len(arrs['exceptions']), len(arrs['constraints']), int(bool(system.remove_cm_motion)), 0,
                            float(constraint_tolerance), *[arrs[k].ctypes.data for k in
                                                           ('mass', 'charge', 'sigma', 'epsilon', 'bonds', 'angles', 'torsions',
                                                            'exclusions', 'exceptions', 'constraints')])
        if system.is_alchemical:
            alch = np.ascontiguousarray(system.alchemical_mask(), np.uint8)
            m.alchemical, m.annihilate_sterics = alch.ctypes.data, int(bool(system.annihilate_sterics))
            m.annihilate_electrostatics = int(bool(system.annihilate_electrostatics))
        self._check(self._lib.rx_set_molecule(self._h, C.byref(m)))
        if getattr(system, 'gb_radius', None) is not None:
            self.set_implicit_solvent(system.gb_radius, system.gb_scale, *system.gb_parameters,
                                      alchemical_obc2=system.is_alchemical and system.alchemical_obc2)

    def set_implicit_solvent(self, radius, scale, alpha, beta, gamma, offset, solute_dielectric, solvent_dielectric, sa_energy,
                             probe_radius, alchemical_obc2=False):
        """OBC implicit solvent for the molecule of the last set_molecule (rx_set_implicit_solvent)."""
        radius = np.ascontiguousarray(radius, np.float64)
        scale = np.ascontiguousarray(scale, np.float64)
        g = _lib.RxGbsa(radius.ctypes.data, scale.ctypes.data, alpha, beta, gamma, offset, solute_dielectric, solvent_dielectric,
                        sa_energy, probe_radius, int(bool(alchemical_obc2)))
        self._check(self._lib.rx_set_implicit_solvent(self._h, C.byref(g)))

    def set_state_integrator(self, state, timestep, collision_rate, n_steps, splitting='V R O R V', reassign_velocities=False):
        """The move of one thermodynamic state where the states carry different moves (after set_integrator)."""
        self._check(self._lib.rx_set_state_integrator(self._h, int(state), float(timestep), float(collision_rate), int(n_steps),
                                                      splitting.replace(' ', '').encode(), int(bool(reassign_velocities))))

    # -- hybrid Monte Carlo (rx_set_hmc_integrator)
    def set_hmc_integrator(self, timestep, n_steps):
        """HMC for every state: each propagation is n_steps trials of n_steps velocity-Verlet steps of `timestep` ps."""
        self._check(self._lib.rx_set_hmc_integrator(self._h, float(timestep), int(n_steps)))

    def set_state_hmc_integrator(self, state, timestep, n_steps):
        """The HMC move of one thermodynamic state (after set_hmc_integrator)."""
        self._check(self._lib.rx_set_state_hmc_integrator(self._h, int(state), float(timestep), int(n_steps)))

    def get_hmc_statistics(self):
        """(accepted, trials) int64 [K] of the HMC trials of the replicas this engine owns (zero elsewhere), cumulative over
        the engine's life.  Diagnostics only: the reference's HMCMove keeps no statistics, so a sampler's storage does not
        save them and a sampler resumed from storage starts them at zero (set_hmc_statistics can put counts back)."""
        acc = np.zeros(self.K, np.int64); trials = np.zeros_like(acc)
        self._check(self._lib.rx_get_hmc_statistics(self._h, _ptr(acc), _ptr(trials)))
        return acc, trials

    def set_hmc_statistics(self, accepted, trials):
        acc = np.ascontiguousarray(accepted, np.int64).reshape(self.K)
        n = np.ascontiguousarray(trials, np.int64).reshape(self.K)
        self._check(self._lib.rx_set_hmc_statistics(self._h, _ptr(acc), _ptr(n)))

    def get_hmc_energies(self):
        """(Eold, Enew) float64 [K] in kJ/mol of every owned replica's last HMC trial (NaN: none)."""
        e0 = np.zeros(self.K); e1 = np.zeros(self.K)
        self._check(self._lib.rx_get_hmc_energies(self._h, _ptr(e0), _ptr(e1)))
        return e0, e1

    # -- Monte Carlo moves (rx_set_mc_subsets, rx_set_state_mc_moves)
    def set_mc_moves(self, moves):
        """The Monte Carlo moves of every state: moves[l] is a list of up to RX_MAX_MC_MOVES (kind, sigma_nm, atom indices),
        kind RX_MC_DISPLACEMENT or RX_MC_ROTATION.  Every distinct subset is uploaded once."""
        if len(moves) != self.M:
            raise ValueError('expected the moves of %d states' % self.M)
        atoms, where = [], {}
        for state in moves:
            for _, _, subset in state:
                key = tuple(int(i) for i in subset)
                if key not in where:
                    where[key] = len(atoms)
                    atoms.extend(key)
        a = np.ascontiguousarray(atoms, np.int32)
        self._check(self._lib.rx_set_mc_subsets(self._h, _ptr(a), len(a)))
        for l, state in enumerate(moves):
            arr = (_lib.RxMcMove * max(len(state), 1))()
            for j, (kind, sigma, subset) in enumerate(state):
                key = tuple(int(i) for i in subset)
                arr[j].kind, arr[j].subset_offset, arr[j].subset_len, arr[j].sigma_nm = int(kind), where[key], len(key), float(sigma)
            self._check(self._lib.rx_set_state_mc_moves(self._h, l, len(state), C.cast(arr, C.c_void_p)))

    def get_mc_statistics(self):
        """(accepted, proposed) int64 [M][RX_MAX_MC_MOVES] of the replicas this engine owns."""
        acc = np.zeros((self.M, _lib.RX_MAX_MC_MOVES), np.int64); prop = np.zeros_like(acc)
        self._check(self._lib.rx_get_mc_statistics(self._h, _ptr(acc), _ptr(prop)))
        return acc, prop

    def get_mc_energy_changes(self):
        """dU (kJ/mol) [K][RX_MAX_MC_MOVES] of every owned replica's last proposal per move slot; NaN where no energy was
        computed (rx_get_mc_energy_changes)."""
        du = np.zeros((self.K, _lib.RX_MAX_MC_MOVES))
        self._check(self._lib.rx_get_mc_energy_changes(self._h, _ptr(du)))
        return du

    def set_mc_statistics(self, accepted, proposed):
        shape = (self.M, _lib.RX_MAX_MC_MOVES)
        acc = np.ascontiguousarray(accepted, np.int64).reshape(shape)
        prop = np.ascontiguousarray(proposed, np.int64).reshape(shape)
        self._check(self._lib.rx_set_mc_statistics(self._h, _ptr(acc), _ptr(prop)))

    # -- constant pressure (rx_set_pressures)
    def set_pressures(self, pressure, dispersion):
        """Switch to NPT: per-state pressures (kJ/mol/nm^3) and dispersion coefficients c_l (kJ/mol nm^3, the correction
        at volume V is c_l / V).  Every owned replica gets the engine's box and a fresh barostat state."""
        p, c = _c64(pressure, (self.M,)), _c64(dispersion, (self.M,))
        self._check(self._lib.rx_set_pressures(self._h, _ptr(p), _ptr(c)))

    def set_boxes(self, edges, first=0):
        """Box edges (count, 3) in nm of replicas [first, first + count)."""
        e = _c64(edges)
        if e.ndim != 2 or e.shape[1] != 3:
            raise ValueError('edges must have shape (count, 3)')
        self._check(self._lib.rx_set_boxes(self._h, first, e.shape[0], _ptr(e)))

    def get_boxes(self, first=None, count=None):
        first = self.k0 if first is None else first
        count = (self.k1 - first) if count is None else count
        out = np.zeros((count, 3))
        self._check(self._lib.rx_get_boxes(self._h, first, count, _ptr(out)))
        return out

    _BARO_FIELDS = ('volume_scale', 'step', 'n_attempted', 'n_accepted')

    def get_barostat(self, first=None, count=None):
        """Barostat state of replicas [first, first + count): dict of arrays volume_scale, step, n_attempted, n_accepted."""
        first = self.k0 if first is None else first
        count = (self.k1 - first) if count is None else count
        arr = (_lib.RxBarostatState * max(count, 1))()
        self._check(self._lib.rx_get_barostat(self._h, first, count, C.cast(arr, C.c_void_p)))
        return {f: np.array([getattr(arr[i], f) for i in range(count)], np.float64 if f == 'volume_scale' else np.int64)
                for f in self._BARO_FIELDS}

    def set_barostat(self, state, first=0):
        count = len(state['volume_scale'])
        arr = (_lib.RxBarostatState * max(count, 1))()
        for i in range(count):
            arr[i].volume_scale = float(state['volume_scale'][i])
            for f in self._BARO_FIELDS[1:]:
                setattr(arr[i], f, int(state[f][i]))
        self._check(self._lib.rx_set_barostat(self._h, first, count, C.cast(arr, C.c_void_p)))

    def set_anisotropic_barostat(self, scale):
        """Switch the NPT engine to the anisotropic barostat: scale = (scale_x, scale_y, scale_z) flags, at least one set.
        Every owned replica gets a fresh per-axis state (rx_set_anisotropic_barostat)."""
        self._check(self._lib.rx_set_anisotropic_barostat(self._h, scale_mask(scale)))

    _ANISO_FIELDS = ('volume_scale', 'n_attempted', 'n_accepted')

    def get_barostat_anisotropic(self, first=None, count=None):
        """Per-axis barostat state of replicas [first, first + count): dict of volume_scale, n_attempted, n_accepted
        (count, 3), step and scale_mask (count,)."""
        first = self.k0 if first is None else first
        count = (self.k1 - first) if count is None else count
        arr = (_lib.RxAnisotropicBarostatState * max(count, 1))()
        self._check(self._lib.rx_get_barostat_anisotropic(self._h, first, count, C.cast(arr, C.c_void_p)))
        out = {f: np.array([list(getattr(arr[i], f)) for i in range(count)], np.float64 if f == 'volume_scale' else np.int64)
               .reshape(count, 3) for f in self._ANISO_FIELDS}
        for f in ('step', 'scale_mask'):
            out[f] = np.array([getattr(arr[i], f) for i in range(count)], np.int64)
        return out

    def set_barostat_anisotropic(self, state, first=0):
        count = len(state['volume_scale'])
        arr = (_lib.RxAnisotropicBarostatState * max(count, 1))()
        for i in range(count):
            arr[i].volume_scale[:] = [float(v) for v in state['volume_scale'][i]]
            for f in self._ANISO_FIELDS[1:]:
                getattr(arr[i], f)[:] = [int(v) for v in state[f][i]]
            arr[i].step, arr[i].scale_mask = int(state['step'][i]), int(state['scale_mask'][i])
        self._check(self._lib.rx_set_barostat_anisotropic(self._h, first, count, C.cast(arr, C.c_void_p)))

    # -- replica state
    def set_positions(self, xyz, first=0):
        xyz = _c64(xyz)
        self._check(self._lib.rx_set_positions(self._h, first, xyz.shape[0], _ptr(xyz)))

    def set_velocities(self, xyz, first=0):
        xyz = _c64(xyz)
        self._check(self._lib.rx_set_velocities(self._h, first, xyz.shape[0], _ptr(xyz)))

    def _out(self, out, count):
        if out is None:
            return np.empty((count, self.N, 3))
        if out.dtype != np.float64 or not out.flags.c_contiguous or out.shape != (count, self.N, 3):
            raise ValueError('out must be a C-contiguous float64 array of shape %s' % ((count, self.N, 3),))
        return out

    def get_positions(self, first=None, count=None, out=None):
        first = self.k0 if first is None else first
        count = (self.k1 - first) if count is None else count
        out = self._out(out, count)
        self._check(self._lib.rx_get_positions(self._h, first, count, _ptr(out)))
        return out

    def get_velocities(self, first=None, count=None, out=None):
        first = self.k0 if first is None else first
        count = (self.k1 - first) if count is None else count
        out = self._out(out, count)
        self._check(self._lib.rx_get_velocities(self._h, first, count, _ptr(out)))
        return out

    def pinned_array(self, shape, dtype=np.float64):
        """A page-aligned array registered with the engine (rx_pin_host_memory): copies to and from it are direct DMA."""
        n = max(int(np.prod(shape)) * np.dtype(dtype).itemsize, 8)
        raw = np.zeros(n + 4096, np.uint8)
        off = (-raw.ctypes.data) % 4096
        a = raw[off:off + int(np.prod(shape)) * np.dtype(dtype).itemsize].view(dtype).reshape(shape)
        self._check(self._lib.rx_pin_host_memory(self._h, _ptr(a), n))
        self._pinned = getattr(self, '_pinned', []) + [raw]     # keeps the allocation alive as long as the engine
        return a

    def get_replica_energies(self):
        pot, kin = np.zeros(self.K), np.zeros(self.K)
        self._check(self._lib.rx_get_replica_energies(self._h, _ptr(pot), _ptr(kin)))
        return pot, kin

    def randomize_velocities(self, seed, stream=0):
        self._check(self._lib.rx_randomize_velocities(self._h, int(seed), int(stream)))

    def minimize(self, tolerance, max_iterations=0):
        """FIRE descent of the owned replicas; returns (rms force [K] in kJ/mol/nm, iterations taken [K])."""
        rms, its = np.zeros(self.K), np.zeros(self.K, np.int32)
        self._check(self._lib.rx_minimize(self._h, float(tolerance), int(max_iterations), _ptr(rms), _ptr(its)))
        return rms, its

    def set_replica_states(self, states):
        s = np.ascontiguousarray(states, dtype=np.int64)
        if s.shape != (self.K,):
            raise ValueError('expected %d replica states' % self.K)
        self._check(self._lib.rx_set_replica_states(self._h, _ptr(s)))

    def get_replica_states(self):
        s = np.zeros(self.K, np.int64)
        self._check(self._lib.rx_get_replica_states(self._h, _ptr(s)))
        return s

    # -- phases
    def propagate(self, seed, iteration, reassign_velocities=False):
        """Returns the per-replica NaN flags; raises EngineError(RX_ERR_NAN) if any is set."""
        flags = np.zeros(self.K, np.int32)
        rc = self._lib.rx_propagate(self._h, int(seed), int(iteration), int(bool(reassign_velocities)), _ptr(flags))
        if rc == _lib.RX_ERR_NAN:
            e = EngineError(rc, self._lib.rx_last_error(self._h).decode())
            e.nan_flags = flags
            raise e
        self._check(rc)
        return flags

    def propagate_retry(self, seed, iteration, reassign_velocities=False):
        """Replicas whose NaN flag is set restart from the state they had when ``propagate`` began; the others stay."""
        flags = np.zeros(self.K, np.int32)
        rc = self._lib.rx_propagate_retry(self._h, int(seed), int(iteration), int(bool(reassign_velocities)), _ptr(flags))
        if rc == _lib.RX_ERR_NAN:
            e = EngineError(rc, self._lib.rx_last_error(self._h).decode())
            e.nan_flags = flags
            raise e
        self._check(rc)
        return flags

    def compute_energies(self, fetch=True, out=None):
        """`out`: a C-contiguous float64 (K, M) array to receive the matrix (page-locked: a direct DMA copy)."""
        u = (self._result(out, (self.K, self.M), np.float64) if out is not None else np.zeros((self.K, self.M))) if fetch else None
        self._check(self._lib.rx_compute_energies(self._h, _ptr(u)))
        return u

    @staticmethod
    def _result(a, shape, dtype):
        if not (isinstance(a, np.ndarray) and a.dtype == dtype and a.shape == tuple(shape) and a.flags.c_contiguous):
            raise ValueError('out must be a C-contiguous %s array of shape %s' % (np.dtype(dtype).name, tuple(shape)))
        return a

    def _mix_out(self, out):
        if out is None:
            return (np.zeros(self.K, np.int64), np.zeros((self.M, self.M), np.int64), np.zeros((self.M, self.M), np.int64))
        st, nacc, nprop = out
        return (self._result(st, (self.K,), np.int64), self._result(nacc, (self.M, self.M), np.int64),
                self._result(nprop, (self.M, self.M), np.int64))

    def set_energies(self, u):
        u = _c64(u, (self.K, self.M))
        self._check(self._lib.rx_set_energies(self._h, _ptr(u)))

    def get_energies(self):
        u = np.zeros((self.K, self.M))
        self._check(self._lib.rx_get_energies(self._h, _ptr(u)))
        return u

    # -- energy history (rx_history_*): row t holds iteration t's (K, M) matrix and (K, U) unsampled block on the device
    def history_append(self, iteration, n_unsampled=0):
        """Row `iteration` from the current matrix and, with n_unsampled > 0, the last compute_energies_at block."""
        self._check(self._lib.rx_history_append(self._h, int(iteration), int(n_unsampled)))

    def history_truncate(self, iteration):
        """Keep iterations 0..iteration."""
        self._check(self._lib.rx_history_truncate(self._h, int(iteration)))

    def history_load(self, u, u_unsampled=None):
        """Replace the history by u (T, K, M) and u_unsampled (T, K, U)."""
        u = _c64(u)
        T = u.shape[0]
        uu = np.zeros((T, self.K, 0)) if u_unsampled is None else _c64(u_unsampled)
        if u.shape != (T, self.K, self.M) or uu.shape[:2] != (T, self.K):
            raise ValueError('expected (T, %d, %d) and (T, %d, U) energies, got %s and %s' % (self.K, self.M, self.K, u.shape,
                                                                                            uu.shape))
        self._check(self._lib.rx_history_load(self._h, T, uu.shape[2], _ptr(u), _ptr(uu)))

    def history_reserve(self, n_iterations, n_unsampled=0):
        self._check(self._lib.rx_history_reserve(self._h, int(n_iterations), int(n_unsampled)))

    def history_length(self):
        """(iterations held, unsampled states per row)."""
        n, u = C.c_int64(), C.c_int32()
        self._check(self._lib.rx_history_length(self._h, C.byref(n), C.byref(u)))
        return n.value, u.value

    def mix_seed(self, seed, stream=_lib.RX_STREAM_NUMBA):
        self._check(self._lib.rx_mix_seed(self._h, stream, int(seed) & 0xFFFFFFFF))

    def mix_skip(self, n_words, stream=_lib.RX_STREAM_NUMBA):
        self._check(self._lib.rx_mix_skip(self._h, stream, int(n_words)))

    def mix_swap_all(self, nswap_attempts=None, fetch=True, out=None):
        """`out`: (states int64 (K,), n_accepted int64 (M, M), n_proposed int64 (M, M)) to receive the results."""
        n = self.K ** 3 if nswap_attempts is None else int(nswap_attempts)
        if not fetch:
            self._check(self._lib.rx_mix_swap_all(self._h, n, None, None, None))
            return None
        st, nacc, nprop = self._mix_out(out)
        self._check(self._lib.rx_mix_swap_all(self._h, n, _ptr(st), _ptr(nacc), _ptr(nprop)))
        return st, nacc, nprop

    def mix_swap_neighbors(self, out=None):
        st, nacc, nprop = self._mix_out(out)
        self._check(self._lib.rx_mix_swap_neighbors(self._h, _ptr(st), _ptr(nacc), _ptr(nprop)))
        return st, nacc, nprop

    def get_mix_counts(self):
        nacc = np.zeros((self.M, self.M), np.int64); nprop = np.zeros((self.M, self.M), np.int64)
        self._check(self._lib.rx_get_mix_counts(self._h, _ptr(nacc), _ptr(nprop)))
        return nacc, nprop

    def mix_stream_position(self, stream=_lib.RX_STREAM_NUMBA):
        v = C.c_uint64()
        self._check(self._lib.rx_mix_stream_position(self._h, stream, C.byref(v)))
        return v.value

    def run_iterations(self, n, mixing, seed, first_iteration, reassign_velocities=False):
        """mixing: None | 'swap-all' | 'swap-neighbors' (replicaexchange.py:223)."""
        code = {None: 0, 'swap-all': 1, 'swap-neighbors': 2}[mixing]
        self._check(self._lib.rx_run_iterations(self._h, int(n), code, int(seed), int(first_iteration),
                                                int(bool(reassign_velocities))))

    # ---- SAMS on the device (rx_sams.cuh; sams.py:395-437, 477-501, 564-691)
    SAMS_METHODS = {'optimal': 0, 'rao-blackwellized': 1}
    SAMS_CRITERIA = {'minimum-visits': 0, 'histogram-flatness': 1, 'logZ-flatness': 2}

    def sams_set(self, log_target_probabilities, logZ, histogram=None, gamma0=1.0, flatness_threshold=0.2,
                 weight_update_method='rao-blackwellized', update_stages='two-stage', flatness_criteria='logZ-flatness',
                 stage=0, t0=0):
        cfg = _lib.RxSamsConfig(float(gamma0), float(flatness_threshold), self.SAMS_METHODS[weight_update_method],
                                1 if update_stages == 'two-stage' else 0, self.SAMS_CRITERIA[flatness_criteria], int(stage), int(t0))
        lt = _c64(log_target_probabilities, (self.M,)); lz = _c64(logZ, (self.M,))
        hh = None if histogram is None else np.ascontiguousarray(histogram, np.int64)
        self._check(self._lib.rx_sams_set(self._h, C.byref(cfg), _ptr(lt), _ptr(lz), None if hh is None else _ptr(hh)))

    def sams_step(self, iteration, update_weights=True, histogram=None):
        hh = None if histogram is None else np.ascontiguousarray(histogram, np.int64)
        self._check(self._lib.rx_sams_step(self._h, int(iteration), int(bool(update_weights)), None if hh is None else _ptr(hh)))

    def sams_get(self):
        """dict(logZ, log_weights, histogram, stage, t0, gamma, states, previous_states) of the device-resident SAMS state."""
        logZ = np.zeros(self.M); lw = np.zeros(self.M); hist = np.zeros(self.M, np.int64)
        st = np.zeros(self.K, np.int64); prev = np.zeros(self.K, np.int64)
        stage = C.c_int32(); t0 = C.c_int64(); gamma = C.c_double()
        self._check(self._lib.rx_sams_get(self._h, _ptr(logZ), _ptr(lw), _ptr(hist), C.byref(stage), C.byref(t0), C.byref(gamma),
                                          _ptr(st), _ptr(prev)))
        return dict(logZ=logZ, log_weights=lw, histogram=hist, stage=stage.value, t0=t0.value, gamma=gamma.value, states=st,
                    previous_states=prev)

    def sams_run_iterations(self, n, seed, first_iteration, reassign_velocities=False):
        self._check(self._lib.rx_sams_run_iterations(self._h, int(n), int(seed), int(first_iteration), int(bool(reassign_velocities))))

    def phase_times(self, reset=False):
        ms = np.zeros(4); cnt = np.zeros(4, np.int64)
        self._check(self._lib.rx_get_phase_times(self._h, _ptr(ms), _ptr(cnt), int(reset)))
        return dict(mix_ms=ms[0], propagate_ms=ms[1], energies_ms=ms[2], rng_ms=ms[3],
                    launches=int(cnt.sum()), launches_by_phase=cnt.tolist())

    def timer_mark(self, which):
        self._check(self._lib.rx_timer_mark(self._h, int(which)))

    def timer_elapsed_ms(self):
        v = C.c_double()
        self._check(self._lib.rx_timer_elapsed(self._h, C.byref(v)))
        return v.value

    def selftest_exp(self, x):
        """The device's correctly rounded exp (the mixing kernels' tie-break function) of a float64 array."""
        x = np.ascontiguousarray(x, np.float64)
        y = np.empty_like(x)
        self._check(self._lib.rx_selftest_exp(self._h, _ptr(x), _ptr(y), C.c_int32(x.size)))
        return y

    def mix_stats(self):
        out = np.zeros(6, np.int64)
        self._check(self._lib.rx_get_mix_stats(self._h, _ptr(out)))
        return dict(rounds=int(out[0]), exact_exp=int(out[1]), passes=int(out[2]), words=int(out[3]),
                    walker_ms=out[4] / 1e3, prepare_wait_ms=out[5] / 1e3)

    @staticmethod
    def plan_propagate(system_kind, n_atoms, kloc, n_sm, smem_optin, box=(1.0, 1.0, 1.0), r_cutoff=0.0,
                       per_state=False, skin_out=-1.0, skin_in=-1.0, cluster=0, no_list=False, no_sort=False):
        """The launch rx_propagate would make (blocks per replica, threads, list capacity, ...) for a device with `n_sm`
        multiprocessors and `smem_optin` bytes of opt-in shared memory per block; host arithmetic, no device needed.
        Arguments after r_cutoff mirror the RX_SKIN, RX_SKIN_IN, RX_CLUSTER, RX_NO_VERLET and RX_NO_SORT overrides."""
        lib = _lib.load()
        q = _lib.RxPropagateQuery(int(system_kind), int(n_atoms), int(kloc), int(bool(per_state)), int(n_sm),
                                  int(smem_optin), (C.c_double * 3)(*[float(b) for b in box]), float(r_cutoff),
                                  float(skin_out), float(skin_in), int(cluster), int(bool(no_list)), int(bool(no_sort)))
        out = _lib.RxPropagatePlan()
        rc = lib.rx_plan_propagate(C.byref(q), C.byref(out))
        if rc != 0:
            raise EngineError(rc, lib.rx_last_error(None).decode())
        return dict(cluster=out.cluster, threads=out.threads, list_capacity=out.list_capacity,
                    sort_atoms=bool(out.sort_atoms), compact=bool(out.compact), smem_bytes=int(out.smem_bytes))

    # -- multi-GPU
    @staticmethod
    def comm_unique_id(nccl_path=None):
        lib = _lib.load()
        buf = C.create_string_buffer(128)
        rc = lib.rx_comm_unique_id((nccl_path or _lib.find_nccl()).encode(), buf)
        if rc != 0:
            raise EngineError(rc, lib.rx_last_error(None).decode())
        return buf.raw

    def comm_init(self, unique_id, nccl_path=None):
        buf = C.create_string_buffer(bytes(unique_id), 128)
        self._check(self._lib.rx_comm_init(self._h, (nccl_path or _lib.find_nccl()).encode(), buf))
