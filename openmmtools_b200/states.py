"""Thermodynamic and sampler state objects with the reference's API surface for the replica-exchange path.

Mirrors /root/reference/openmmtools/states.py: ``ThermodynamicState`` (:385), ``SamplerState`` (:1933),
``CompoundThermodynamicState`` (:2694), ``GlobalParameterState`` (:3100) and
``create_thermodynamic_state_protocol`` (:39-141).  No OpenMM objects are held: the "system" is a
:class:`openmmtools_b200.system.System` parameter record, and energies are evaluated by the CUDA engine
(``ThermodynamicState.reduced_potential`` -> ``rx_compute_energies``).  OpenMM-typed methods
(``create_context``, ``apply_to_context`` ...) raise ``NotImplementedError``.  A pressure puts a periodic LJ system in the
NPT ensemble with an isotropic Monte Carlo barostat that the CUDA engine runs (states.py:1741-1771).  A system holding a
``MonteCarloBarostat`` or ``MonteCarloAnisotropicBarostat`` record (openmmtools_b200.system) is NPT at that barostat's
pressure; the anisotropic one scales one edge per attempt, chosen among its scaled axes, which must share one pressure
(states.py:1656-1693; a z-only barostat is accepted).  Surface tensions and membrane barostats are not provided.
"""
import copy
import numpy as np
from . import unit
from .constants import kB
from .system import System, BAROSTATS, MonteCarloBarostat, MonteCarloAnisotropicBarostat


# ------------------------------------------------------------------------------------------------------
# exceptions (states.py:272-381)
# ------------------------------------------------------------------------------------------------------
class ThermodynamicsError(Exception):
    (MULTIPLE_THERMOSTATS, NO_THERMOSTAT, NONE_TEMPERATURE, INCONSISTENT_THERMOSTAT, MULTIPLE_BAROSTATS,
     NO_BAROSTAT, UNSUPPORTED_BAROSTAT, UNSUPPORTED_ANISOTROPIC_BAROSTAT, SURFACE_TENSION_NOT_SUPPORTED,
     INCONSISTENT_BAROSTAT, BAROSTATED_NONPERIODIC, INCONSISTENT_INTEGRATOR, INCOMPATIBLE_SAMPLER_STATE,
     INCOMPATIBLE_ENSEMBLE) = range(14)

    error_messages = {
        NONE_TEMPERATURE: 'Temperature cannot be None.',
        INCOMPATIBLE_SAMPLER_STATE: 'The sampler state has a different number of particles.',
        INCOMPATIBLE_ENSEMBLE: 'Cannot apply to a context in a different thermodynamic ensemble.',
        UNSUPPORTED_BAROSTAT: 'NPT ensembles are outside the GPU replica-exchange hot path.',
        BAROSTATED_NONPERIODIC: 'Non-periodic systems cannot have a barostat.',
        MULTIPLE_BAROSTATS: 'System has multiple barostats.',
        UNSUPPORTED_ANISOTROPIC_BAROSTAT: 'MonteCarloAnisotropicBarostat is supported only if the pressure along all '
                                          'scaled axes is the same and at least one axis is scaled.',
    }

    def __init__(self, code, *args):
        msg = self.error_messages.get(code, 'thermodynamics error %d' % code).format(*args)
        super().__init__(msg)
        self.code = code


class SamplerStateError(Exception):
    (INCONSISTENT_VELOCITIES, INCONSISTENT_POSITIONS) = range(2)
    error_messages = {INCONSISTENT_VELOCITIES: 'Velocities have different length than positions.',
                      INCONSISTENT_POSITIONS: 'Specified positions with inconsistent number of particles.'}

    def __init__(self, code, *args):
        super().__init__(self.error_messages[code].format(*args))
        self.code = code


class GlobalParameterError(Exception):
    (PARAMETER_NOT_DEFINED, INCOMPATIBLE_PARAMETER_VALUE) = range(2)

    def __init__(self, code, msg):
        super().__init__(msg)
        self.code = code


# ------------------------------------------------------------------------------------------------------
class ThermodynamicState:
    """Thermodynamic state of a system (states.py:385-1926): (system, temperature) in the NVT ensemble, or
    (system, temperature, pressure) in the NPT ensemble.

    A pressure adds what ``MonteCarloBarostat(pressure, temperature)`` adds in the reference (states.py:1761-1771): an
    isotropic Monte Carlo volume move at the state's temperature, attempted every 25 steps (OpenMM's default frequency,
    fixed here).  Only periodic systems take a pressure; surface tensions are not provided.

    A system holding a barostat record makes the state NPT at that barostat's pressure unless ``pressure`` is given.  With
    a ``MonteCarloAnisotropicBarostat`` the state keeps its scaled axes: ``pressure`` then sets the pressure of all three
    axes, and ``pressure = None`` removes the barostat.
    """

    def __init__(self, system, temperature=None, pressure=None, surface_tension=None):
        if not isinstance(system, System):
            raise TypeError('openmmtools_b200.states.ThermodynamicState needs an openmmtools_b200 System '
                            '(see openmmtools_b200.testsystems); got %r' % type(system))
        if temperature is None:
            raise ThermodynamicsError(ThermodynamicsError.NONE_TEMPERATURE)
        if surface_tension is not None:
            raise NotImplementedError('surface tension (membrane barostats) is outside the replica-exchange hot path')
        baro = _read_barostat(system)
        self._standard_system = _without_barostats(system)
        self._barostat_scale = None if baro is None else baro[1]   # anisotropic: (scale_x, scale_y, scale_z)
        self._rehash()
        self._temperature = None
        self._pressure = None
        self.temperature = temperature
        self.pressure = baro[0] * unit.bar if pressure is None and baro is not None else pressure

    # -- system
    @property
    def system(self):
        """A copy of the system in this thermodynamic state (states.py:510-539)."""
        return self.get_system()

    @system.setter
    def system(self, value):
        self.set_system(value)

    def set_system(self, system, fix_state=False):
        """A system with a barostat record brings its ensemble along; one without keeps the state's."""
        baro = _read_barostat(system)
        self._standard_system = _without_barostats(system)
        if baro is not None:
            self._barostat_scale = baro[1]
            self._rehash()
            self.pressure = baro[0] * unit.bar
        else:
            self._rehash()

    def get_system(self, remove_thermostat=False, remove_barostat=False):
        """A copy of the standard system; an anisotropic state's carries its barostat at the state's pressure."""
        system = self._standard_system.copy()
        if not remove_barostat and self._barostat_scale is not None and self._pressure is not None:
            system.addForce(self._anisotropic_barostat())
        return system

    def _anisotropic_barostat(self):
        return MonteCarloAnisotropicBarostat(self._pressure * unit.bar, self._temperature * unit.kelvin, *self._barostat_scale)

    def _rehash(self):
        """The standard system's hash; an anisotropic barostat's kind and scaled axes count, its pressure does not."""
        system = self._standard_system
        if self._barostat_scale is not None:
            system = copy.copy(system)
            system.forces = [MonteCarloAnisotropicBarostat(1.0 * unit.bar, 300.0 * unit.kelvin, *self._barostat_scale)]
        self._standard_system_hash = system.standard_hash()

    # -- thermodynamic parameters
    @property
    def temperature(self):
        return self._temperature * unit.kelvin

    @temperature.setter
    def temperature(self, value):
        if value is None:
            raise ThermodynamicsError(ThermodynamicsError.NONE_TEMPERATURE)
        t = float(unit.to_md(value, unit.kelvin, 'temperature'))
        if not t > 0:
            raise ValueError('temperature must be positive')
        self._temperature = t

    @property
    def kT(self):
        return kB * self.temperature

    @property
    def beta(self):
        return 1.0 / self.kT

    @property
    def pressure(self):
        """Pressure of the NPT ensemble, or None in the NVT ensemble (states.py:679-703)."""
        return None if self._pressure is None else self._pressure * unit.bar

    @pressure.setter
    def pressure(self, value):
        if value is None:
            self._pressure = None
            if self._barostat_scale is not None:   # the anisotropic barostat goes with its pressure
                self._barostat_scale = None
                self._rehash()
            return
        if not self.is_periodic:
            raise ThermodynamicsError(ThermodynamicsError.BAROSTATED_NONPERIODIC)
        if not (isinstance(value, unit.Quantity) and value.unit.is_compatible(unit.bar)):
            raise TypeError('pressure must be a Quantity with units of pressure (e.g. 1.0 * unit.bar), got %r' % (value,))
        p = float(value / unit.bar)
        if not p > 0:
            raise ValueError('pressure must be positive')
        self._pressure = p

    @property
    def _pressure_md(self):
        """The pressure in kJ/mol/nm^3 (1 bar = 0.0602214076 kJ/mol/nm^3), or None."""
        if self._pressure is None:
            return None
        return float(unit.to_md(self._pressure * unit.bar * unit.AVOGADRO_CONSTANT_NA))

    @property
    def barostat(self):
        """An anisotropic state's MonteCarloAnisotropicBarostat record (at the state's pressure and temperature); None
        otherwise: the isotropic barostat is not an object here (the engine runs it), see ``pressure``."""
        return self._anisotropic_barostat() if self._barostat_scale is not None and self._pressure is not None else None

    @property
    def surface_tension(self):
        return None

    @property
    def default_box_vectors(self):
        return self._standard_system.getDefaultPeriodicBoxVectors()

    @property
    def volume(self):
        return self.get_volume()

    def get_volume(self, ignore_ensemble=False):
        if not self.is_periodic:
            return None
        bv = self._standard_system.box_vectors
        return float(abs(np.linalg.det(bv))) * unit.nanometer ** 3

    @property
    def n_particles(self):
        return self._standard_system.n_particles

    @property
    def is_periodic(self):
        return self._standard_system.usesPeriodicBoundaryConditions()

    # -- energies
    def reduced_potential(self, context_or_sampler_state):
        """u = beta * U(x) for this state (states.py:818-909); evaluated by the CUDA engine."""
        return float(self.reduced_potential_at_states(context_or_sampler_state, [self])[0])

    @classmethod
    def reduced_potential_at_states(cls, context, thermodynamic_states):
        """Reduced potentials of one configuration in several compatible states (states.py:911-992).

        ``context`` is a :class:`SamplerState` here (there is no OpenMM Context on this path).
        """
        if not isinstance(context, SamplerState):
            raise NotImplementedError('pass a SamplerState: there is no OpenMM Context in openmmtools_b200')
        from . import _backend
        return _backend.reduced_potentials(thermodynamic_states, context)

    # -- compatibility
    def is_state_compatible(self, thermodynamic_state):
        """Same standard system and ensemble, i.e. the two states differ only in thermodynamic parameters
        (states.py:994-1050)."""
        return (self._standard_system_hash == thermodynamic_state._standard_system_hash and
                (self._pressure is None) == (thermodynamic_state._pressure is None))

    def is_context_compatible(self, context):
        raise NotImplementedError('no OpenMM Context on the GPU path')

    def create_context(self, integrator, platform=None, platform_properties=None):
        raise NotImplementedError('no OpenMM Context on the GPU path; the engine owns the device state')

    def apply_to_context(self, context):
        raise NotImplementedError('no OpenMM Context on the GPU path')

    # -- engine-facing view of this state (overridden/extended by CompoundThermodynamicState)
    def _engine_parameters(self):
        s = self._standard_system
        p = dict(temperature=self._temperature, lambda_sterics=s.global_parameters.get('lambda_sterics', 1.0),
                 lambda_electrostatics=s.global_parameters.get('lambda_electrostatics', 1.0), ho_K=s.ho_K, ho_x0=s.ho_x0, ho_U0=s.ho_U0, pressure=self._pressure_md)
        if getattr(s, 'alchemical_regions', None) is not None:   # each region's lambda_sterics<suffix>
            for n in s.lambda_sterics_names():
                p[n] = s.global_parameters.get(n, 1.0)
        return p

    # -- copies share the (immutable) standard system like the reference (states.py:1235-1253)
    def __copy__(self):
        new = self.__class__.__new__(self.__class__)
        new.__dict__.update(self.__dict__)
        return new

    def __deepcopy__(self, memo):
        new = self.__class__.__new__(self.__class__)
        for k, v in self.__dict__.items():
            new.__dict__[k] = v if k == '_standard_system' else copy.deepcopy(v, memo)
        return new

    def __getstate__(self, skip_system=False):
        d = {k: v for k, v in self.__dict__.items()}
        if skip_system:
            d.pop('_standard_system')
        return d

    def __setstate__(self, d):
        self.__dict__.update(d)
        self.__dict__.setdefault('_pressure', None)
        self.__dict__.setdefault('_barostat_scale', None)


def _read_barostat(system):
    """(pressure in bar, scaled axes or None when isotropic) of the system's barostat record; None without one.  Raises
    what the reference raises for a system it cannot put in the NPT ensemble (states.py:1656-1693)."""
    baros = [f for f in getattr(system, 'forces', ()) if isinstance(f, BAROSTATS)]
    if not baros:
        return None
    if len(baros) > 1:
        raise ThermodynamicsError(ThermodynamicsError.MULTIPLE_BAROSTATS)
    if not system.usesPeriodicBoundaryConditions():
        raise ThermodynamicsError(ThermodynamicsError.BAROSTATED_NONPERIODIC)
    b = baros[0]
    if b.getFrequency() != 25:
        raise NotImplementedError('only barostat frequency 25 is provided, got %d' % b.getFrequency())
    if isinstance(b, MonteCarloBarostat):
        return b._pressure, None
    scale = tuple(b._scale)
    scaled = {p for p, s in zip(b._pressure, scale) if s}   # (the unscaled axes' pressures do not count)
    if len(scaled) != 1:
        raise ThermodynamicsError(ThermodynamicsError.UNSUPPORTED_ANISOTROPIC_BAROSTAT)
    return scaled.pop(), scale


def _without_barostats(system):
    s = system.copy()
    s.forces = []
    return s


# ------------------------------------------------------------------------------------------------------
class _FromStore:
    """Marker: the energy of an attached SamplerState is read from its sampler's host store (multistatesampler.py)."""

    def __repr__(self):
        return '<energy in the host store>'


_FROM_STORE = _FromStore()


class SamplerState:
    """Positions, velocities and box vectors of one replica (states.py:1933-2520)."""

    def __init__(self, positions, velocities=None, box_vectors=None):
        # a sampler with host-resident states keeps the arrays of all its replicas in one page-locked store and attaches
        # the states to it (positions/velocities are views, energies are read through `_store`); assigning new arrays
        # marks the store dirty so that the sampler picks them up
        self._store = None
        self._store_index = -1
        self._positions = None
        self._velocities = None
        self._box_vectors = None
        self._potential_energy = None
        self._kinetic_energy = None
        self._collective_variables = None
        self._unitless_positions_cache = None
        self.positions = positions
        self.velocities = velocities
        self.box_vectors = box_vectors

    @classmethod
    def from_context(cls, context_state, ignore_collective_variables=False):
        raise NotImplementedError('no OpenMM Context on the GPU path')

    @staticmethod
    def _as_array(value, name):
        a = np.array(unit.to_md(value, unit.nanometer if name == 'positions' else None, name), dtype=np.float64)
        if a.ndim != 2 or a.shape[1] != 3:
            raise ValueError('%s must have shape (n_particles, 3)' % name)
        return a

    @property
    def positions(self):
        return unit.Quantity(self._positions, unit.nanometer)

    @positions.setter
    def positions(self, value):
        if value is None:
            raise SamplerStateError(SamplerStateError.INCONSISTENT_POSITIONS)
        a = self._as_array(value, 'positions')
        if self._positions is not None and a.shape != self._positions.shape:
            raise SamplerStateError(SamplerStateError.INCONSISTENT_POSITIONS)
        self._positions = a
        if self._store is not None:
            self._store.dirty = True
        # new positions invalidate the cached potential energy (states.py:2386-2390)
        self._potential_energy = None
        self._collective_variables = None

    @property
    def velocities(self):
        return None if self._velocities is None else unit.Quantity(self._velocities, unit.nanometer / unit.picosecond)

    @velocities.setter
    def velocities(self, value):
        if value is None:
            self._velocities = None
        else:
            a = np.array(unit.to_md(value, unit.nanometer / unit.picosecond, 'velocities'), dtype=np.float64)
            if a.shape != self._positions.shape:
                raise SamplerStateError(SamplerStateError.INCONSISTENT_VELOCITIES)
            self._velocities = a
        if self._store is not None:
            self._store.dirty = True
        self._kinetic_energy = None

    @property
    def box_vectors(self):
        return None if self._box_vectors is None else unit.Quantity(self._box_vectors, unit.nanometer)

    @box_vectors.setter
    def box_vectors(self, value):
        if value is None:
            self._box_vectors = None
        else:
            self._box_vectors = np.array(unit.to_md(value, unit.nanometer, 'box_vectors'), dtype=np.float64).reshape(3, 3)

    @property
    def potential_energy(self):
        pe = self._potential_energy
        if pe is _FROM_STORE:
            pe = float(self._store.pot[self._store_index])
        if pe is None:
            return None
        return pe * unit.kilojoule_per_mole

    @potential_energy.setter
    def potential_energy(self, value):
        if value is not None:
            raise AttributeError("Cannot set potential energy as it is a function of Context")
        self._potential_energy = None

    @property
    def kinetic_energy(self):
        ke = self._kinetic_energy
        if ke is _FROM_STORE:
            ke = float(self._store.kin[self._store_index])
        if ke is None:
            return None
        return ke * unit.kilojoule_per_mole

    @kinetic_energy.setter
    def kinetic_energy(self, value):
        if value is not None:
            raise AttributeError("Cannot set kinetic energy as it is a function of Context")
        self._kinetic_energy = None

    @property
    def total_energy(self):
        if self._potential_energy is None or self._kinetic_energy is None:
            return None
        return self.potential_energy + self.kinetic_energy

    @property
    def collective_variables(self):
        return self._collective_variables

    @property
    def volume(self):
        if self._box_vectors is None:
            return None
        return float(abs(np.linalg.det(self._box_vectors))) * unit.nanometer ** 3

    @property
    def area_xy(self):
        if self._box_vectors is None:
            return None
        return float(self._box_vectors[0][0] * self._box_vectors[1][1]) * unit.nanometer ** 2

    @property
    def n_particles(self):
        return len(self._positions)

    def is_context_compatible(self, context):
        raise NotImplementedError('no OpenMM Context on the GPU path')

    def update_from_context(self, *a, **k):
        raise NotImplementedError('no OpenMM Context on the GPU path')

    def apply_to_context(self, *a, **k):
        raise NotImplementedError('no OpenMM Context on the GPU path')

    def has_nan(self):
        """True if any position is NaN (states.py:2281)."""
        return bool(np.isnan(self._positions).any())

    def __getitem__(self, item):
        """Slice particles (states.py:2297-2325)."""
        ss = SamplerState.__new__(SamplerState)
        ss.__dict__.update(self.__dict__)
        if np.issubdtype(type(item), np.integer):
            item = slice(item, item + 1) if item != -1 else slice(item, None)
        ss._positions = self._positions[item].copy()
        ss._velocities = None if self._velocities is None else self._velocities[item].copy()
        ss._box_vectors = copy.deepcopy(self._box_vectors)
        ss._potential_energy = None
        ss._kinetic_energy = None
        ss._store = None
        ss._store_index = -1
        return ss

    def __getstate__(self, ignore_velocities=False):
        """Dictionary with the reference's keys (states.py:2327-2343)."""
        velocities = None if ignore_velocities else self.velocities
        return dict(positions=self.positions, velocities=velocities, box_vectors=self.box_vectors,
                    potential_energy=self.potential_energy, kinetic_energy=self.kinetic_energy,
                    collective_variables=self.collective_variables)

    def __setstate__(self, serialization, ignore_velocities=False):
        self._store = getattr(self, '_store', None)
        self._store_index = getattr(self, '_store_index', -1)
        self._positions = None
        self._velocities = getattr(self, '_velocities', None)
        self._unitless_positions_cache = None
        self._collective_variables = None
        self.positions = serialization['positions']
        if not ignore_velocities:
            self._velocities = None
            self.velocities = serialization['velocities']
        self._box_vectors = None
        self.box_vectors = serialization['box_vectors']
        pe, ke = serialization.get('potential_energy'), serialization.get('kinetic_energy')
        self._potential_energy = None if pe is None else float(unit.to_md(pe))
        self._kinetic_energy = None if ke is None else float(unit.to_md(ke))

    def __copy__(self):
        return copy.deepcopy(self)

    # -- engine-side update (what update_from_context does in the reference, states.py:2215-2255)
    def _energies_md(self):
        """(potential, kinetic) as plain floats in kJ/mol, or None."""
        pe, ke = self.potential_energy, self.kinetic_energy
        return (None if pe is None else float(unit.to_md(pe)), None if ke is None else float(unit.to_md(ke)))

    def _update(self, positions, velocities, potential, kinetic):
        if self._store is not None:
            self._store.dirty = True
        self._positions = np.array(positions, dtype=np.float64)
        self._velocities = None if velocities is None else np.array(velocities, dtype=np.float64)
        self._potential_energy = None if potential is None else float(potential)
        self._kinetic_energy = None if kinetic is None else float(kinetic)


# ------------------------------------------------------------------------------------------------------
# Composable states (states.py:2694-3046, 3100+)
# ------------------------------------------------------------------------------------------------------
class GlobalParameterState:
    """A set of global parameters of the system, e.g. the alchemical lambdas (states.py:3100-3800)."""

    class GlobalParameter:
        """Descriptor for one parameter with a validator (states.py:3330-3400)."""

        def __init__(self, variable_name, standard_value, validator=None):
            self.variable_name = variable_name
            self.standard_value = standard_value
            self.validator_func = validator

        def __set_name__(self, owner, name):
            pass

        def __get__(self, instance, owner=None):
            if instance is None:
                return self
            self._check_controlled(instance)
            return instance._parameters[self.variable_name]

        def __set__(self, instance, new_value):
            self._check_controlled(instance)
            if self.variable_name not in instance._parameters or instance._parameters[self.variable_name] is None:
                if new_value is not None or self.variable_name not in instance._parameters:
                    raise GlobalParameterError(GlobalParameterError.PARAMETER_NOT_DEFINED,
                                               "Cannot set the parameter {} in the system as it was not defined.".format(self.variable_name))
            if self.validator_func is not None and new_value is not None:
                new_value = self.validator_func(instance, new_value)
            instance._parameters[self.variable_name] = new_value

        def validator(self, validator):
            self.validator_func = validator
            return validator

        def _check_controlled(self, instance):
            # a state with a parameter name suffix controls only the suffixed names (states.py:3469-3479)
            suffix = instance.__dict__.get('_parameters_name_suffix')
            if suffix is not None:
                raise AttributeError('This state does not control {} but {}.'.format(
                    self.variable_name, self.variable_name + '_' + suffix))

    def __init__(self, parameters_name_suffix=None, **kwargs):
        self._initialize(parameters_name_suffix=parameters_name_suffix, **kwargs)

    @classmethod
    def _get_controlled_parameters(cls, parameters_name_suffix=None):
        """name (with '_' + parameters_name_suffix appended, if given) -> descriptor (states.py:3698-3730)."""
        suffix = '' if parameters_name_suffix is None else '_' + parameters_name_suffix
        out = {}
        for klass in reversed(cls.__mro__):
            for name, d in vars(klass).items():
                if isinstance(d, GlobalParameterState.GlobalParameter):
                    out[d.variable_name + suffix] = d
        return out

    def _initialize(self, parameters_name_suffix=None, **kwargs):
        """kwargs by their unsuffixed names; stored under the suffixed ones (states.py:3932-3963)."""
        self.__dict__['_parameters_name_suffix'] = None
        controlled = self._get_controlled_parameters()
        suffixed = self._get_controlled_parameters(parameters_name_suffix)
        self._parameters = {name: None for name in suffixed}
        for name, value in kwargs.items():
            if name not in controlled:
                raise GlobalParameterError(GlobalParameterError.PARAMETER_NOT_DEFINED,
                                           'Unknown parameter {}'.format(name))
            d = controlled[name]
            if d.validator_func is not None and value is not None:
                value = d.validator_func(self, value)
            self._parameters[name if parameters_name_suffix is None else name + '_' + parameters_name_suffix] = value
        self.__dict__['_parameters_name_suffix'] = parameters_name_suffix

    def _suffixed_descriptor(self, key):
        """The descriptor of a suffixed parameter name this state controls, or None."""
        suffix = self.__dict__.get('_parameters_name_suffix')
        if suffix is None or key not in self.__dict__.get('_parameters', {}):
            return None
        return self._get_controlled_parameters(suffix)[key]

    def __getattr__(self, key):
        # only called when normal lookup fails: the suffixed parameters (states.py:3830-3839)
        if self._suffixed_descriptor(key) is not None:
            return self._parameters[key]
        raise AttributeError("{} object has no attribute '{}'".format(type(self).__name__, key))

    def __setattr__(self, key, value):
        d = self._suffixed_descriptor(key)
        if d is None:
            object.__setattr__(self, key, value)
            return
        if self._parameters[key] is None and value is not None:
            raise GlobalParameterError(GlobalParameterError.PARAMETER_NOT_DEFINED,
                                       'Cannot set the parameter {} in the system as it was not defined.'.format(key))
        if d.validator_func is not None and value is not None:
            value = d.validator_func(self, value)
        self._parameters[key] = value

    @classmethod
    def from_system(cls, system, parameters_name_suffix=None):
        """Read the parameters from the system's global-parameter defaults (alchemy.py:227-253); with a suffix, the
        parameters named ``name + '_' + parameters_name_suffix`` (states.py:3281-3334)."""
        suffix = '' if parameters_name_suffix is None else '_' + parameters_name_suffix
        controlled = cls._get_controlled_parameters()
        found = {n: system.global_parameters[n + suffix] for n in controlled if n + suffix in system.global_parameters}
        if not found:
            raise GlobalParameterError(GlobalParameterError.PARAMETER_NOT_DEFINED,
                                       'System has no global parameters {}.'.format(
                                           set(cls._get_controlled_parameters(parameters_name_suffix))))
        return cls(parameters_name_suffix=parameters_name_suffix, **found)

    def apply_to_system(self, system):
        for n, v in self._parameters.items():
            if v is None:
                continue
            if n not in system.global_parameters:
                raise GlobalParameterError(GlobalParameterError.PARAMETER_NOT_DEFINED,
                                           'Could not find global parameter {} in the system.'.format(n))
            system.global_parameters[n] = v

    def check_system_consistency(self, system):
        for n, v in self._parameters.items():
            if v is None:
                continue
            if n not in system.global_parameters:
                raise GlobalParameterError(GlobalParameterError.PARAMETER_NOT_DEFINED,
                                           'Could not find global parameter {} in the system.'.format(n))
            if system.global_parameters[n] != v:
                raise GlobalParameterError(GlobalParameterError.INCOMPATIBLE_PARAMETER_VALUE,
                                           'Global parameter {} is inconsistent.'.format(n))

    def apply_to_context(self, context):
        raise NotImplementedError('no OpenMM Context on the GPU path')

    def __eq__(self, other):
        return type(self) is type(other) and self._parameters == other._parameters

    def __ne__(self, other):
        return not self == other

    def __str__(self):
        return str(self._parameters)

    def __getstate__(self):
        # unsuffixed names plus the suffix, as the reference serialises them (states.py:3879-3898)
        suffix = self._parameters_name_suffix
        cut = 0 if suffix is None else len(suffix) + 1
        params = {n[:len(n) - cut]: v for n, v in self._parameters.items()}
        return dict(_parameters=params, _parameters_name_suffix=suffix)

    def __setstate__(self, s):
        suffix = s.get('_parameters_name_suffix')
        self.__dict__['_parameters_name_suffix'] = None
        self._parameters = {(n if suffix is None else n + '_' + suffix): v for n, v in s['_parameters'].items()}
        self.__dict__['_parameters_name_suffix'] = suffix


class CompoundThermodynamicState(ThermodynamicState):
    """A ThermodynamicState extended by composable states whose attributes pass through (states.py:2694-3046)."""

    def __init__(self, thermodynamic_state, composable_states):
        # share the standard system with the wrapped state like the reference's dynamic subclassing does
        self.__dict__.update(copy.copy(thermodynamic_state).__dict__)
        self.__dict__['_composable_states'] = [copy.deepcopy(s) for s in composable_states]
        for s in self._composable_states:
            s.check_system_consistency if False else None
            s_params = getattr(s, '_parameters', {})
            missing = [n for n, v in s_params.items() if v is not None and n not in self._standard_system.global_parameters]
            if missing:
                raise GlobalParameterError(GlobalParameterError.PARAMETER_NOT_DEFINED,
                                           'Could not find global parameter {} in the system.'.format(missing[0]))

    def _find(self, name):
        for s in self.__dict__.get('_composable_states', ()):
            if name in getattr(s, '_parameters', {}):
                return s
            if isinstance(getattr(type(s), name, None), (property, GlobalParameterState.GlobalParameter)):
                return s
        return None

    def __getattr__(self, name):
        # only called when normal lookup fails
        if name.startswith('__'):
            raise AttributeError(name)
        s = self._find(name)
        if s is not None:
            return getattr(s, name)
        for cs in self.__dict__.get('_composable_states', ()):
            if hasattr(type(cs), name):
                return getattr(cs, name)
        raise AttributeError("{} object has no attribute '{}'".format(type(self).__name__, name))

    def __setattr__(self, name, value):
        if name in self.__dict__ or hasattr(type(self), name):
            object.__setattr__(self, name, value)
            return
        s = self._find(name)
        if s is not None:
            setattr(s, name, value)
        else:
            object.__setattr__(self, name, value)

    def get_system(self, **kwargs):
        system = super().get_system(**kwargs)
        for s in self._composable_states:
            s.apply_to_system(system)
        return system

    def set_system(self, system, fix_state=False):
        system = system.copy()
        for s in self._composable_states:
            if fix_state:
                s.apply_to_system(system)
            else:
                s.check_system_consistency(system)
        super().set_system(system)

    def is_state_compatible(self, thermodynamic_state):
        return super().is_state_compatible(thermodynamic_state)

    def _engine_parameters(self):
        p = super()._engine_parameters()
        for s in self._composable_states:
            for n, v in getattr(s, '_parameters', {}).items():
                if v is not None and (n.startswith('lambda_sterics') or n == 'lambda_electrostatics'):   # (with a region's suffix, if any)
                    p[n] = v
        return p

    def __getstate__(self, **kwargs):
        d = super().__getstate__(**kwargs)
        return d

    def __setstate__(self, d):
        self.__dict__.update(d)


def create_thermodynamic_state_protocol(system, protocol, constants=None, composable_states=None):
    """One state per protocol point (states.py:39-141).

    ``protocol`` maps attribute names (``temperature``, ``lambda_sterics`` ...) to equal-length lists.
    """
    lengths = {len(v) for v in protocol.values()}
    if len(lengths) != 1:
        raise ValueError('The protocol parameter values have different lengths!')
    n = lengths.pop()
    if constants is None:
        constants = {}
    if isinstance(system, ThermodynamicState):
        base = system
    else:
        temperature = constants.get('temperature', protocol['temperature'][0] if 'temperature' in protocol else None)
        if temperature is None:
            raise ValueError('If a System is passed the constants must specify the temperature.')
        base = ThermodynamicState(system, temperature=temperature)
    if composable_states is not None:
        if isinstance(composable_states, GlobalParameterState):
            composable_states = [composable_states]
        base = CompoundThermodynamicState(base, composable_states=list(composable_states))
    for name, value in constants.items():
        setattr(base, name, value)
    states = []
    for i in range(n):
        s = copy.deepcopy(base)
        for name, values in protocol.items():
            if not hasattr(s, name):
                raise AttributeError('{} object has no attribute {}'.format(type(s).__name__, name))
            setattr(s, name, values[i])
        states.append(s)
    return states


def group_by_compatibility(states):
    """Indices of mutually compatible states (states.py:186-217)."""
    groups = {}
    for i, s in enumerate(states):
        groups.setdefault(s._standard_system_hash, []).append(i)
    return list(groups.values())
