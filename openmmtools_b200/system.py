"""A light parameter record standing in for ``openmm.System`` on the replica-exchange path.

The reference builds OpenMM ``System`` objects (NonbondedForce / CustomNonbondedForce / CustomExternalForce,
/root/reference/openmmtools/testsystems.py:779-788,1956-1997; alchemy/alchemy.py:1539-2038) and OpenMM evaluates
them.  Here the same physics is described by plain numbers that the CUDA engine consumes; nothing in this module
imports OpenMM.
"""
import copy
import hashlib
import numpy as np

LJ, HARMONIC, MOLECULE = 'lj', 'harmonic', 'molecule'


def _bar(value, name='pressure'):
    from . import unit
    if not (isinstance(value, unit.Quantity) and value.unit.is_compatible(unit.bar)):
        raise TypeError('%s must be a Quantity with units of pressure (e.g. 1.0 * unit.bar), got %r' % (name, value))
    return value.value_in_unit(unit.bar)


def _kelvin(value):
    from . import unit
    return float(unit.to_md(value, unit.kelvin, 'temperature'))


class MonteCarloBarostat:
    """Record of OpenMM's isotropic ``MonteCarloBarostat(defaultPressure, defaultTemperature, frequency=25)``.

    ``ThermodynamicState(system, temperature)`` on a system holding it is NPT at its pressure, exactly as
    ``ThermodynamicState(system, temperature, pressure)`` on the system without it.  The CUDA engine runs the move."""

    def __init__(self, defaultPressure, defaultTemperature, frequency=25):
        self.setDefaultPressure(defaultPressure)
        self.setDefaultTemperature(defaultTemperature)
        self.setFrequency(frequency)

    def getDefaultPressure(self):
        from . import unit
        return self._pressure * unit.bar

    def setDefaultPressure(self, pressure):
        self._pressure = float(_bar(pressure))

    def getDefaultTemperature(self):
        from . import unit
        return self._temperature * unit.kelvin

    def setDefaultTemperature(self, temperature):
        self._temperature = _kelvin(temperature)

    def getFrequency(self):
        return self._frequency

    def setFrequency(self, frequency):
        self._frequency = int(frequency)

    def _hash_key(self):
        return b'MonteCarloBarostat'


class MonteCarloAnisotropicBarostat:
    """Record of OpenMM's ``MonteCarloAnisotropicBarostat(defaultPressure, defaultTemperature, scaleX, scaleY, scaleZ,
    frequency=25)``: each attempt scales one box edge, chosen among the scaled axes.  ``defaultPressure`` is a pressure
    per axis (x, y, z), or one pressure for all three."""

    def __init__(self, defaultPressure, defaultTemperature, scaleX=True, scaleY=True, scaleZ=True, frequency=25):
        self.setDefaultPressure(defaultPressure)
        self.setDefaultTemperature(defaultTemperature)
        self._scale = [bool(scaleX), bool(scaleY), bool(scaleZ)]
        self.setFrequency(frequency)

    def getDefaultPressure(self):
        from . import unit
        return unit.Quantity(np.array(self._pressure), unit.bar)

    def setDefaultPressure(self, pressure):
        from . import unit
        if isinstance(pressure, (list, tuple)) and len(pressure) == 3 and all(isinstance(p, unit.Quantity) for p in pressure):
            p = [_bar(q) for q in pressure]
        else:
            p = _bar(pressure)
        p = np.broadcast_to(np.asarray(p, np.float64), (3,))
        self._pressure = tuple(float(v) for v in p)

    def getDefaultTemperature(self):
        from . import unit
        return self._temperature * unit.kelvin

    def setDefaultTemperature(self, temperature):
        self._temperature = _kelvin(temperature)

    def getScaleX(self):
        return self._scale[0]

    def getScaleY(self):
        return self._scale[1]

    def getScaleZ(self):
        return self._scale[2]

    def setScaleX(self, scale):
        self._scale[0] = bool(scale)

    def setScaleY(self, scale):
        self._scale[1] = bool(scale)

    def setScaleZ(self, scale):
        self._scale[2] = bool(scale)

    def getFrequency(self):
        return self._frequency

    def setFrequency(self, frequency):
        self._frequency = int(frequency)

    def _hash_key(self):
        return b'MonteCarloAnisotropicBarostat' + repr(tuple(self._scale)).encode()


BAROSTATS = (MonteCarloBarostat, MonteCarloAnisotropicBarostat)


class System:
    """Parameters of one of the supported systems (md units: nm, ps, dalton, kJ/mol)."""

    def __init__(self, kind, masses, box_vectors=None):
        if kind not in (LJ, HARMONIC, MOLECULE):
            raise ValueError('unsupported system kind %r' % (kind,))
        self.kind = kind
        self.masses = np.array(masses, dtype=np.float64)
        self.box_vectors = None if box_vectors is None else np.array(box_vectors, dtype=np.float64).reshape(3, 3)
        # -- Lennard-Jones fluid (NonbondedForce, CutoffPeriodic)
        self.sigma = None
        self.epsilon = None
        self.charge = None
        self.cutoff = None
        self.switching_distance = None
        self.use_switching_function = False
        self.use_dispersion_correction = False
        # -- alchemical modification (AbsoluteAlchemicalFactory)
        self.alchemical_atoms = None          # sorted tuple of atom indices, None = not alchemically modified
        self.annihilate_sterics = False
        self.annihilate_electrostatics = True   # (molecules; the LJ fluid has no charges)
        self.alchemical_obc2 = False            # (molecules in OBC2: the alchemical expression's own constants)
        self.softcore_alpha = 0.5
        self.softcore_a = 1.0
        self.softcore_b = 1.0
        self.softcore_c = 6.0
        self.alchemical_dispersion_correction = False
        # two alchemical regions: ((name, atoms, annihilate_sterics), (name, atoms, annihilate_sterics)), regions 1 and 2
        # (alchemical_atoms is then their union); None: one region or none
        self.alchemical_regions = None
        # -- harmonic oscillator (CustomExternalForce global parameters)
        self.ho_K = None
        self.ho_x0 = (0.0, 0.0, 0.0)
        self.ho_U0 = 0.0
        # -- small molecule in vacuum (HarmonicBond/Angle, PeriodicTorsion, NonbondedForce NoCutoff + exceptions, HBonds
        #    constraints, CMMotionRemover): what AmberPrmtopFile.createSystem builds for AlanineDipeptideVacuum
        self.bonds = None          # float64[nb, 4]  i, j, K (kJ/mol/nm^2), r0 (nm)        1/2 K (r - r0)^2
        self.angles = None         # float64[na, 5]  i, j, k, K (kJ/mol/rad^2), theta0     1/2 K (t - t0)^2
        self.torsions = None       # float64[nt, 7]  i, j, k, l, n, phase, k (kJ/mol)      k (1 + cos(n phi - phase))
        self.exclusions = None     # int[ne, 2]      pairs without any nonbonded interaction (1-2, 1-3)
        self.exceptions = None     # float64[nx, 5]  i, j, q_i q_j (scaled), sigma, epsilon (scaled): the 1-4 pairs
        self.constraints = None    # float64[nc, 3]  i, j, distance (nm)
        self.remove_cm_motion = False
        # -- OBC generalized Born implicit solvent (GBSAOBCForce, createSystem(implicitSolvent=OBC1|OBC2)); None: vacuum
        self.gb_radius = None      # float64[n]  radius (nm)
        self.gb_scale = None       # float64[n]  screening factor
        self.gb_parameters = None  # (alpha, beta, gamma, offset, solute dielectric, solvent dielectric, sa_energy, probe radius)
        # -- OpenMM-style global parameters with their defaults (read by GlobalParameterState.from_system)
        self.global_parameters = {}
        # -- forces added with addForce: barostat records only (the other forces are the parameters above)
        self.forces = []

    # -- OpenMM-flavoured accessors used by user code on this path
    def getNumParticles(self):
        return len(self.masses)

    def getParticleMass(self, i):
        from . import unit
        return self.masses[i] * unit.dalton

    def getDefaultPeriodicBoxVectors(self):
        from . import unit
        return unit.Quantity(self.box_vectors.copy(), unit.nanometer)

    def setDefaultPeriodicBoxVectors(self, a, b, c):
        from . import unit
        self.box_vectors = np.array([unit.to_md(a), unit.to_md(b), unit.to_md(c)], dtype=np.float64)

    def addForce(self, force):
        """Add a barostat record (MonteCarloBarostat or MonteCarloAnisotropicBarostat); returns its index."""
        if not isinstance(force, BAROSTATS):
            raise NotImplementedError('only barostat records can be added to a System, got %r' % type(force).__name__)
        self.forces.append(force)
        return len(self.forces) - 1

    def getForces(self):
        return list(self.forces)

    def getNumForces(self):
        return len(self.forces)

    def getForce(self, index):
        return self.forces[index]

    def removeForce(self, index):
        del self.forces[index]

    def usesPeriodicBoundaryConditions(self):
        return self.kind == LJ

    def getNumConstraints(self):
        return 0 if self.constraints is None else len(self.constraints)

    @property
    def n_particles(self):
        return len(self.masses)

    @property
    def is_alchemical(self):
        return self.alchemical_atoms is not None

    def alchemical_mask(self):
        m = np.zeros(self.n_particles, np.uint8)
        if self.alchemical_atoms:
            m[list(self.alchemical_atoms)] = 1
        return m

    def alchemical_region_ids(self):
        """Per-atom region id: 0 environment, 1 and 2 the atoms of the two alchemical regions."""
        ids = np.zeros(self.n_particles, np.uint8)
        for r, (_, atoms, _) in enumerate(self.alchemical_regions or ()):
            ids[list(atoms)] = r + 1
        return ids

    def lambda_sterics_names(self):
        """The global parameter controlling each alchemical region's sterics (lambda_sterics<suffix>)."""
        if self.alchemical_regions is None:
            return ('lambda_sterics',)
        return tuple('lambda_sterics' + ('' if name is None else '_' + name) for name, _, _ in self.alchemical_regions)

    def copy(self):
        return copy.deepcopy(self)

    # -- the equivalent of ThermodynamicState._standard_system_hash (states.py:1447-1504): everything except the
    # thermodynamic parameters (temperature, lambdas, HO K/x0/U0 which are global parameters in the reference)
    def standard_hash(self):
        h = hashlib.sha1()
        h.update(self.kind.encode())
        h.update(self.masses.tobytes())
        if self.box_vectors is not None:
            h.update(self.box_vectors.tobytes())
        if self.kind == LJ:
            for a in (self.sigma, self.epsilon, self.charge):
                h.update(np.asarray(a, dtype=np.float64).tobytes())
            h.update(repr((self.cutoff, self.switching_distance, self.use_switching_function,
                           self.use_dispersion_correction, self.alchemical_atoms, self.annihilate_sterics,
                           self.softcore_alpha, self.softcore_a, self.softcore_b, self.softcore_c,
                           self.alchemical_dispersion_correction)).encode())
            if getattr(self, 'alchemical_regions', None) is not None:   # (one-region systems keep their hash)
                h.update(repr(self.alchemical_regions).encode())
        if self.kind == MOLECULE:
            for a in (self.sigma, self.epsilon, self.charge, self.bonds, self.angles, self.torsions, self.exclusions,
                      self.exceptions, self.constraints):
                h.update(np.asarray(a, dtype=np.float64).tobytes())
            h.update(repr(self.remove_cm_motion).encode())
            if getattr(self, 'gb_radius', None) is not None:   # (vacuum systems keep their hash)
                for a in (self.gb_radius, self.gb_scale):
                    h.update(np.asarray(a, dtype=np.float64).tobytes())
                h.update(repr(tuple(float(v) for v in self.gb_parameters)).encode())
            if self.is_alchemical:   # (other molecules keep their hash)
                h.update(repr((self.alchemical_atoms, self.annihilate_sterics, self.annihilate_electrostatics,
                               self.softcore_alpha, self.softcore_a, self.softcore_b, self.softcore_c)).encode())
        for f in getattr(self, 'forces', ()):   # a barostat's kind and scaled axes, not its pressure (systems without keep their hash)
            h.update(f._hash_key())
        return h.hexdigest()

    def __getstate__(self):
        return self.__dict__.copy()

    def __setstate__(self, d):
        self.__dict__.update(d)
        self.__dict__.setdefault('alchemical_regions', None)
        self.__dict__.setdefault('forces', [])
        self.__dict__.setdefault('annihilate_electrostatics', True)
        self.__dict__.setdefault('alchemical_obc2', False)
