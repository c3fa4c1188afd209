"""The test systems the replica-exchange configurations use, as light parameter records.

Mirrors /root/reference/openmmtools/testsystems.py: ``HarmonicOscillator`` (:685-840) and
``LennardJonesFluid`` (:1872-2030) with the same constructor arguments, defaults and derived quantities
(box edge from the reduced density, cutoff 3 sigma, switching distance cutoff - switch_width, sub-random
initial positions), ``AlanineDipeptideVacuum`` (:3352-3388) and ``AlanineDipeptideImplicit`` (:3422-3459), and the toluene
systems (:3533-3636) from the reference's AMBER input files (``amber.py``; the parsed parameters ship as data/*.json).  The
other reference systems are out of scope.
"""
import numpy as np
from . import unit
from .constants import kB
from .system import System, LJ, HARMONIC, MOLECULE
from . import sobol


class TestSystem:
    """Base class: ``.system``, ``.positions`` (Quantity, nm), ``.name``, ``analytical_properties``."""
    __test__ = False   # not a pytest class

    def __init__(self, **kwargs):
        self._system = None
        self._positions = None
        self.topology = None

    @property
    def system(self):
        return self._system

    @system.setter
    def system(self, value):
        self._system = value

    @property
    def positions(self):
        return self._positions

    @positions.setter
    def positions(self, value):
        self._positions = value

    @property
    def name(self):
        return self.__class__.__name__

    @property
    def analytical_properties(self):
        return [m[4:] for m in dir(self) if m.startswith('get_') and m != 'get_name']


def subrandom_particle_positions(nparticles, box_vectors, method='sobol'):
    """Deterministic sub-random positions in the box (testsystems.py:236-289); float32 like the reference."""
    if method != 'sobol':
        raise NotImplementedError("only method='sobol' is provided")
    bv = np.asarray(unit.to_md(box_vectors), dtype=np.float64).reshape(3, 3)
    x = np.array(sobol.sobol_generate(3, nparticles, 1), np.float32)
    positions = np.zeros([nparticles, 3], np.float32)
    for dim in range(3):
        positions[:, dim] = x[dim, :] * bv[dim, dim]
    return unit.Quantity(positions, unit.nanometers)


class HarmonicOscillator(TestSystem):
    """A 3D harmonic oscillator: one particle, U = (K/2) ((x-x0)^2 + y^2 + z^2) + U0 (testsystems.py:761-788)."""

    def __init__(self, K=100.0 * unit.kilocalories_per_mole / unit.angstroms ** 2, mass=39.948 * unit.amu,
                 U0=0.0 * unit.kilojoules_per_mole, **kwargs):
        TestSystem.__init__(self, **kwargs)
        edge = 1000.0
        system = System(HARMONIC, [unit.to_md(mass, unit.dalton, 'mass')],
                        box_vectors=[[edge, 0, 0], [0, edge, 0], [0, 0, edge]])
        system.ho_K = float(unit.to_md(K, unit.kilojoule_per_mole / unit.nanometer ** 2, 'K'))
        system.ho_x0 = (0.0, 0.0, 0.0)
        system.ho_U0 = float(unit.to_md(U0, unit.kilojoule_per_mole, 'U0'))
        system.global_parameters = {'testsystems_HarmonicOscillator_K': system.ho_K,
                                    'testsystems_HarmonicOscillator_x0': 0.0,
                                    'testsystems_HarmonicOscillator_U0': system.ho_U0}
        self.K, self.mass, self.U0 = K, mass, U0
        self.system = system
        self.positions = unit.Quantity(np.zeros([1, 3], np.float32), unit.angstroms)
        self.ndof = 3

    def get_potential_expectation(self, state):
        return (3. / 2.) * kB * state.temperature

    def get_potential_standard_deviation(self, state):
        return (3. / 2.) * kB * state.temperature   # as the reference (testsystems.py:838-840)


class LennardJonesFluid(TestSystem):
    """A periodic fluid of Lennard-Jones particles (testsystems.py:1872-2030), zero charge only."""

    def __init__(self, nparticles=1000, reduced_density=0.05, mass=39.9 * unit.amu, sigma=3.4 * unit.angstrom,
                 epsilon=0.238 * unit.kilocalories_per_mole, cutoff=None, switch_width=3.4 * unit.angstrom,
                 shift=False, dispersion_correction=True, lattice=False, charge=None, ewaldErrorTolerance=None,
                 **kwargs):
        TestSystem.__init__(self, **kwargs)
        if charge is not None:
            raise NotImplementedError('charged Lennard-Jones fluids (PME) are outside the replica-exchange hot path')
        if shift:
            raise NotImplementedError('shift=True (CustomNonbondedForce constant shift) is not provided')
        if lattice:
            raise NotImplementedError('lattice=True needs mdtraj in the reference; not provided')
        sig = float(unit.to_md(sigma, unit.nanometer, 'sigma'))
        eps = float(unit.to_md(epsilon, unit.kilojoule_per_mole, 'epsilon'))
        m = float(unit.to_md(mass, unit.dalton, 'mass'))
        rc = 3.0 * sig if cutoff is None else float(unit.to_md(cutoff, unit.nanometer, 'cutoff'))
        # testsystems.py:1932-1939
        number_density = reduced_density / sig ** 3
        volume = nparticles / number_density
        box_edge = volume ** (1. / 3.)
        system = System(LJ, [m] * nparticles, box_vectors=np.eye(3) * box_edge)
        system.sigma = np.full(nparticles, sig)
        system.epsilon = np.full(nparticles, eps)
        system.charge = np.zeros(nparticles)
        system.cutoff = rc
        system.use_dispersion_correction = bool(dispersion_correction)
        system.use_switching_function = False
        system.switching_distance = rc
        if switch_width is not None and not shift:   # testsystems.py:1986-1989
            system.use_switching_function = True
            system.switching_distance = rc - float(unit.to_md(switch_width, unit.nanometer, 'switch_width'))
        if rc > box_edge / 2:
            raise ValueError('cutoff (%g nm) exceeds half the box edge (%g nm)' % (rc, box_edge))
        self.system = system
        self.positions = subrandom_particle_positions(nparticles, system.getDefaultPeriodicBoxVectors())
        self.nparticles = nparticles
        self.reduced_density = reduced_density


def _load_data(name):
    import json, os
    return json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'data', name)))


def _molecule(d, constraints, hydrogenMass):
    """The System createSystem(constraints=constraints, nonbondedCutoff=None) builds from the parsed prmtop d (vacuum)."""
    if hydrogenMass is not None:
        raise NotImplementedError('hydrogen mass repartitioning is not provided')
    name = getattr(constraints, '__name__', constraints)
    if name not in ('HBonds', None):
        raise NotImplementedError("constraints must be 'HBonds' or None")
    system = System(MOLECULE, d['mass'])
    system.charge = np.array(d['charge']); system.sigma = np.array(d['sigma']); system.epsilon = np.array(d['epsilon'])
    hb = name == 'HBonds'
    system.bonds = np.array([[b[0], b[1], b[2], b[3]] for b in d['bonds'] if not (hb and b[4])], dtype=np.float64).reshape(-1, 4)
    system.constraints = np.array([[b[0], b[1], b[3]] for b in d['bonds'] if hb and b[4]], dtype=np.float64).reshape(-1, 3)
    system.angles = np.array(d['angles'], dtype=np.float64).reshape(-1, 5)
    system.torsions = np.array(d['torsions'], dtype=np.float64).reshape(-1, 7)
    system.exclusions = np.array(d['exclusions'], dtype=np.int64).reshape(-1, 2)
    system.exceptions = np.array(d['exceptions'], dtype=np.float64).reshape(-1, 5)
    system.remove_cm_motion = True     # createSystem(removeCMMotion=True) is the default
    return system


def _add_obc(system, gb, **create_system_kwargs):
    """createSystem(implicitSolvent=...): the file's GB radii and screening factors with the model's parameters."""
    from .amber import obc_parameters
    system.gb_parameters = obc_parameters(**create_system_kwargs)
    system.gb_radius = np.array(gb['radii'], dtype=np.float64)
    system.gb_scale = np.array(gb['screen'], dtype=np.float64)
    return system


class AlanineDipeptideVacuum(TestSystem):
    """Alanine dipeptide (ff96) in vacuum (testsystems.py:3352-3388): what AmberPrmtopFile.createSystem(implicitSolvent=None,
    constraints=constraints, nonbondedCutoff=None) builds from alanine-dipeptide.prmtop -- harmonic bonds and angles, periodic
    torsions, Coulomb + Lennard-Jones over all pairs with 1-2/1-3 exclusions and scaled 1-4 pairs, constraints on the bonds
    to hydrogen (their bond terms dropped), centre-of-mass motion removal -- and the positions of alanine-dipeptide.crd.

    ``constraints``: 'HBonds' (the reference default, app.HBonds) or None."""

    def __init__(self, constraints='HBonds', hydrogenMass=None, **kwargs):
        TestSystem.__init__(self, **kwargs)
        d = _load_data('alanine_dipeptide_vacuum.json')
        self.system = _molecule(d, constraints, hydrogenMass)
        self.positions = unit.Quantity(np.array(d['positions'], dtype=np.float64), unit.nanometer)
        self.atom_names = list(d['names'])


class AlanineDipeptideImplicit(TestSystem):
    """Alanine dipeptide (ff96) in OBC1 implicit solvent (testsystems.py:3422-3459): AlanineDipeptideVacuum's force field
    plus the GB model createSystem(implicitSolvent=OBC1) adds -- the prmtop's mbondi2 radii and screening factors, solvent
    dielectric 78.5, the ACE non-polar term.

    ``constraints``: 'HBonds' (the reference default, app.HBonds) or None."""

    def __init__(self, constraints='HBonds', hydrogenMass=None, **kwargs):
        TestSystem.__init__(self, **kwargs)
        d = _load_data('alanine_dipeptide_vacuum.json')
        self.system = _add_obc(_molecule(d, constraints, hydrogenMass), _load_data('alanine_dipeptide_implicit.json'),
                               implicitSolvent='OBC1')
        self.positions = unit.Quantity(np.array(d['positions'], dtype=np.float64), unit.nanometer)
        self.atom_names = list(d['names'])


class TolueneVacuum(TestSystem):
    """Toluene GAFF/AM1-BCC in vacuum (testsystems.py:3533-3562), from benzene-toluene-implicit/solvent.{prmtop,inpcrd}."""

    def __init__(self, constraints='HBonds', hydrogenMass=None, **kwargs):
        TestSystem.__init__(self, **kwargs)
        d = _load_data('toluene_implicit.json')
        self.system = _molecule(d, constraints, hydrogenMass)
        self.positions = unit.Quantity(np.array(d['positions'], dtype=np.float64), unit.nanometer)
        self.atom_names = list(d['names'])


class TolueneImplicit(TestSystem):
    """Toluene GAFF/AM1-BCC in implicit solvent (testsystems.py:3568-3620): createSystem(**kwargs) with the defaults
    implicitSolvent=OBC1, constraints=HBonds, nonbondedMethod=NoCutoff; the prmtop's mbondi radii.  OBC1 and OBC2 are
    provided; HCT, GBn, GBn2, salt and cutoffs raise NotImplementedError."""

    def __init__(self, **kwargs):
        TestSystem.__init__(self)
        kw = dict(implicitSolvent='OBC1', constraints='HBonds', hydrogenMass=None)
        kw.update(kwargs)
        d = _load_data('toluene_implicit.json')
        constraints, hydrogenMass = kw.pop('constraints'), kw.pop('hydrogenMass')
        self.system = _add_obc(_molecule(d, constraints, hydrogenMass), d, **kw)
        self.positions = unit.Quantity(np.array(d['positions'], dtype=np.float64), unit.nanometer)
        self.atom_names = list(d['names'])


class TolueneImplicitHCT(TolueneImplicit):
    def __init__(self, **kwargs):
        TolueneImplicit.__init__(self, implicitSolvent='HCT', **kwargs)


class TolueneImplicitOBC1(TolueneImplicit):
    def __init__(self, **kwargs):
        TolueneImplicit.__init__(self, implicitSolvent='OBC1', **kwargs)


class TolueneImplicitOBC2(TolueneImplicit):
    def __init__(self, **kwargs):
        TolueneImplicit.__init__(self, implicitSolvent='OBC2', **kwargs)


class TolueneImplicitGBn(TolueneImplicit):
    def __init__(self, **kwargs):
        TolueneImplicit.__init__(self, implicitSolvent='GBn', **kwargs)


class TolueneImplicitGBn2(TolueneImplicit):
    def __init__(self, **kwargs):
        TolueneImplicit.__init__(self, implicitSolvent='GBn2', **kwargs)


class LennardJonesGrid(TestSystem):   # pragma: no cover
    def __init__(self, *a, **k):
        raise NotImplementedError('out of scope for the replica-exchange hot path')
