"""Alchemical modification of the Lennard-Jones test system and of small molecules, and the AlchemicalState that controls it.

Mirrors /root/reference/openmmtools/alchemy/alchemy.py for the pieces the replica-exchange path exercises:
``AlchemicalState`` (:90-410), ``AlchemicalRegion`` (:417-427) and
``AbsoluteAlchemicalFactory.create_alchemical_system`` (:637-754).  What the factory does to a zero-charge LJ
fluid (:1539-2038) is restated as parameters of the CUDA energy function: non-alchemical pairs keep plain LJ
(NonbondedForce with the alchemical epsilons zeroed, :1903-1909), alchemical/non-alchemical pairs use soft-core
sterics controlled by ``lambda_sterics`` (:1383-1388, interaction group :1915), alchemical/alchemical pairs use
the same expression with lambda fixed to 1 unless ``annihilate_sterics`` (:1776-1777, group :1919).  Small molecules:
see below; alchemical bonds, angles and torsions are not provided.

Two alchemical regions (a list of two ``AlchemicalRegion``, e.g. ``name=None`` or ``'A'`` plus ``'B'``) are the
dual-topology / separated-topology set-up: the epsilons of both regions are zeroed in the NonbondedForce, each region r
gets its own environment x r and r x r groups driven by ``lambda_sterics<suffix_r>`` (suffix ``'_' + name``, or none for
``name=None``; :1695-1700, 1752-1777), and pairs across the two regions have no interaction (no
``alchemical_regions_interactions``, :1684-1685).  Control them with one ``AlchemicalState`` per region, built with
``parameters_name_suffix``::

    regions = [AlchemicalRegion(alchemical_atoms=range(5), name='A'),
               AlchemicalRegion(alchemical_atoms=range(5, 10), name='B', annihilate_sterics=True)]
    system = AbsoluteAlchemicalFactory().create_alchemical_system(fluid.system, regions)
    state_a = AlchemicalState.from_system(system, parameters_name_suffix='A')
    state_b = AlchemicalState.from_system(system, parameters_name_suffix='B')

Up to two regions; both must use the same soft-core constants (OpenMM keeps one value per global parameter name,
:2009-2017), their ``annihilate_sterics`` may differ.

A small molecule (``MOLECULE`` systems: TolueneVacuum, TolueneImplicit, AlanineDipeptide*, in vacuum or OBC1/OBC2 implicit
solvent) takes one region.  Its pairs and 1-4 exceptions with one alchemical atom get soft-core sterics driven by
``lambda_sterics`` and Coulomb scaled by ``lambda_electrostatics`` (:1380-1450, 1840-1880; NoCutoff, so the soft-core
electrostatic radius is r); pairs of two alchemical atoms the same with each lambda fixed to 1 unless
``annihilate_sterics`` / ``annihilate_electrostatics``.  The OBC terms are scaled by w_i = lambda_electrostatics alch_i +
(1 - alch_i) as the reference rewrites them (OBC1: :2223-2300; OBC2: :2144-2221, with that expression's own constants)::

    toluene = testsystems.TolueneImplicit()
    system = AbsoluteAlchemicalFactory().create_alchemical_system(toluene.system, AlchemicalRegion(alchemical_atoms=range(15)))
    protocol = {'lambda_electrostatics': [1.0, 0.5, 0.0, 0.0, 0.0], 'lambda_sterics': [1.0, 1.0, 1.0, 0.5, 0.0]}
"""
import collections
import numpy as np
from . import unit
from .states import GlobalParameterState, GlobalParameterError   # noqa: F401
from .system import System, LJ, MOLECULE
from .amber import OBC_MODELS


class AlchemicalStateError(GlobalParameterError):
    pass


class AlchemicalState(GlobalParameterState):
    """lambda_sterics, lambda_electrostatics, lambda_bonds, lambda_angles, lambda_torsions in [0, 1]
    (alchemy.py:90-410)."""

    class _LambdaParameter(GlobalParameterState.GlobalParameter):
        def __init__(self, name):
            super().__init__(name, standard_value=1.0, validator=self.lambda_validator)

        @staticmethod
        def lambda_validator(self_, new_value):
            if new_value is None:
                return None
            if not (0.0 <= new_value <= 1.0):      # alchemy.py:213-219
                raise ValueError('{} must be between 0 and 1'.format(new_value))
            return float(new_value)

    lambda_sterics = _LambdaParameter('lambda_sterics')
    lambda_electrostatics = _LambdaParameter('lambda_electrostatics')
    lambda_bonds = _LambdaParameter('lambda_bonds')
    lambda_angles = _LambdaParameter('lambda_angles')
    lambda_torsions = _LambdaParameter('lambda_torsions')

    def set_alchemical_parameters(self, new_value):
        """Set all defined lambda parameters to the given value (alchemy.py:255-269)."""
        for name, v in self._parameters.items():
            if v is not None:
                setattr(self, name, new_value)


_AR_FIELDS = ['alchemical_atoms', 'alchemical_bonds', 'alchemical_angles', 'alchemical_torsions',
              'annihilate_electrostatics', 'annihilate_sterics', 'softcore_alpha', 'softcore_a', 'softcore_b',
              'softcore_c', 'softcore_beta', 'softcore_d', 'softcore_e', 'softcore_f', 'name']
AlchemicalRegion = collections.namedtuple('AlchemicalRegion', _AR_FIELDS)
# defaults as alchemy.py:417-427
AlchemicalRegion.__new__.__defaults__ = (None, None, None, None, True, False, 0.5, 1, 1, 6, 0.0, 1, 1, 2, None)
_SOFTCORE_FIELDS = ('softcore_alpha', 'softcore_a', 'softcore_b', 'softcore_c', 'softcore_beta', 'softcore_d',
                    'softcore_e', 'softcore_f')


class AbsoluteAlchemicalFactory:
    """Factory of alchemically modified systems (alchemy.py:430-754): the LJ fluid's sterics, small molecules' sterics,
    electrostatics and OBC terms."""

    def __init__(self, consistent_exceptions=False, switch_width=1.0 * unit.angstroms,
                 alchemical_pme_treatment='exact', alchemical_rf_treatment='switched',
                 disable_alchemical_dispersion_correction=False, split_alchemical_forces=True):
        self.consistent_exceptions = consistent_exceptions
        self.switch_width = switch_width
        self.alchemical_pme_treatment = alchemical_pme_treatment
        self.alchemical_rf_treatment = alchemical_rf_treatment
        self.disable_alchemical_dispersion_correction = disable_alchemical_dispersion_correction
        self.split_alchemical_forces = split_alchemical_forces

    def create_alchemical_system(self, reference_system, alchemical_regions, alchemical_regions_interactions=frozenset()):
        if alchemical_regions_interactions != frozenset():       # alchemy.py:661-662
            raise NotImplementedError('Interactions between alchemical regions is untested')
        if not isinstance(reference_system, System) or reference_system.kind not in (LJ, MOLECULE):
            raise NotImplementedError('only the Lennard-Jones fluid and small molecules can be alchemically modified on this path')
        if isinstance(alchemical_regions, AlchemicalRegion):
            alchemical_regions = [alchemical_regions]
        if reference_system.kind == MOLECULE:
            return self._alchemically_modify_molecule(reference_system, list(alchemical_regions))
        regions = list(alchemical_regions)
        if len(regions) == 0:
            raise ValueError('alchemical_atoms must be specified')
        if len(regions) > 2:
            raise NotImplementedError('more than two alchemical regions are not provided')
        n = reference_system.n_particles
        region_atoms = []
        for region in regions:
            if region.alchemical_atoms is None or len(list(region.alchemical_atoms)) == 0:
                raise ValueError('alchemical_atoms must be specified')     # alchemy.py:835
            atoms = sorted(set(int(a) for a in region.alchemical_atoms))
            if atoms[0] < 0 or atoms[-1] >= n:
                raise ValueError('alchemical atom index out of range')
            if any(x for x in (region.alchemical_bonds, region.alchemical_angles, region.alchemical_torsions)
                   if x not in (None, False, [], ())):
                raise NotImplementedError('bonded alchemical terms are outside the hot path (the LJ fluid has none)')
            region_atoms.append(atoms)
        if len(regions) == 2:
            if set(region_atoms[0]) & set(region_atoms[1]):                 # alchemy.py:674-689
                raise ValueError('Two regions have duplicate atoms.')
            if regions[0].name == regions[1].name:                          # alchemy.py:691-694
                raise ValueError('Two alchemical regions have the same name')
            if any(getattr(regions[0], f) != getattr(regions[1], f) for f in _SOFTCORE_FIELDS):
                raise NotImplementedError('the alchemical regions must share their soft-core constants (one value per '
                                          'global parameter name, alchemy.py:2009-2017)')
        region = regions[0]
        if reference_system.is_alchemical:
            raise ValueError('the system is already alchemically modified')
        system = reference_system.copy()
        system.alchemical_atoms = tuple(sorted(a for atoms in region_atoms for a in atoms))
        system.annihilate_sterics = bool(region.annihilate_sterics)
        if len(regions) == 2:
            system.alchemical_regions = tuple((r.name, tuple(atoms), bool(r.annihilate_sterics))
                                              for r, atoms in zip(regions, region_atoms))
        system.softcore_alpha = float(region.softcore_alpha)
        system.softcore_a = float(region.softcore_a)
        system.softcore_b = float(region.softcore_b)
        system.softcore_c = float(region.softcore_c)
        # alchemy.py:1787-1790
        system.alchemical_dispersion_correction = (not self.disable_alchemical_dispersion_correction) and \
            reference_system.use_dispersion_correction
        # lambda_electrostatics is defined by the factory even for zero charges (the electrostatic forces exist but
        # are identically zero), so AlchemicalState.from_system finds both parameters
        system.global_parameters = dict(reference_system.global_parameters)
        for r in regions:
            suffix = '' if r.name is None else '_' + r.name                  # alchemy.py:1695-1700
            system.global_parameters['lambda_sterics' + suffix] = 1.0
            system.global_parameters['lambda_electrostatics' + suffix] = 1.0
        return system

    # the literals of the reference's alchemical OBC2 expression (alchemy.py:2184-2203): offset, probe radius and the
    # surface-area energy whose 4 pi multiple is its 28.3919551
    _OBC2_LITERALS = (0.009, 0.14, 28.3919551 / (4.0 * np.pi))

    def _alchemically_modify_molecule(self, reference_system, regions):
        if len(regions) == 0:
            raise ValueError('alchemical_atoms must be specified')
        if len(regions) > 1:      # both GB paths refuse them (alchemy.py:2167-2168, 2258-2259); vacuum follows suit
            raise NotImplementedError('a molecule takes one alchemical region')
        region = regions[0]
        if region.alchemical_atoms is None or len(list(region.alchemical_atoms)) == 0:
            raise ValueError('alchemical_atoms must be specified')
        atoms = sorted(set(int(a) for a in region.alchemical_atoms))
        if atoms[0] < 0 or atoms[-1] >= reference_system.n_particles:
            raise ValueError('alchemical atom index out of range')
        if any(x not in (None, False, [], ()) for x in (region.alchemical_bonds, region.alchemical_angles, region.alchemical_torsions)):
            raise NotImplementedError('alchemical bonds, angles and torsions are not provided for molecules')
        if (region.softcore_beta, region.softcore_d, region.softcore_e, region.softcore_f) != (0.0, 1, 1, 2):
            raise NotImplementedError('soft-core electrostatics (softcore_beta/d/e/f other than 0, 1, 1, 2) are not provided')
        if self.consistent_exceptions:
            raise NotImplementedError('consistent_exceptions is not provided for molecules')
        if reference_system.is_alchemical:
            raise ValueError('the system is already alchemically modified')
        gb = reference_system.gb_parameters
        obc2 = gb is not None and tuple(gb[:3]) == OBC_MODELS['OBC2']
        if obc2 and not np.allclose((gb[3], gb[7], gb[6]), self._OBC2_LITERALS, rtol=1e-9, atol=0.0):
            raise NotImplementedError('the alchemical OBC2 expression has offset 0.009 nm, probe radius 0.14 nm and '
                                      'surface-area energy 2.25936 kJ/mol/nm^2 built in; this system has %r' % (tuple(gb),))
        system = reference_system.copy()
        system.alchemical_atoms = tuple(atoms)
        system.annihilate_sterics = bool(region.annihilate_sterics)
        system.annihilate_electrostatics = bool(region.annihilate_electrostatics)
        system.softcore_alpha = float(region.softcore_alpha)
        system.softcore_a = float(region.softcore_a)
        system.softcore_b = float(region.softcore_b)
        system.softcore_c = float(region.softcore_c)
        system.alchemical_obc2 = obc2
        system.global_parameters = dict(reference_system.global_parameters)
        system.global_parameters['lambda_sterics'] = 1.0
        system.global_parameters['lambda_electrostatics'] = 1.0
        return system

    @staticmethod
    def get_energy_components(alchemical_system, alchemical_state, positions, platform=None):
        raise NotImplementedError('per-force energy dissection needs OpenMM; see tests/ for the component checks')
