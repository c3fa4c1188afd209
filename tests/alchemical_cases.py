"""Alchemical molecules beyond toluene and alanine dipeptide, built from the test molecules of test_gpu_molecule.MOLECULES
and implicit_helpers.obc: 32 atoms with the region on the top bit of the mask, a fully alchemical molecule, the general
constraint path (sweeps, Newton M-SHAKE), a region with no lambda-controlled pair, a ligand among solvent molecules, non-default
soft-core sterics (the c != 6 branch), a single atom, and a molecule whose OBC2 pairs are engulfed.  Shared by the host tests
of the oracle and the device tests of tests/test_gpu_alchemical_molecule_variants.py."""
import numpy as np
from implicit_helpers import obc
from test_gpu_molecule import MOLECULES
from openmmtools_b200.alchemy import AbsoluteAlchemicalFactory, AlchemicalRegion


def _water_of(system):
    """The three atoms of the rigid water holding the first constraint."""
    c = np.asarray(system.constraints)
    i, j = int(c[0, 0]), int(c[0, 1])
    atoms = {i, j}
    for a, b, _ in c:
        if int(a) in atoms or int(b) in atoms:
            atoms |= {int(a), int(b)}
    return sorted(atoms)


def _ion_of(system):
    return [int(np.argmax(np.asarray(system.masses) == 22.99))]


def engulfed_methane(model='OBC2'):
    """Methane in OBC with a carbon of radius 0.3 nm and screening factor 1: its scaled radius (0.291 nm) reaches past each
    hydrogen (0.109 nm away) by more than the hydrogen's offset radius (0.111 nm), so the four (H, C) pairs are engulfed
    (sr_C - r > rt_H) and the alchemical OBC2 expression's term C is on for them.  The boundary is at r = 0.18 nm."""
    s, x = MOLECULES['methane']()
    s = obc(s, model)
    s.gb_radius = np.array(s.gb_radius, float); s.gb_scale = np.array(s.gb_scale, float)
    s.gb_radius[0], s.gb_scale[0] = 0.3, 1.0
    return s, x


def _base(name):
    """(system, positions) of a base molecule: 'name' or 'name/OBC1', 'name/OBC2'."""
    mol, _, model = name.partition('/')
    if mol == 'engulfed-methane':
        return engulfed_methane(model or 'OBC2')
    s, x = MOLECULES[mol]()
    return (obc(s, model) if model else s), x


# name: (base, region of the base system (a list, or a function of it), factory keywords).  'annihilate' marks the cases
# whose region holds pairs of two alchemical atoms, where the swapped flags (True, False) select other lambdas.
CASES = {
    'decane-obc2-top': ('decane/OBC2', list(range(16, 32)), {}),                          # 32 atoms, bit 31, star path
    'decane-all-annihilated': ('decane', list(range(32)), dict(annihilate_sterics=True, annihilate_electrostatics=True)),
    'propane-allbonds-obc1-half': ('propane-AllBonds-shuffled/OBC1', list(range(0, 11, 2)), {}),   # sweeps
    'mixture-obc2-half': ('mixture-shuffled/OBC2', list(range(1, 14, 2)), {}),                     # Newton M-SHAKE
    'methane-obc1-carbon': ('methane/OBC1', [0], {}),                                     # n_tap = 0
    'waters-ion-obc2-ion': ('waters-ion-shuffled/OBC2', _ion_of, {}),
    'waters-ion-obc2-water': ('waters-ion-shuffled/OBC2', _water_of, {}),
    'torsion-probe-sc-c4': ('torsion-probe', [0], dict(softcore_alpha=0.3, softcore_a=2, softcore_b=2, softcore_c=4)),
    'torsion-probe-sc-c12': ('torsion-probe', [0, 4], dict(softcore_alpha=0.3, softcore_a=2, softcore_b=2, softcore_c=12)),
    'ion-obc1': ('ion/OBC1', [0], {}),                                                    # n = 1
    'engulfed-methane-obc2': ('engulfed-methane/OBC2', [0], {}),
}
SWAPPED = ('decane-obc2-top', 'propane-allbonds-obc1-half', 'mixture-obc2-half', 'torsion-probe-sc-c12')


def make(name, swapped=False):
    """(base system, positions, alchemical system) of case `name`; swapped: annihilate_sterics=True,
    annihilate_electrostatics=False."""
    base, region, kw = CASES[name]
    s, x = _base(base)
    atoms = region(s) if callable(region) else region
    kw = dict(kw)
    if swapped:
        kw.update(annihilate_sterics=True, annihilate_electrostatics=False)
    asys = AbsoluteAlchemicalFactory().create_alchemical_system(s, AlchemicalRegion(alchemical_atoms=atoms, **kw))
    return s, np.ascontiguousarray(x, np.float64), asys


def variants():
    """(name, swapped) of every case and flag setting."""
    return [(n, False) for n in CASES] + [(n, True) for n in SWAPPED]
