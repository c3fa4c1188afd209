"""Shared by the implicit-solvent tests: OBC parameters for the test molecules of helpers.py, the T4-lysozyme L99A ligand
of tests/golden (AMBER 9 sander single points at igb=2), and a numpy restatement of the OBC + ACE energy."""
import os
import re
import numpy as np
from openmmtools_b200 import amber, testsystems, unit
from openmmtools_b200.system import System, MOLECULE

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
# sander's Coulomb constant (charges stored x 18.2223) against the 138.935456 kJ nm/mol/e^2 of this project, in kcal A/mol/e^2
SANDER_ELEC_SCALE = 138.935456 / 4.184 * 10.0 / 18.2223 ** 2
# mbondi2-like radius (nm) and OBC screening factor by element, for the molecules of helpers.py (told apart by mass)
_ELEMENT_GB = [(1.1, 0.12, 0.85), (12.5, 0.17, 0.72), (14.5, 0.155, 0.79), (16.5, 0.15, 0.85), (24.0, 0.17, 0.8), (1e9, 0.175, 0.8)]


def obc(system, model='OBC1', ace=True):
    """A copy of `system` in OBC implicit solvent, radii and screening factors assigned by element."""
    s = system.copy()
    s.gb_radius = np.array([next(r for m, r, _ in _ELEMENT_GB if mass < m) for mass in s.masses])
    s.gb_scale = np.array([next(c for m, _, c in _ELEMENT_GB if mass < m) for mass in s.masses])
    s.gb_parameters = amber.obc_parameters(model, gbsaModel='ACE' if ace else None)
    return s


def with_model(system, model='OBC1', ace=True):
    """A copy of an implicit-solvent system with another OBC model / without the ACE term."""
    s = system.copy()
    s.gb_parameters = amber.obc_parameters(model, gbsaModel='ACE' if ace else None)
    return s


def implicit_system(name, constraints='HBonds'):
    t = {'alanine-dipeptide': lambda: testsystems.AlanineDipeptideImplicit(constraints=constraints),
         'toluene': lambda: testsystems.TolueneImplicit(constraints=constraints)}[name]()
    return t.system, np.ascontiguousarray(t.positions.value_in_unit(unit.nanometer), np.float64)


def ligand(constraints=None, coordinates='ligand.crd'):
    """The T4-lysozyme L99A ligand (18 atoms, GAFF, mbondi2) as createSystem(implicitSolvent=OBC1, gbsaModel=None) builds it."""
    d = amber.read_prmtop(os.path.join(GOLDEN, 't4-ligand.prmtop'))
    s = System(MOLECULE, d['mass'])
    s.charge, s.sigma, s.epsilon = d['charge'], d['sigma'], d['epsilon']
    hb = constraints == 'HBonds'
    s.bonds = np.array([b[:4] for b in d['bonds'] if not (hb and b[4])], np.float64).reshape(-1, 4)
    s.constraints = np.array([[b[0], b[1], b[3]] for b in d['bonds'] if hb and b[4]], np.float64).reshape(-1, 3)
    s.angles = np.array(d['angles'], np.float64).reshape(-1, 5)
    s.torsions = np.array(d['torsions'], np.float64).reshape(-1, 7)
    s.exclusions = np.array(d['exclusions'], np.int64).reshape(-1, 2)
    s.exceptions = np.array(d['exceptions'], np.float64).reshape(-1, 5)
    s.remove_cm_motion = True
    s.gb_radius, s.gb_scale = d['radii'], d['screen']
    s.gb_parameters = amber.obc_parameters('OBC1', gbsaModel=None)
    return s, amber.read_inpcrd(os.path.join(GOLDEN, 't4-' + coordinates))


def sander_energies(path):
    """The first energy record of a sander output: {name: kcal/mol}."""
    text = open(path).read()
    block = text[text.index('NSTEP'):]
    block = block[:block.index('\n\n\n')]
    return {k.strip(): float(v) for k, v in re.findall(r'([A-Za-z0-9\- ]+?)\s*=\s*(-?\d+\.\d+)', block)}


def numpy_gb_energy(system, x):
    """The OBC + ACE energy (kJ/mol), vectorised over all ordered pairs: an independent restatement of the model."""
    al, be, ga, off, e_in, e_out, sa, probe = system.gb_parameters
    rho = np.asarray(system.gb_radius, float)
    rt = rho - off
    sr = np.asarray(system.gb_scale, float) * rt
    q = np.asarray(system.charge, float)
    n = len(rho)
    r = np.linalg.norm(x[:, None, :] - x[None, :, :], axis=-1)
    off_diag = ~np.eye(n, dtype=bool)
    rr = np.where(off_diag, r, 1.0)
    U = rr + sr[None, :]
    L = np.maximum(rt[:, None], np.abs(rr - sr[None, :]))
    I = 0.5 * (1 / L - 1 / U + 0.25 * (rr - sr[None, :] ** 2 / rr) * (1 / U ** 2 - 1 / L ** 2) + 0.5 * np.log(L / U) / rr)
    I = np.where(off_diag & (rr + sr[None, :] > rt[:, None]), I, 0.0).sum(axis=1)
    psi = I * rt
    B = 1.0 / (1.0 / rt - np.tanh(al * psi - be * psi ** 2 + ga * psi ** 3) / rho)
    P = -138.935456 * (1.0 / e_in - 1.0 / e_out)
    BB = B[:, None] * B[None, :]
    f = np.sqrt(r ** 2 + BB * np.exp(-r ** 2 / (4.0 * BB)))
    iu = np.triu_indices(n, 1)
    E = 0.5 * P * np.sum(q ** 2 / B) + P * np.sum((q[:, None] * q[None, :] / f)[iu])
    return E + np.sum(4.0 * np.pi * sa * (rho + probe) ** 2 * (rho / B) ** 6)
