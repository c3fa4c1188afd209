"""ctypes wrapper over oracle/liborc_gb.so (rx_oracle_gb.c): a small molecule in OBC implicit solvent.

TEST INFRASTRUCTURE ONLY, like oracle.py: imported by tests/ and tools/.  The product package (openmmtools_b200/) must
never import this module.
"""
import ctypes as C
import os
import subprocess
import numpy as np
from . import oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(_HERE, 'liborc_gb.so')
# (the flags of oracle/Makefile)
_CFLAGS = ['-O2', '-fPIC', '-fopenmp', '-fno-fast-math', '-ffp-contract=off', '-fvisibility=hidden', '-Wall', '-Wno-unused-result']


def build(force=False):
    newest = max(os.path.getmtime(os.path.join(_HERE, f)) for f in ('rx_oracle_gb.c', 'rx_oracle_mol.c'))
    if force or not os.path.exists(_LIB) or os.path.getmtime(_LIB) < newest:
        subprocess.check_call(['/usr/bin/gcc'] + _CFLAGS + ['-shared', '-o', _LIB, os.path.join(_HERE, 'rx_oracle_gb.c'), '-lm'])
    return _LIB


class _OrcGB(C.Structure):
    _fields_ = [('radius', C.c_void_p), ('scale', C.c_void_p), ('alpha', C.c_double), ('beta', C.c_double), ('gamma', C.c_double),
                ('offset', C.c_double), ('solute_dielectric', C.c_double), ('solvent_dielectric', C.c_double),
                ('sa_energy', C.c_double), ('probe_radius', C.c_double)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_LIB)
        for name in ('orc_gb_energy', 'orc_gb_mol_energy', 'orc_gb_langevin'):
            getattr(_lib, name).restype = C.c_double
    return _lib


_p = oracle._p


class Molecule(oracle.Molecule):
    """A small molecule in OBC implicit solvent: `system` is an openmmtools_b200.system.System of kind 'molecule' with GB
    radii (system.gb_radius, gb_scale, gb_parameters).  energy / langevin include the OBC energy and forces; kinetic and the
    constraint arrays are oracle.Molecule's."""

    def __init__(self, system):
        oracle.Molecule.__init__(self, system)
        if getattr(system, 'gb_radius', None) is None:
            raise ValueError('the system has no GB radii: use oracle.Molecule for a molecule in vacuum')
        self.gb_radius = np.ascontiguousarray(system.gb_radius, np.float64)
        self.gb_scale = np.ascontiguousarray(system.gb_scale, np.float64)
        self.gb = _OrcGB(_p(self.gb_radius).value, _p(self.gb_scale).value, *system.gb_parameters)

    def energy(self, x, forces=False):
        x = np.ascontiguousarray(x, np.float64)
        f = np.zeros_like(x) if forces else None
        U = lib().orc_gb_mol_energy(C.byref(self.s), C.byref(self.gb), _p(x), _p(f) if forces else None)
        return (U, f) if forces else U

    def gb_energy(self, x, forces=False):
        """The OBC + ACE energy alone and, with forces=True, its forces."""
        x = np.ascontiguousarray(x, np.float64)
        f = np.zeros_like(x) if forces else None
        U = lib().orc_gb_energy(C.byref(self.s), C.byref(self.gb), _p(x), _p(f) if forces else None)
        return (U, f) if forces else U

    def born_radii(self, x):
        """(Born radii, number of engulfed pairs) at x."""
        B = np.zeros(self.N)
        e = lib().orc_gb_born_radii(C.byref(self.s), C.byref(self.gb), _p(np.ascontiguousarray(x, np.float64)), _p(B))
        return B, e

    def langevin(self, x, v, noise, kT, dt, gamma, n_steps, program='VRORV', tol=1e-10):
        """In-place constrained V/R/O splitting steps with injected noise [n_steps*nO, N, 3]; returns the final potential."""
        assert x.dtype == np.float64 and v.dtype == np.float64 and x.flags.c_contiguous and v.flags.c_contiguous
        noise = np.ascontiguousarray(noise, np.float64)
        return lib().orc_gb_langevin(C.byref(self.s), C.byref(self.gb), _p(x), _p(v), _p(noise), C.c_double(kT), C.c_double(dt),
                                     C.c_double(gamma), C.c_int(n_steps), program.replace(' ', '').encode(), C.c_double(tol))
