"""ctypes wrapper over oracle/liborc_npt.so (rx_oracle_npt.c): the alchemical LJ fluid at constant pressure.

TEST INFRASTRUCTURE ONLY, like oracle.py: imported by tests/.  The product package (openmmtools_b200/) must never import
this module.
"""
import ctypes as C
import os
import subprocess
import numpy as np
from . import oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(_HERE, 'liborc_npt.so')
# (the flags of oracle/Makefile)
_CFLAGS = ['-O2', '-fPIC', '-fopenmp', '-fno-fast-math', '-ffp-contract=off', '-fvisibility=hidden', '-Wall', '-Wno-unused-result']


def build(force=False):
    newest = max(os.path.getmtime(os.path.join(_HERE, f)) for f in ('rx_oracle_npt.c', 'rx_oracle.c'))
    if force or not os.path.exists(_LIB) or os.path.getmtime(_LIB) < newest:
        subprocess.check_call(['/usr/bin/gcc'] + _CFLAGS + ['-shared', '-o', _LIB, os.path.join(_HERE, 'rx_oracle_npt.c'), '-lm'])
    return _LIB


class Barostat(C.Structure):
    _fields_ = [('volume_scale', C.c_double), ('step', C.c_int32), ('n_attempted', C.c_int32), ('n_accepted', C.c_int32),
                ('reserved', C.c_int32)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_LIB)
        _lib.orc_npt_barostat_step.restype = C.c_int
        _lib.orc_npt_barostat_step.argtypes = [C.c_void_p] * 4 + [C.c_double] * 5 + [C.c_void_p] * 3 + [C.c_double] * 2 + [C.c_void_p]
        _lib.orc_npt_langevin.restype = C.c_int
        _lib.orc_npt_energy_matrix.restype = None
    return _lib


_p = oracle._p


def energy_matrix(osys, x, boxes, lambdas, betas, pressure, dispersion, offsets=None):
    """u[k][l] = beta_l (U_l(x_k; box_k) + offset_l + dispersion_l / V_k + pressure_l V_k), f64."""
    x = np.ascontiguousarray(x, np.float64); boxes = np.ascontiguousarray(boxes, np.float64)
    arrs = [np.ascontiguousarray(a, np.float64) for a in (lambdas, betas, pressure, dispersion)]
    off = None if offsets is None else np.ascontiguousarray(offsets, np.float64)
    u = np.zeros((x.shape[0], len(arrs[0])))
    lib().orc_npt_energy_matrix(C.byref(osys.p), _p(osys.sigma), _p(osys.eps), _p(osys.alch), C.c_int(x.shape[0]), _p(x), _p(boxes),
                                C.c_int(len(arrs[0])), *[_p(a) for a in arrs[:2]], None if off is None else _p(off),
                                _p(arrs[2]), _p(arrs[3]), _p(u))
    return u


def barostat_state(volume_scale, step=0, n_attempted=0, n_accepted=0):
    return Barostat(float(volume_scale), int(step), int(n_attempted), int(n_accepted), 0)


def barostat_step(osys, x, box, st, u1, u2, lam, kT, pressure, dispersion, min_edge):
    """One attempt; x (N, 3) and box (3,) float64 arrays and st (Barostat) are updated in place.
    Returns (1 accepted | 0 rejected | -1 refused, w or None)."""
    w = C.c_double(np.nan)
    r = lib().orc_npt_barostat_step(C.byref(osys.p), _p(osys.sigma), _p(osys.eps), _p(osys.alch), lam, kT, pressure,
                                    dispersion, min_edge, _p(x), _p(box), C.byref(st), u1, u2, C.byref(w))
    return r, (None if r < 0 else w.value)


def langevin(osys, x, v, noise, box, st, uniforms, lam, kT, dt, gamma, n_steps, pressure, dispersion, min_edge,
             program='VRORV'):
    """n_steps steps with the barostat every 25 (in place on x, v, box, st).  Returns (decisions, potential incl. c / V)."""
    d = oracle.DynParams(0, n_steps, dt, gamma, kT, lam, 0.0, (C.c_double * 3)(0, 0, 0), 0.0)
    uniforms = np.ascontiguousarray(uniforms, np.float64)
    n_max = len(uniforms) // 2
    dec = np.zeros(max(n_max, 1), np.int32)
    U = C.c_double()
    noise = np.ascontiguousarray(noise, np.float64)
    n = lib().orc_npt_langevin(C.byref(osys.p), C.byref(d), program.replace(' ', '').encode(), _p(osys.sigma), _p(osys.eps),
                               _p(osys.alch), _p(osys.mass), _p(x), _p(v), _p(noise), _p(box), C.byref(st),
                               C.c_double(pressure), C.c_double(dispersion), C.c_double(min_edge), _p(uniforms),
                               C.c_int(n_max), _p(dec), C.byref(U))
    assert n >= 0, n
    return dec[:n].tolist(), U.value
