"""ctypes wrapper over oracle/liborc_npt_aniso.so (rx_oracle_npt_aniso.c): the anisotropic Monte Carlo barostat on the
alchemical LJ fluid, with the axis draws and uniforms as inputs.

TEST INFRASTRUCTURE ONLY, like npt.py: imported by tests/.  The product package (openmmtools_b200/) must never import this
module.
"""
import ctypes as C
import os
import subprocess
import numpy as np
from . import oracle
from .npt import _CFLAGS

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(_HERE, 'liborc_npt_aniso.so')


def build(force=False):
    newest = max(os.path.getmtime(os.path.join(_HERE, f)) for f in ('rx_oracle_npt_aniso.c', 'rx_oracle_npt.c', 'rx_oracle.c'))
    if force or not os.path.exists(_LIB) or os.path.getmtime(_LIB) < newest:
        subprocess.check_call(['/usr/bin/gcc'] + _CFLAGS + ['-shared', '-o', _LIB, os.path.join(_HERE, 'rx_oracle_npt_aniso.c'),
                                                            '-lm'])
    return _LIB


class AnisotropicBarostat(C.Structure):
    _fields_ = [('volume_scale', C.c_double * 3), ('n_attempted', C.c_int32 * 3), ('n_accepted', C.c_int32 * 3),
                ('step', C.c_int32), ('scale_mask', C.c_int32)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_LIB)
        _lib.orc_npt_aniso_barostat_step.restype = C.c_int
        _lib.orc_npt_aniso_barostat_step.argtypes = ([C.c_void_p] * 4 + [C.c_double] * 5 + [C.c_void_p] * 3 + [C.c_int] +
                                                     [C.c_double] * 2 + [C.c_void_p])
        _lib.orc_npt_aniso_langevin.restype = C.c_int
    return _lib


_p = oracle._p


def barostat_state(volume_scale, scale_mask=7, step=0):
    """Per-axis state; volume_scale is one number for every axis or three."""
    st = AnisotropicBarostat()
    st.volume_scale[:] = [float(v) for v in np.broadcast_to(np.asarray(volume_scale, np.float64), (3,))]
    st.step, st.scale_mask = int(step), int(scale_mask)
    return st


def barostat_step(osys, x, box, st, axis, u1, u2, lam, kT, pressure, dispersion, min_edge):
    """One attempt on `axis`; x (N, 3), box (3,) and st are updated in place.  Returns (1 | 0 | -1, w or None)."""
    w = C.c_double(np.nan)
    r = lib().orc_npt_aniso_barostat_step(C.byref(osys.p), _p(osys.sigma), _p(osys.eps), _p(osys.alch), lam, kT, pressure,
                                          dispersion, min_edge, _p(x), _p(box), C.byref(st), int(axis), u1, u2, C.byref(w))
    return r, (None if r < 0 else w.value)


def langevin(osys, x, v, noise, box, st, axes, uniforms, lam, kT, dt, gamma, n_steps, pressure, dispersion, min_edge,
             program='VRORV'):
    """n_steps steps with an attempt every 25 (in place on x, v, box, st): attempt i on axes[i] with uniforms[2 i],
    [2 i + 1].  Returns (decisions, potential incl. c / V)."""
    d = oracle.DynParams(0, n_steps, dt, gamma, kT, lam, 0.0, (C.c_double * 3)(0, 0, 0), 0.0)
    uniforms = np.ascontiguousarray(uniforms, np.float64)
    axes = np.ascontiguousarray(axes, np.int32)
    n_max = min(len(uniforms) // 2, len(axes))
    dec = np.zeros(max(n_max, 1), np.int32)
    U = C.c_double()
    noise = np.ascontiguousarray(noise, np.float64)
    n = lib().orc_npt_aniso_langevin(C.byref(osys.p), C.byref(d), program.replace(' ', '').encode(), _p(osys.sigma),
                                     _p(osys.eps), _p(osys.alch), _p(osys.mass), _p(x), _p(v), _p(noise), _p(box),
                                     C.byref(st), C.c_double(pressure), C.c_double(dispersion), C.c_double(min_edge),
                                     axes.ctypes.data_as(C.c_void_p), _p(uniforms), C.c_int(n_max), _p(dec), C.byref(U))
    assert n >= 0, n
    return dec[:n].tolist(), U.value
