#!/usr/bin/env python
"""Golden vectors for hybrid Monte Carlo from the REAL reference code (build container only).

``openmmtools/integrators.py`` is executed unmodified against the recording stand-in for ``openmm.CustomIntegrator`` of
make_integrator_golden.py: ``HMCIntegrator(temperature, nsteps, timestep)`` yields its own step program (the
``addComputePerDof`` / ``addComputeGlobal`` / ``addComputeSum`` strings and the constrain / update-context markers) and
its global variables.  The program is interpreted in float64 under CustomIntegrator's documented semantics (``f`` and
``energy`` at the current positions, ``gaussian`` a fresh standard normal per degree of freedom, ``uniform`` a fresh
uniform per evaluation, ``step(x)`` = 1 for x >= 0, if-blocks on globals) with injected Gaussians and uniforms, and
forces from the oracle's LJ model, the harmonic oscillator or the oracle's alanine dipeptide (HBonds constraints:
``addConstrainPositions`` / ``addConstrainVelocities`` are SHAKE along the bond vectors of the positions of the previous
constraint step and RATTLE, as tests/hmc_oracle.py and oracle/rx_oracle_mol.c solve them, to 1e-10).  As
``HMCMove.apply`` does, a case takes ``nsteps`` integrator steps (trials).

Output: tests/golden/hmc_golden.npz -- per case the program text, the initial globals, the inputs and, per trial, the
positions, velocities, Eold, Enew and accept.
"""
import os, re, sys
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests')); sys.path.insert(0, HERE)
from openmmtools_b200 import unit as u
from helpers import lj_setup, oracle_system, KB
import hmc_oracle

CASES = [  # system, nsteps (steps per trial = trials per apply), dt (ps), T (K), lambda (LJ)
    ('lj', 2, 0.002, 300.0, 1.0),
    ('lj', 3, 0.015, 300.0, 0.5),
    ('lj', 5, 0.001, 350.0, 0.2),
    ('harmonic', 4, 0.6, 300.0, None),
    ('harmonic', 3, 0.9, 250.0, None),
    ('aladip', 3, 0.002, 300.0, None),
    ('aladip', 2, 0.004, 300.0, None),
]
TOL = 1e-10
HO_K = 90.0   # kJ/mol/nm^2 (the mass 39.948 Da gives a period of about 4.2 ps)


def case_inputs(idx):
    """(x0 [N,3], mass [N], energy_forces(x) -> (U, F), gaussians [trials, N, 3], uniforms [trials], constraints or
    None) of case idx."""
    kind, nsteps, dt, T, lam = CASES[idx]
    rng = np.random.default_rng(700 + idx)
    if kind == 'lj':
        s = lj_setup(N=48, n_alch=5, seed=200 + idx)
        osys = oracle_system(s)
        x, mass = s['x'].copy(), s['mass'].copy()

        def ef(y):
            U, _, f = osys.energy(y, lam, forces=True)
            return U, f
    elif kind == 'aladip':
        from openmmtools_b200 import testsystems
        from oracle import oracle
        a = testsystems.AlanineDipeptideVacuum(constraints='HBonds')
        x = np.ascontiguousarray(a.positions.value_in_unit(u.nanometer), np.float64)
        mol = oracle.Molecule(a.system)
        mass = mol.mass.copy()
        ef = hmc_oracle.molecule(mol)
        gauss = rng.normal(size=(nsteps, len(mass), 3))
        return x, mass, ef, gauss, rng.uniform(size=nsteps), mol.cons.copy()
    else:
        N = 8
        x0 = np.array([0.1, -0.2, 0.3])
        x, mass = x0 + rng.normal(scale=0.05, size=(N, 3)), np.full(N, 39.948)

        def ef(y):
            d = y - x0
            return 0.5 * HO_K * np.sum(d * d), -HO_K * d
    gauss = rng.normal(size=(nsteps, len(mass), 3))
    unif = rng.uniform(size=nsteps)
    return x, mass, ef, gauss, unif, None


def evaluate(expr, names):
    """One Lepton expression of the HMC program: + - * / ^, sqrt, exp, step and names."""
    fns = {'sqrt': np.sqrt, 'exp': np.exp, 'step': lambda a: np.where(np.asarray(a) >= 0.0, 1.0, 0.0)}
    with np.errstate(over='ignore', invalid='ignore'):
        return eval(expr.replace('^', '**'), {'__builtins__': {}, **fns}, names)


def interpret(program, globals0, dt, x, mass, energy_forces, gauss, unif, n_calls, cons=None):
    """Run the recorded program n_calls times.  program: ('perdof'|'global'|'sum', var, expr), ('if', cond), ('end',),
    ('constrain_x',), ('constrain_v',), ('update_context',); cons: constraints (i, j, d) or None.  Returns per call
    (x, v, Eold, Enew, accept)."""
    g = dict(globals0)
    per, v = {}, np.zeros_like(x)
    m = np.asarray(mass, np.float64)[:, None]
    cache = {}
    x_ref = x   # the positions of the previous constraint step: SHAKE's bond vectors
    ig = iu = 0
    out = []

    def names():
        d = dict(g); d.update(per); d.update(x=x, v=v, m=m, dt=dt)
        return d

    class Lazy(dict):
        def __missing__(self, key):
            if key in ('f', 'energy'):
                if 'U' not in cache:
                    cache['U'], cache['f'] = energy_forces(x)
                return cache['U'] if key == 'energy' else cache['f']
            raise KeyError(key)

    for _ in range(n_calls):
        skip = 0
        for ins in program:
            if ins[0] == 'end':
                skip = max(0, skip - 1); continue
            if ins[0] == 'if':
                lhs, rhs = [s.strip() for s in ins[1].split('=')]
                if skip or not (g[lhs] == float(rhs)):
                    skip += 1
                continue
            if skip or ins[0] == 'update_context':
                continue
            if ins[0] in ('constrain_x', 'constrain_v'):
                if cons is not None and len(cons):
                    if ins[0] == 'constrain_x':
                        x = hmc_oracle.shake(cons, mass, x_ref, x, TOL); cache.clear()
                    else:
                        v = hmc_oracle.rattle(cons, mass, x, v, TOL)
                x_ref = x
                continue
            d = Lazy(names())
            expr = ins[2]
            if re.search(r'\bgaussian\b', expr):
                d['gaussian'] = gauss[ig]; ig += 1
            if re.search(r'\buniform\b', expr):
                d['uniform'] = unif[iu]; iu += 1
            val = evaluate(expr, d)
            if ins[0] == 'perdof':
                val = np.array(val, np.float64) + np.zeros_like(x)
                if ins[1] == 'x':
                    x = val; cache.clear()
                elif ins[1] == 'v':
                    v = val
                else:
                    per[ins[1]] = val
            elif ins[0] == 'sum':
                g[ins[1]] = float(np.sum(np.array(val, np.float64) + np.zeros_like(x)))
            elif ins[0] == 'global':
                g[ins[1]] = float(val)
            else:
                raise NotImplementedError(ins)
        out.append((x.copy(), v.copy(), g['Eold'], g['Enew'], g['accept']))
    assert ig == len(gauss) and iu == len(unif)
    return out, g


def program_text(program):
    return np.array(['|'.join(map(str, p)) for p in program])


def program_from_text(text):
    return [tuple(str(t).split('|')) for t in text]


if __name__ == '__main__':
    from make_integrator_golden import load_reference_integrators
    mod = load_reference_integrators()
    out = {}
    for idx, (kind, nsteps, dt, T, lam) in enumerate(CASES):
        integ = mod.HMCIntegrator(temperature=T * u.kelvin, nsteps=nsteps, timestep=dt * u.picoseconds)
        x, mass, ef, gauss, unif, cons = case_inputs(idx)
        res, g = interpret(integ.program, integ.globals, integ.dt, x, mass, ef, gauss, unif, nsteps, cons)
        out['case%d_program' % idx] = program_text(integ.program)
        out['case%d_global_names' % idx] = np.array(list(integ.globals))
        out['case%d_global_values' % idx] = np.array([integ.globals[k] for k in integ.globals])
        out['case%d_dt' % idx] = np.array(integ.dt)
        out['case%d_x' % idx] = np.stack([r[0] for r in res])
        out['case%d_v' % idx] = np.stack([r[1] for r in res])
        out['case%d_E' % idx] = np.array([[r[2], r[3], r[4]] for r in res])
        out['case%d_counts' % idx] = np.array([g['naccept'], g['ntrials']])
        print(kind, nsteps, 'accepted', [r[4] for r in res])
    dst = os.path.join(HERE, 'hmc_golden.npz')
    np.savez_compressed(dst, **out)
    print('wrote', dst, os.path.getsize(dst))
    print(out['case0_program'])
