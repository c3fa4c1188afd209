"""Host restatement in float64 of the molecule kernels' Langevin program (k_propagate_mol, rx_molecule.cuh), on any force
function: the entry RATTLE of the incoming velocities, the centre-of-mass velocity removed at the start of every step
(remove_cm), then the splitting's V, R and O operations, each followed by the constraint steps (SHAKE / RATTLE sweeps as
oracle/rx_oracle_mol.c solves them), with the noise of helpers.device_noise.  The C oracles' `langevin` takes their own
unmodified force field only; this one takes an energy_forces(x) -> (U, F) callable (an alchemical molecule at one state),
and tests/test_mol_langevin_oracle_host.py holds it to the C oracles where both apply."""
import numpy as np


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]   # (the C oracle's order of additions)


def shake(cons, mass, x0, x, tol):
    """Positions x moved onto the constraints (i, j, d), displacements along the bond vectors of x0 (Gauss-Seidel sweeps)."""
    x = x.copy()
    for _ in range(500):
        done = True
        for i, j, d in cons:
            r, r0 = x[i] - x[j], x0[i] - x0[j]
            d2 = d * d
            diff = d2 - _dot(r, r)
            if abs(diff) > tol * d2:
                done = False
                wi, wj = 1.0 / mass[i], 1.0 / mass[j]
                g = diff / (2.0 * (wi + wj) * _dot(r, r0))
                x[i] += g * wi * r0; x[j] -= g * wj * r0
        if done:
            break
    return x


def rattle(cons, mass, x, v, tol):
    """Velocities v with their components along the constraints removed (Gauss-Seidel sweeps)."""
    v = v.copy()
    for _ in range(500):
        done = True
        for i, j, _ in cons:
            r, dv = x[i] - x[j], v[i] - v[j]
            rv, r2 = _dot(r, dv), _dot(r, r)
            if abs(rv) > tol * r2:
                done = False
                wi, wj = 1.0 / mass[i], 1.0 / mass[j]
                g = rv / ((wi + wj) * r2)
                v[i] -= g * wi * r; v[j] += g * wj * r
        if done:
            break
    return v


def run(x, v, mass, kT, energy_forces, noise, dt, gamma, n_steps, program, cons=None, remove_cm=False, tol=1e-10):
    """n_steps of the splitting `program` (V, R, O; spaces ignored) from positions x and velocities v with standard normals
    noise [n_steps * nO, N, 3]; energy_forces(x) -> (U, F).  cons: constraints (i, j, d) or None.  Returns (x, v, U at the
    final positions)."""
    prog = program.replace(' ', '')
    mass = np.asarray(mass, np.float64)
    m = mass[:, None]
    cons = [(int(i), int(j), float(d)) for i, j, d in (cons if cons is not None else [])]
    x, v = np.array(x, np.float64), np.array(v, np.float64)
    nV, nR, nO = prog.count('V'), prog.count('R'), prog.count('O')
    hO = dt / (nO if nO else 1)
    a, b = np.exp(-gamma * hO), np.sqrt(1.0 - np.exp(-2.0 * gamma * hO))
    sg = np.sqrt(kT / m)
    if cons:   # incoming velocities obey the constraints
        v = rattle(cons, mass, x, v, tol)
    f, oc = None, 0
    for _ in range(n_steps):
        if remove_cm:
            v = v - (m * v).sum(0) / mass.sum()
        for op in prog:
            if op == 'V':
                if f is None:
                    f = energy_forces(x)[1]
                v = v + (dt / nV) * f / m
            elif op == 'R':
                h = dt / nR
                x0 = x
                x = x + h * v
                if cons:
                    xu = x
                    x = shake(cons, mass, x0, x, tol)
                    v = v + (x - xu) / h
                f = None
            else:
                v = a * v + b * sg * noise[oc]
                oc += 1
            if cons:
                v = rattle(cons, mass, x, v, tol)
    return x, v, energy_forces(x)[0]
