"""Host restatement of the device's hybrid Monte Carlo (rx_set_hmc_integrator) in float64: HMCIntegrator's step program
(integrators.py:959-997) with the device's Philox draws, on any force/energy function, with the constraint steps (SHAKE /
RATTLE sweeps as oracle/rx_oracle_mol.c solves them) when the system has constraints."""
import numpy as np
from helpers import philox4x32_10, philox_normal3


def _key(seed, iteration):
    return (seed & 0xFFFFFFFF, ((seed >> 32) ^ (iteration >> 32)) & 0xFFFFFFFF)


def draws(seed, iteration, replica, N, n_trials):
    """(standard normals [n_trials, N, 3] of the velocity draws, uniforms [n_trials]) of replica `replica`: Philox counters
    (atom, 0x90000000 + trial, replica, iteration) and (trial, 0xB0000000, replica, iteration)."""
    key = _key(seed, iteration)
    ctr = np.zeros((n_trials, N, 4), np.uint32)
    ctr[..., 0] = np.arange(N)[None, :]
    ctr[..., 1] = (0x90000000 + np.arange(n_trials, dtype=np.uint64))[:, None].astype(np.uint32)
    ctr[..., 2] = replica
    ctr[..., 3] = iteration & 0xFFFFFFFF
    g = philox_normal3(philox4x32_10(ctr, key))
    cu = np.zeros((n_trials, 4), np.uint32)
    cu[:, 0] = np.arange(n_trials); cu[:, 1] = 0xB0000000; cu[:, 2] = replica; cu[:, 3] = iteration & 0xFFFFFFFF
    words = philox4x32_10(cu, key)
    u = (words[:, 0].astype(np.float64) + 0.5) * 2.0 ** -32
    return g, u


def shake(cons, mass, x0, x, tol):
    """Positions x moved onto the constraints (i, j, d), displacements along the bond vectors of x0 (Gauss-Seidel sweeps)."""
    x = x.copy()
    for _ in range(500):
        done = True
        for i, j, d in cons:
            i, j = int(i), int(j)
            r, r0 = x[i] - x[j], x0[i] - x0[j]
            diff = d * d - r @ r
            if abs(diff) > tol * d * d:
                done = False
                wi, wj = 1.0 / mass[i], 1.0 / mass[j]
                g = diff / (2.0 * (wi + wj) * (r @ r0))
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
            i, j = int(i), int(j)
            r, dv = x[i] - x[j], v[i] - v[j]
            rv, r2 = r @ dv, r @ r
            if abs(rv) > tol * r2:
                done = False
                wi, wj = 1.0 / mass[i], 1.0 / mass[j]
                g = rv / ((wi + wj) * r2)
                v[i] -= g * wi * r; v[j] += g * wj * r
        if done:
            break
    return v


def trial(x, mass, kT, energy_forces, gauss, u, dt, n_steps, cons=None, tol=1e-10, on_step=None):
    """One trial from positions x with standard normals `gauss` [N, 3] and uniform u.  energy_forces(x) -> (U, F); cons:
    constraints (i, j, d) or None; on_step(x): called with the positions after every step.  Returns (x, v, Eold, Enew,
    accepted)."""
    mass = np.asarray(mass, np.float64)
    m = mass[:, None]
    cons = [] if cons is None else list(cons)
    v = np.sqrt(kT / m) * gauss
    v = rattle(cons, mass, x, v, tol)
    U, f = energy_forces(x)
    e_old = 0.5 * np.sum(m * v * v) + U
    x_old = x.copy()
    for _ in range(n_steps):
        v = v + 0.5 * dt * f / m
        x1 = x + dt * v
        xc = shake(cons, mass, x, x1, tol) if cons else x1
        x = xc
        U, f = energy_forces(x)
        v = v + 0.5 * dt * f / m + (x - x1) / dt
        v = rattle(cons, mass, x, v, tol)
        if on_step is not None:
            on_step(x)
    e_new = 0.5 * np.sum(m * v * v) + U
    with np.errstate(over='ignore', invalid='ignore'):
        accepted = bool(np.exp(-(e_new - e_old) / kT) - u >= 0.0)   # step(exp(-(Enew-Eold)/kT) - uniform)
    if not accepted:
        x = x * 0.0 + x_old
    return x, v, e_old, e_new, accepted


def run(x, mass, kT, energy_forces, gauss, u, dt, n_steps, cons=None, tol=1e-10, on_step=None):
    """len(u) trials.  on_step(t, x): called with the trial's index and the positions after every step.  Returns (x, v,
    [(Eold, Enew, accepted) per trial])."""
    out, v = [], None
    for t in range(len(u)):
        cb = None if on_step is None else (lambda y, t=t: on_step(t, y))
        x, v, e0, e1, acc = trial(x, mass, kT, energy_forces, gauss[t], u[t], dt, n_steps, cons, tol, cb)
        out.append((e0, e1, acc))
    return x, v, out


def harmonic(K, x0):
    """(U, F) of the harmonic oscillator U = K/2 sum |x_i - x0|^2."""
    x0 = np.asarray(x0, np.float64)

    def ef(x):
        d = x - x0
        return 0.5 * K * np.sum(d * d), -K * d
    return ef


def lj(osys, lam):
    """(U, F) of the oracle's LJ system at lambda_sterics = lam."""
    def ef(x):
        U, _, f = osys.energy(x, lam, forces=True)
        return U, f
    return ef


def molecule(osys):
    """(U, F) of an oracle molecule (oracle.Molecule, or oracle.implicit's OBC system)."""
    def ef(x):
        U, f = osys.energy(np.ascontiguousarray(x), forces=True)
        return U, f
    return ef
