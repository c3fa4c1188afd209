"""Host restatement of the Monte Carlo rigid-body moves of openmmtools_b200/csrc/rx_mc.cuh.

Given positions, a subset, the proposal's randoms and the acceptance uniform, ``step`` returns the new positions and the
decision; the energies come from the caller (the oracle's LJ / region / molecule energies).  ``draws`` restates the
device's Philox blocks with helpers.philox4x32_10.  The proposal maps follow the reference's displace_positions,
_generate_uniform_quaternion, _rotation_matrix_from_quaternion and rotate_positions, and the accept rule its
MetropolizedMove.apply (/root/reference/openmmtools/mcmc.py:869-941, 1735-1760, 1802-1906); tests/test_mc_moves.py holds
them against the functions lifted from the reference."""
import numpy as np
from helpers import philox4x32_10

DISPLACEMENT, ROTATION = 0, 1
TAG = 0xE0000000


def draws(seed, iteration, replica, slot):
    """(proposal words [4] uint32, acceptance uniform) of replica `replica` in move slot `slot`."""
    key = (seed & 0xFFFFFFFF, ((seed >> 32) ^ (iteration >> 32)) & 0xFFFFFFFF)
    ctr = np.array([[slot, TAG, replica, iteration & 0xFFFFFFFF], [slot, TAG + 1, replica, iteration & 0xFFFFFFFF]], np.uint32)
    w = philox4x32_10(ctr, key).astype(np.uint64)
    u = (float(w[1, 0] >> np.uint64(5)) * 67108864.0 + float(w[1, 1] >> np.uint64(6))) / 9007199254740992.0
    return w[0], u


def uniforms(words):
    return (np.asarray(words, np.float64) + 0.5) / 4294967296.0


def normals(words):
    """Three standard normals (Box-Muller on words 0, 1 and 2, 3)."""
    u = uniforms(words)
    ra, rb = np.sqrt(-2.0 * np.log(u[0])), np.sqrt(-2.0 * np.log(u[2]))
    return np.array([ra * np.cos(2 * np.pi * u[1]), ra * np.sin(2 * np.pi * u[1]), rb * np.cos(2 * np.pi * u[3])])


def quaternion(u):
    """Shoemake's uniform quaternion (w, x, y, z) of three uniforms."""
    return np.array([np.sqrt(1 - u[0]) * np.sin(2 * np.pi * u[1]), np.sqrt(1 - u[0]) * np.cos(2 * np.pi * u[1]),
                     np.sqrt(u[0]) * np.sin(2 * np.pi * u[2]), np.sqrt(u[0]) * np.cos(2 * np.pi * u[2])])


def rotation_matrix(q):
    w, x, y, z = q
    Nq = float(np.sum(np.asarray(q) ** 2))
    s = 2.0 / Nq if Nq > 0.0 else 0.0
    X, Y, Z = x * s, y * s, z * s
    return np.array([[1.0 - (y * Y + z * Z), x * Y - w * Z, x * Z + w * Y],
                     [x * Y + w * Z, 1.0 - (x * X + z * Z), y * Z - w * X],
                     [x * Z - w * Y, y * Z + w * X, 1.0 - (x * X + y * Y)]])


def proposal(kind, words, sigma=0.0):
    """The displacement vector or the rotation matrix the device draws from `words`."""
    return sigma * normals(words) if kind == DISPLACEMENT else rotation_matrix(quaternion(uniforms(words[:3])))


def propose(kind, x, subset, T, box=None, store=np.float32):
    """(all positions with the subset moved, rounded to the storage precision and, on a periodic box, wrapped into it in
    f32; False when a periodic rotation is rejected because a rotated offset from the subset's first atom reaches half a
    box edge)."""
    x = np.array(x, np.float64)
    sub = np.asarray(subset)
    ok = True
    if kind == DISPLACEMENT:
        v = x[sub] + T
    else:
        base = x[sub[0]] if box is not None else np.zeros(3)
        o = x[sub] - base
        if box is not None:
            o = o - box * np.round(o / box)
            ok = bool(np.all(np.abs(o @ T.T) < 0.5 * box))
        m = o.sum(0) / len(sub)
        v = (base + m) + (o - m) @ T.T
    v = v.astype(store)
    if box is not None:     # wrapped in the storage precision, as the device's k_propagate wraps (wrap_into)
        L, iL = np.asarray(box, store), (1.0 / np.asarray(box, np.float64)).astype(store)
        v = (v - L * np.floor(v * iL)).astype(store)
    new = x.copy()
    new[sub] = v.astype(np.float64)
    return new, ok


def accept(dU, beta, u, ok=True):
    """MetropolizedMove.apply's rule with the replica's beta: dU finite and beta dU <= 0 or u < exp(-beta dU)."""
    return bool(ok and np.isfinite(dU) and (beta * dU <= 0.0 or u < np.exp(-beta * dU)))


def step(energy, x, subset, kind, T, u, beta, box=None, store=np.float32):
    """One move: (positions after it, accepted, dU or None when the proposal was rejected before any energy)."""
    new, ok = propose(kind, x, subset, T, box, store)
    dU = energy(new) - energy(np.asarray(x, np.float64)) if ok else None
    yes = accept(dU if ok else np.nan, beta, u, ok)
    return (new if yes else np.array(x, np.float64)), yes, dU
