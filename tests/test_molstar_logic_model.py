"""CPU model of k_propagate_mol<STAR>'s constraint path (csrc/rx_molecule.cuh: MolStar, mol_star_load / _invert / _rattle /
_shake) against the oracle's SHAKE / RATTLE sweeps (oracle/rx_oracle_mol.c, the restatement of the constrained R step of
/root/reference/openmmtools/integrators.py:1404-1460): the coefficient tables E, S of a cluster of <= 3 constraints over <= 4
atoms, the closed-form inverse of coup o (r r^T) formed once per position update, velocity projections as matrix-vector
products, SHAKE as chord iterations on the same inverse.  Statement for statement what the kernel does, in numpy."""
import numpy as np
import pytest
from openmmtools_b200 import testsystems, unit

KB = 8.31446261815324e-3


def clusters_of(cons, n):
    parent = list(range(n))

    def find(a):
        while parent[a] != a:
            a = parent[a]
        return a
    for i, j, _ in cons:
        parent[find(int(i))] = find(int(j))
    out = {}
    for c in cons:
        out.setdefault(find(int(c[0])), []).append(c)
    return list(out.values())


class Star:
    """mol_star_load: atoms in order of first appearance, padded tables."""

    def __init__(self, cons, mass):
        assert len(cons) <= 3
        self.nc = len(cons)
        at = []
        for i, j, _ in cons:
            for a in (int(i), int(j)):
                if a not in at:
                    at.append(a)
        assert len(at) <= 4                     # a connected cluster of nc constraints has at most nc + 1 atoms
        self.na, self.idx = len(at), at + [at[0]] * (4 - len(at))
        self.S, self.E, self.d2 = np.zeros((4, 3)), np.zeros((3, 4)), np.ones(3)
        for b, (i, j, d) in enumerate(cons):
            self.d2[b] = d * d
            for n, a in enumerate(at):
                self.S[n, b] = (1.0 / mass[a] if a == int(i) else 0.0) - (1.0 / mass[a] if a == int(j) else 0.0)
                self.E[b, n] = float(a == int(i)) - float(a == int(j))
        self.coup = self.E @ self.S
        self.r, self.Ai = np.zeros((3, 3)), np.eye(3)

    def invert(self):       # mol_star_invert: adjugate / determinant, unit diagonal for the padding
        A = self.coup * (self.r @ self.r.T)
        for a in range(self.nc, 3):
            A[a, a] = 1.0
        c00 = A[1, 1] * A[2, 2] - A[1, 2] * A[2, 1]; c01 = A[1, 0] * A[2, 2] - A[1, 2] * A[2, 0]; c02 = A[1, 0] * A[2, 1] - A[1, 1] * A[2, 0]
        idet = 1.0 / (A[0, 0] * c00 - A[0, 1] * c01 + A[0, 2] * c02)
        self.Ai = idet * np.array([
            [c00, A[0, 2] * A[2, 1] - A[0, 1] * A[2, 2], A[0, 1] * A[1, 2] - A[0, 2] * A[1, 1]],
            [-c01, A[0, 0] * A[2, 2] - A[0, 2] * A[2, 0], A[0, 2] * A[1, 0] - A[0, 0] * A[1, 2]],
            [c02, A[0, 1] * A[2, 0] - A[0, 0] * A[2, 1], A[0, 0] * A[1, 1] - A[0, 1] * A[1, 0]]])
        assert np.allclose(self.Ai @ A, np.eye(3), atol=1e-12)

    def init(self, X):
        self.r = self.E @ X[self.idx]
        self.invert()

    def rattle(self, V):
        v = V[self.idx].copy()
        g = np.einsum('aq,aq->a', self.r, self.E @ v)
        lam = self.Ai @ g
        for n in range(self.na):
            V[self.idx[n]] = v[n] - (self.S[n] * lam) @ self.r

    def shake(self, X, tol):
        x = X[self.idx].copy()
        for it in range(60):
            rc = self.E @ x
            g = np.where(np.arange(3) < self.nc, self.d2 - np.einsum('aq,aq->a', rc, rc), 0.0)
            if np.all(np.abs(g) <= tol * self.d2):
                break
            lam = 0.5 * (self.Ai @ g)
            x += (self.S * lam) @ self.r
        for n in range(self.na):
            X[self.idx[n]] = x[n]
        self.r = rc
        self.invert()
        return it


def test_cluster_tables_of_alanine_dipeptide():
    a = testsystems.AlanineDipeptideVacuum()
    cl = clusters_of(a.system.constraints, 22)
    assert sorted(len(c) for c in cl) == [1, 1, 1, 3, 3, 3]           # N-H, N-H, CA-H and three methyl groups
    for c in cl:
        s = Star(c, a.system.masses)
        assert s.na == s.nc + 1
        # the coupling matrix of mol_load_cluster (general path), entry by entry
        for p, (i, j, _) in enumerate(c):
            for q, (k, l, _) in enumerate(c):
                wi, wj = 1.0 / a.system.masses[int(i)], 1.0 / a.system.masses[int(j)]
                ref = (wi if i == k else 0) - (wi if i == l else 0) - (wj if j == k else 0) + (wj if j == l else 0)
                assert abs(s.coup[p, q] - ref) < 1e-15


@pytest.mark.parametrize('T', [300.0, 600.0, 1200.0])
def test_one_constrained_R_step_matches_the_oracle(T):
    from oracle import oracle
    a = testsystems.AlanineDipeptideVacuum()
    x0 = np.ascontiguousarray(a.positions.value_in_unit(unit.nanometer), np.float64)
    m = oracle.Molecule(a.system)
    rng = np.random.default_rng(int(T))
    v0 = rng.normal(size=x0.shape) * np.sqrt(KB * T / m.mass)[:, None]
    stars = [Star(c, m.mass) for c in clusters_of(a.system.constraints, 22)]
    # entry convention of the kernel: cache at the incoming positions, incoming velocities projected
    X, V = x0.copy(), v0.copy()
    for s in stars:
        s.init(X); s.rattle(V)
    xo, vo = x0.copy(), np.ascontiguousarray(v0.copy())
    import ctypes as C
    oracle.lib().orc_mol_rattle(C.byref(m.s), xo.ctypes.data_as(C.c_void_p), vo.ctypes.data_as(C.c_void_p), C.c_double(1e-14))
    assert np.abs(V - vo).max() < 1e-11
    h, tol = 0.002, 1e-12
    for step in range(5):
        # R: move, SHAKE (chord iterations on the cached inverse), velocity correction, RATTLE with the rebuilt cache
        V = V - (m.mass[:, None] * V).sum(0) / m.mass.sum()      # CMMotionRemover at the start of the step
        xu = X + h * V
        X = xu.copy()
        its = [s.shake(X, tol) for s in stars]
        assert max(its) <= 9, its                      # ~1.5-2 digits per iteration
        V = V + (X - xu) / h
        for s in stars:
            s.rattle(V)
        m.langevin(xo, vo, np.zeros((0, 22, 3)), KB * T, h, 5.0, 1, 'R', tol=1e-14)
        assert np.abs(X - xo).max() < 2e-12, (step, np.abs(X - xo).max())
        assert np.abs(V - vo).max() < 2e-9, (step, np.abs(V - vo).max())
        c = a.system.constraints
        i, j = c[:, 0].astype(int), c[:, 1].astype(int)
        assert np.abs(np.linalg.norm(X[i] - X[j], axis=1) - c[:, 2]).max() < 1e-12
        assert np.abs(np.einsum('cq,cq->c', X[i] - X[j], V[i] - V[j])).max() < 1e-12


def water_dimer():
    """Two rigid TIP3P waters in vacuum (NoCutoff): no bonded terms, three distance constraints per molecule -- a cluster of
    three constraints over three atoms (a cycle), what SETTLE solves in OpenMM."""
    from openmmtools_b200.system import System, MOLECULE
    rOH, rHH = 0.09572, 0.15139
    h = np.sqrt(rOH ** 2 - (rHH / 2) ** 2)
    w = np.array([[0.0, 0.0, 0.0], [rHH / 2, h, 0.0], [-rHH / 2, h, 0.0]])
    R = np.array([[0.36, 0.48, 0.8], [-0.8, 0.6, 0.0], [0.48, 0.64, -0.6]])     # a rotation
    x = np.concatenate([w, w @ R.T + np.array([0.05, -0.28, 0.12])])
    s = System(MOLECULE, np.array([15.9994, 1.008, 1.008] * 2))
    s.charge = np.array([-0.834, 0.417, 0.417] * 2)
    s.sigma = np.array([0.315075, 0.1, 0.1] * 2)      # (hydrogens: epsilon = 0, any positive sigma)
    s.epsilon = np.array([0.635968, 0.0, 0.0] * 2)
    s.bonds = np.zeros((0, 4)); s.angles = np.zeros((0, 5)); s.torsions = np.zeros((0, 7)); s.exceptions = np.zeros((0, 5))
    s.exclusions = np.array([[0, 1], [0, 2], [1, 2], [3, 4], [3, 5], [4, 5]], np.int64)
    s.constraints = np.array([[0, 1, rOH], [0, 2, rOH], [1, 2, rHH], [3, 4, rOH], [3, 5, rOH], [4, 5, rHH]])
    s.remove_cm_motion = False
    return s, np.ascontiguousarray(x)


def test_rigid_water_is_a_cluster_the_same_path_solves():
    from oracle import oracle
    s, x0 = water_dimer()
    m = oracle.Molecule(s)
    cl = clusters_of(s.constraints, 6)
    assert [len(c) for c in cl] == [3, 3]
    stars = [Star(c, m.mass) for c in cl]
    assert all(st.na == 3 and st.nc == 3 for st in stars)
    rng = np.random.default_rng(1)
    v0 = rng.normal(size=x0.shape) * np.sqrt(KB * 300.0 / m.mass)[:, None]
    X, V = x0.copy(), v0.copy()
    for st in stars:
        st.init(X); st.rattle(V)
    import ctypes as C
    xo, vo = x0.copy(), np.ascontiguousarray(v0.copy())
    oracle.lib().orc_mol_rattle(C.byref(m.s), xo.ctypes.data_as(C.c_void_p), vo.ctypes.data_as(C.c_void_p), C.c_double(1e-14))
    assert np.abs(V - vo).max() < 1e-10
    h = 0.002
    for step in range(5):
        xu = X + h * V
        X = xu.copy()
        its = [st.shake(X, 1e-12) for st in stars]
        assert max(its) <= 12, its
        V = V + (X - xu) / h
        for st in stars:
            st.rattle(V)
        m.langevin(xo, vo, np.zeros((0, 6, 3)), KB * 300.0, h, 5.0, 1, 'R', tol=1e-14)
        assert np.abs(X - xo).max() < 5e-12 and np.abs(V - vo).max() < 5e-9, (step, np.abs(X - xo).max(), np.abs(V - vo).max())


def emulate_kernel(m, stars, x0, v0, noise, kT, dt, gamma, n_steps, remove_cm):
    """k_propagate_mol's step loop, statement for statement, with f64 forces from the oracle: V R O R V with the lazy force
    flag, the cluster path after every operation, the kernel's entry convention (cache built, incoming velocities projected)."""
    X, V = x0.copy(), v0.copy()
    for st in stars:
        st.init(X); st.rattle(V)
    a, b = np.exp(-gamma * dt), np.sqrt(1.0 - np.exp(-2.0 * gamma * dt))
    sg = np.sqrt(kT / m.mass)[:, None]
    hV = hR = dt / 2
    f, oc = None, 0
    for _ in range(n_steps):
        if remove_cm:
            V = V - (m.mass[:, None] * V).sum(0) / m.mass.sum()
        for op in 'VRORV':
            if op == 'V':
                if f is None:
                    f = m.energy(np.ascontiguousarray(X), forces=True)[1]
                V = V + hV * f / m.mass[:, None]
            elif op == 'R':
                xu = X + hR * V
                X = xu.copy()
                for st in stars:
                    st.shake(X, 1e-10)
                V = V + (X - xu) / hR
                f = None
            else:
                V = a * V + b * sg * noise[oc]; oc += 1
            for st in stars:
                st.rattle(V)
    return X, V


@pytest.mark.parametrize('which', ['alanine dipeptide', 'water dimer', 'decane shuffled', 'ten waters'])
def test_whole_step_sequence_matches_the_oracle(which):
    import ctypes as C
    from oracle import oracle
    from helpers import device_noise, alkane, waters
    if which == 'water dimer':
        s, x0 = water_dimer()
    elif which == 'decane shuffled':      # clusters of 2 and 3 constraints, i > j, clusters interleaved in the list
        s, x0 = alkane(10, terms_per_torsion=3, shuffle=5)
    elif which == 'ten waters':
        s, x0 = waters(10, shuffle=3)
    else:
        a = testsystems.AlanineDipeptideVacuum()
        s, x0 = a.system, np.ascontiguousarray(a.positions.value_in_unit(unit.nanometer), np.float64)
    n = len(x0)
    m = oracle.Molecule(s)
    kT, dt, gamma, n_steps = KB * 420.0, 0.002, 5.0, 40
    v0 = np.random.default_rng(2).normal(size=x0.shape) * np.sqrt(kT / m.mass)[:, None]
    noise = device_noise(99, 3, 0, n, n_steps).astype(np.float64)
    xo, vo = x0.copy(), np.ascontiguousarray(v0.copy())
    oracle.lib().orc_mol_rattle(C.byref(m.s), xo.ctypes.data_as(C.c_void_p), vo.ctypes.data_as(C.c_void_p), C.c_double(1e-10))
    m.langevin(xo, vo, noise, kT, dt, gamma, n_steps, 'VRORV', tol=1e-10)
    stars = [Star(c, m.mass) for c in clusters_of(s.constraints, n)]
    X, V = emulate_kernel(m, stars, x0, v0, noise, kT, dt, gamma, n_steps, bool(s.remove_cm_motion))
    assert np.abs(X - xo).max() < 1e-9 and np.abs(V - vo).max() < 1e-7, (np.abs(X - xo).max(), np.abs(V - vo).max())
