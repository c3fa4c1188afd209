"""The instruments of test_gpu_hmc_variants.py, checked without a device: the constraint clusters that route each molecule
to the kernel path the GPU test claims for it, the list-rebuild threshold of its rebuild-inside-a-rejected-trial test, the
quadrature of its flexible-bond test, and that the same bound detects velocity Verlet without the accept test."""
import numpy as np
import pytest
import helpers as H
from helpers import KB, lj_setup, constraint_clusters

MOL_MAXC = 4   # clusters of up to this many constraints: Newton M-SHAKE; more: sweeps (rx_molecule.cuh)


def largest_cluster(name):
    from test_gpu_molecule import MOLECULES
    s, _ = MOLECULES[name]()
    cl = constraint_clusters(s.constraints, s.n_particles)
    return s, sorted(len(c) for c in cl)


# name -> (cluster sizes, path): MolStar when every cluster has at most 3 constraints (rxi_propagate's STAR), else the
# general path, M-SHAKE up to MOL_MAXC and sweeps above.
ROUTES = {
    'mixture': ([1, 2, 3, 4], 'mshake'), 'mixture-shuffled': ([1, 2, 3, 4], 'mshake'), 'methane': ([4], 'mshake'),
    'propane-AllBonds': ([10], 'sweeps'), 'propane-AllBonds-shuffled': ([10], 'sweeps'),
    'waters': ([3] * 10, 'star'), 'waters-ion-shuffled': ([3] * 10, 'star'),
    'decane': ([2] * 8 + [3] * 2, 'star'), 'decane-3terms-shuffled': ([2] * 8 + [3] * 2, 'star'),
    'torsion-probe': ([], None), 'ion': ([], None), 'diatomic': ([1], 'star'),
}


@pytest.mark.parametrize('name', sorted(ROUTES))
def test_each_molecule_routes_to_the_path_its_gpu_case_claims(name):
    s, sizes = largest_cluster(name)
    want, path = ROUTES[name]
    assert sizes == want
    if sizes:
        top = sizes[-1]
        assert path == ('star' if top <= 3 else 'mshake' if top <= MOL_MAXC else 'sweeps')
    if name.startswith('waters'):   # every cluster a 3-cycle (a rigid water)
        for c in constraint_clusters(s.constraints, s.n_particles):
            assert len({int(a) for r in c for a in r[:2]}) == 3
    if name == 'decane':            # tables above 48 KB: the HMC kernel needs the shared-memory opt-in
        assert s.n_particles == 32


def test_gpu_molecule_cases_cover_every_path():
    from test_gpu_hmc_variants import MOLECULE_CASES, STAR_ELIGIBLE
    paths = {ROUTES[n][1] for n in MOLECULE_CASES if n in ROUTES}
    assert {'star', 'mshake', 'sweeps', None} <= paths
    assert all(ROUTES.get(n, (None, 'star'))[1] == 'star' for n in STAR_ELIGIBLE)


# ---- the rebuild threshold: list_geometry's rules (rx_dynamics.cu) restated ------------------------------------------------
def half_out(box, r_cutoff, skin_out, skin_in):
    rl = min([r_cutoff + skin_out] + [0.5 * b for b in box])
    eff_out = rl - r_cutoff
    skin_in = min(skin_in, eff_out / 3.0)
    return 0.5 * (eff_out - skin_in)


@pytest.mark.parametrize('N,cl', [(256, 1), (777, 4), (2048, 2)])
def test_rebuild_threshold_of_the_shrunk_skins(N, cl):
    """With RX_SKIN = 0.09 and RX_SKIN_IN = 0.03 an outer rebuild comes once an atom has moved 0.03 nm, the list is kept
    and the atoms are sorted (re-dealt at a rebuild) at the cluster widths the GPU test runs."""
    from test_gpu_hmc_variants import HALF_OUT
    from openmmtools_b200._engine import Engine
    from openmmtools_b200._lib import RX_SYSTEM_LJ_ALCH
    s = lj_setup(N=N, n_alch=6, seed=N)
    assert half_out(s['box'], s['rc'], 0.09, 0.03) == pytest.approx(HALF_OUT, abs=1e-12)
    p = Engine.plan_propagate(RX_SYSTEM_LJ_ALCH, N, 2, 132, 227 * 1024, box=tuple(s['box']), r_cutoff=s['rc'],
                              skin_out=0.09, skin_in=0.03, cluster=cl)
    assert p['cluster'] == cl and p['list_capacity'] > 0 and p['sort_atoms'] == 1


# ---- the flexible bond: quadrature, and the control without the accept test -----------------------------------------------
BOND_K, BOND_R0 = 250000.0, 0.1275
BOND_MU = 35.45 * 1.008 / (35.45 + 1.008)
# (replicas, K, steps per trial = trials per launch, launches, dt = 1 / omega)
BOND_STATS = (128, 300.0, 10, 220, 1.0 / np.sqrt(BOND_K / BOND_MU))


def flexible_hcl():
    """Cl-H with one harmonic bond (k = 250 000 kJ/mol/nm^2, r0 = 0.1275 nm); the 1-2 exclusion leaves no other term."""
    return H._mol_system(['Cl', 'H'], np.array([[0.0, 0.0, 0.0], [BOND_R0, 0.0, 0.0]]), np.array([-0.2, 0.2]), [(0, 1)],
                         None, jitter=0.0)


def bond_msd_quadrature(kT):
    """<(r - r0)^2> under the density r^2 exp(-k (r - r0)^2 / 2kT), r > 0 (trapezoid over +-12 widths)."""
    w = np.sqrt(kT / BOND_K)
    r = np.linspace(max(BOND_R0 - 12 * w, 0.0), BOND_R0 + 12 * w, 200001)
    p = r * r * np.exp(-0.5 * BOND_K * (r - BOND_R0) ** 2 / kT)
    return np.trapezoid(p * (r - BOND_R0) ** 2, r) / np.trapezoid(p, r)


def test_flexible_hcl_is_one_bond_and_nothing_else():
    s, _ = flexible_hcl()
    assert len(s.bonds) == 1 and s.bonds[0][2] == BOND_K and s.bonds[0][3] == BOND_R0
    assert not len(s.constraints) and not len(s.angles) and not len(s.torsions)
    assert BOND_MU == pytest.approx(1.0 / (1.0 / s.masses[0] + 1.0 / s.masses[1]), rel=1e-12)


def test_bond_quadrature_equals_brute_force_cartesian_integration():
    """The same average as a midpoint sum over a Cartesian grid of the relative coordinate (one octant, by symmetry): no
    r^2 Jacobian written by hand."""
    kT = KB * 300.0
    h = 2.5e-4
    g = (np.arange(int(0.15 / h)) + 0.5) * h
    msd_num = msd_den = 0.0
    for xv in g:   # (slab by slab, to keep memory small)
        r = np.sqrt(xv * xv + g[:, None] ** 2 + g[None, :] ** 2)
        p = np.exp(-0.5 * BOND_K * (r - BOND_R0) ** 2 / kT)
        msd_num += np.sum(p * (r - BOND_R0) ** 2); msd_den += np.sum(p)
    assert bond_msd_quadrature(kT) == pytest.approx(msd_num / msd_den, rel=2e-4)
    assert bond_msd_quadrature(kT) == pytest.approx(kT / BOND_K, rel=0.01)   # (nearly the harmonic kT/k)


def verlet_without_accept_test(rng):
    """The two atoms under velocity Verlet, velocities redrawn before every trial and every trial kept; the per-chain mean
    of (r - r0)^2 over the launches the GPU test averages."""
    K, T, n_steps, n_launches, dt = BOND_STATS
    kT = KB * T
    m = np.array([35.45, 1.008])[None, :, None]
    x = np.zeros((K, 2, 3)); x[:, 1, 0] = BOND_R0

    def force(x):
        d = x[:, 1] - x[:, 0]
        r = np.linalg.norm(d, axis=1)[:, None]
        f1 = -BOND_K * (r - BOND_R0) * d / r
        return np.stack([-f1, f1], axis=1)
    out = []
    for it in range(n_launches):
        for _ in range(n_steps):
            v = rng.normal(size=x.shape) * np.sqrt(kT / m)
            f = force(x)
            for _ in range(n_steps):
                v = v + 0.5 * dt * f / m; x = x + dt * v; f = force(x); v = v + 0.5 * dt * f / m
        if it >= n_launches // 10:
            out.append((np.linalg.norm(x[:, 1] - x[:, 0], axis=1) - BOND_R0) ** 2)
    return np.mean(out, axis=0)


def test_the_bond_bound_detects_verlet_without_the_accept_test():
    r = verlet_without_accept_test(np.random.default_rng(7)) / bond_msd_quadrature(KB * BOND_STATS[1])
    K = BOND_STATS[0]
    assert abs(r.mean() - 1.0) > 5 * r.std(ddof=1) / np.sqrt(K) + 0.01, (r.mean(), r.std(ddof=1) / np.sqrt(K))
