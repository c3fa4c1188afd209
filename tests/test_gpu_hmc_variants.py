"""Hybrid Monte Carlo on the device beyond test_gpu_hmc.py: every molecule constraint path (MolStar, Newton M-SHAKE,
sweeps) and cluster shape, OBC1/OBC2 with and without ACE, the LJ layouts the HMC instantiations of k_propagate launch,
list rebuilds and re-deals inside rejected trials, several launches, the fixed-point range rule, the NaN rule and the
retry, the stationary distribution of a flexible bond, and the sampler on a molecule in implicit solvent.

Every oracle-parity case compares each trial of each launch with tests/hmc_oracle.py fed the device's draws
(test_gpu_hmc.check_replica) and asserts that it ran both decisions and a rejected trial followed by another trial of the
same launch (so the restore after a rejection is compared, not only its end state).  Timesteps and temperatures were
picked on the host with the oracle for acceptance between about 0.3 and 0.8 on these draws, with every trial's
|u - exp(-dH/kT)| several times the energy tolerance of check_replica away from a tie."""
import os
import numpy as np
import pytest
import hmc_oracle as ho
from helpers import KB, lj_setup, oracle_system, min_image, gpu_engine, scattered_alch
from regions_ref import RegionsReference
from test_gpu_hmc import SEED, IT, check_replica, lj_engine, harmonic_engine, f32
from test_gpu_molecule import MOLECULES
from test_hmc_variants_host import flexible_hcl, bond_msd_quadrature, BOND_R0, BOND_STATS
from openmmtools_b200 import _lib, mcmc, unit, states, testsystems, multistate
from openmmtools_b200._engine import EngineError

pytestmark = pytest.mark.gpu


def assert_exercised(per_replica, n_steps):
    """Both decisions occur, and some rejected trial is followed by another trial of the same launch."""
    d = [t[2] for trials in per_replica for t in trials]
    assert 0 < sum(d) < len(d), d
    assert any(not tr[i][2] and i % n_steps != n_steps - 1 for tr in per_replica for i in range(len(tr))), d


def constraint_error(cons, x):
    i, j = cons[:, 0].astype(int), cons[:, 1].astype(int)
    return np.abs(np.linalg.norm(x[..., i, :] - x[..., j, :], axis=-1) - cons[:, 2]).max()


# ---- A, B. molecules: both constraint paths, every cluster shape, vacuum and OBC -------------------------------------------
def oracle_molecule(system):
    if system.gb_parameters is not None:
        from oracle import implicit as oi
        return oi.Molecule(system)
    from oracle import oracle
    return oracle.Molecule(system)


def molecule_start(system, x, m, K):
    rng = np.random.default_rng(2)
    x0 = np.stack([x + rng.normal(0, 0.002, x.shape) for _ in range(K)])
    if len(m.cons):   # start on the constraints (a trial rejected back to the start is then on them too)
        x0 = np.stack([ho.shake(m.cons, m.mass, xk, xk, 1e-12) for xk in x0])
    return x0


def run_molecule(system, x, n_steps, dt, temps=(300.0, 450.0), launches=2, exercised=True, tol_x=2e-5, tol_v=1e-2):
    """K = 2 replicas on the permuted states [1, 0], `launches` launches from iteration IT, against the oracle.  Returns
    the oracle molecule, the device's positions and each replica's trials."""
    K = 2
    temps = np.asarray(temps, float)
    m = oracle_molecule(system)
    e = gpu_engine(_lib.RX_SYSTEM_MOLECULE, K, K, system.n_particles)
    e.set_molecule(system, constraint_tolerance=1e-10)
    e.set_states(temps, np.ones(K))
    e.set_hmc_integrator(dt, n_steps)
    x0 = molecule_start(system, x, m, K)
    e.set_positions(x0); e.set_velocities(np.zeros_like(x0))
    perm = np.array([1, 0])
    e.set_replica_states(perm)
    its = tuple(range(IT, IT + launches))
    for it in its:
        e.propagate(SEED, it)
    xg, vg = e.get_positions(), e.get_velocities()
    cons = m.cons if len(m.cons) else None
    per = [check_replica(e, k, x0[k], m.mass, KB * temps[perm[k]], ho.molecule(m), dt, n_steps, xg, vg, tol_x=tol_x,
                         tol_v=tol_v, cons=cons, iterations=its) for k in range(K)]
    if exercised:
        assert_exercised(per, n_steps)
    if cons is not None:
        assert constraint_error(cons, xg) < 1e-10
    e.close()
    return m, xg, per


# (n_steps, dt ps) per molecule at 300 / 450 K.  Largest constraint cluster (test_hmc_variants_host.py checks it): 4 for
# mixture and methane (Newton M-SHAKE), 10 for propane-AllBonds (sweeps), 3 for waters, decane and alanine dipeptide
# (MolStar), 1 for diatomic (MolStar), none for torsion-probe and ion.
MOLECULE_CASES = {
    'mixture': (8, 0.005), 'mixture-shuffled': (8, 0.0035), 'methane': (8, 0.0045),
    'propane-AllBonds': (8, 0.0035), 'propane-AllBonds-shuffled': (8, 0.0035),
    'waters': (5, 0.008), 'waters-ion-shuffled': (6, 0.007),
    'decane': (7, 0.004), 'decane-3terms-shuffled': (8, 0.003),
    'torsion-probe': (8, 0.0035), 'alanine-dipeptide': (8, 0.003),
}
STAR_ELIGIBLE = ('waters', 'decane', 'alanine-dipeptide')
# The clusters of rigid waters are chaotic at the steps that bring their acceptance into the band: in the oracle itself a
# 1e-7 nm displacement of the start grows to 2e-5 nm over these launches (to 0.1 nm at 7 fs, 8 x 8 steps, 600 / 900 K),
# so their positions are compared to 2e-4 nm and velocities to 5e-2 nm/ps.  (Their steps cannot grow further: near 10 fs
# SHAKE stops converging, in the oracle's sweeps and on the device.)
CHAOTIC = {'waters': dict(tol_x=2e-4, tol_v=5e-2), 'waters-ion-shuffled': dict(tol_x=2e-4, tol_v=5e-2)}


@pytest.mark.parametrize('name,no_star', [(n, False) for n in MOLECULE_CASES] + [(n, True) for n in STAR_ELIGIBLE])
def test_molecule_trials_match_oracle(monkeypatch, name, no_star):
    if no_star:   # the general cluster path (M-SHAKE) for a molecule MolStar would take
        monkeypatch.setenv('RX_MOL_NO_STAR', '1')
    system, x = MOLECULES[name]()
    run_molecule(system, x, *MOLECULE_CASES[name], **CHAOTIC.get(name, {}))


@pytest.mark.parametrize('no_star', [False, True])
def test_free_rigid_rotor_decisions_match_oracle(monkeypatch, no_star):
    """The constrained diatomic has U = 0: a free rigid rotor, dH = 0 up to the constraint solves, every trial accepted on
    the device as in the oracle."""
    if no_star:
        monkeypatch.setenv('RX_MOL_NO_STAR', '1')
    system, x = MOLECULES['diatomic']()
    _, _, per = run_molecule(system, x, 6, 0.004, exercised=False)
    assert all(t[2] for tr in per for t in tr)


def test_free_particle_energy_is_kinetic_and_trials_are_counted():
    """n = 1: no terms, no clusters.  H is 1/2 m v^2 of the drawn velocity in every trial (dH = 0, every trial accepted)."""
    system, x = MOLECULES['ion']()
    n_steps, dt, temps = 5, 0.004, np.array([300.0, 450.0])
    m, _, per = run_molecule(system, x, n_steps, dt, temps=temps, exercised=False)
    for k, l in enumerate([1, 0]):
        ke = []
        for it in (IT, IT + 1):
            g, _ = ho.draws(SEED, it, k, 1, n_steps)
            v = np.sqrt(KB * temps[l] / m.mass[:, None]) * g
            ke += list(0.5 * np.sum(m.mass[:, None] * v * v, axis=(1, 2)))
        assert np.allclose([t[0] for t in per[k]], ke, rtol=1e-12, atol=0) and all(t[0] == t[1] and t[2] for t in per[k])


def toluene(model, ace):
    from implicit_helpers import implicit_system, with_model
    system, x = implicit_system('toluene')
    return with_model(system, model, ace), x


@pytest.mark.parametrize('model,ace', [('OBC1', True), ('OBC1', False), ('OBC2', True), ('OBC2', False)])
def test_toluene_in_obc_trials_match_oracle(model, ace):
    run_molecule(*toluene(model, ace), 8, 0.003)


@pytest.mark.parametrize('name,model,ace,n_steps,dt', [
    ('mixture', 'OBC1', True, 7, 0.004),                 # GB with the general constraint path
    ('decane', 'OBC2', True, 7, 0.004),                  # 32 atoms: the largest GB arrays, tables above 48 KB
    ('waters-ion-shuffled', 'OBC2', False, 5, 0.007)])
def test_molecules_in_obc_trials_match_oracle(name, model, ace, n_steps, dt):
    """The rigid waters in OBC2 accept 19 of these 20 trials (the solvent screens the charges), and at steps long enough
    for more rejections SHAKE no longer converges or the clusters turn chaotic (CHAOTIC): their trials are compared with
    the oracle's, but the rejection is the last trial of its launch."""
    from implicit_helpers import obc
    system, x = MOLECULES[name]()
    waters = name.startswith('waters')
    run_molecule(obc(system, model, ace), x, n_steps, dt, exercised=not waters, **CHAOTIC.get(name, {}))


# ---- C, D. LJ layouts ------------------------------------------------------------------------------------------------------
# The dilute fluid accepts nearly every trial at 2 fs (DESIGN 4.6): 8 steps of 50 fs give about 0.4-0.6 up to 1100 atoms.
# dH grows with N, so larger fluids take shorter steps.
DT_LJ, N_LJ = 0.05, 8


def run_lj(monkeypatch, N, cl=None, sort=True, switch=True, c=6.0, regions=False, dts=(DT_LJ, DT_LJ), n_steps=N_LJ,
           env=(), s=None):
    """K = 2 replicas on the permuted states [1, 0] (lambda 1.0 / 0.4, 300 / 330 K), per-state timesteps when dts differ;
    one launch against the oracle.  Returns the device's (positions, velocities, statistics, energies)."""
    if cl is not None:
        monkeypatch.setenv('RX_CLUSTER', str(cl))
    if not sort:
        monkeypatch.setenv('RX_NO_SORT', '1')
    for kv in env:
        monkeypatch.setenv(*kv)
    K = 2
    lambdas, temps = np.array([1.0, 0.4]), np.array([300.0, 330.0])
    if regions:
        s = s or lj_setup(N=N, seed=N, alch=scattered_alch(N, cluster=8))
        ids = np.where(s['alch'] != 0, 1 + np.arange(N) % 2, 0).astype(np.uint8)
        eng = gpu_engine(_lib.RX_SYSTEM_LJ_ALCH, K, 2, N, box=tuple(s['box']), r_cutoff=s['rc'], r_switch=s['rs'],
                         use_switch=switch, softcore_c=c)
        eng.set_particles(s['sigma'], s['eps'], s['mass'], (ids != 0).astype(np.uint8))
        eng.set_alchemical_regions(ids, False, False)
        eng.set_states(temps, lambda_sterics=lambdas, lambda_sterics_2=1.0 - lambdas)
        eng.set_hmc_integrator(dts[0], n_steps)
        ref = RegionsReference(s, ids)
        ef = [lambda y, l=l: ref.energy(y, lambdas[l], 1.0 - lambdas[l], forces=True) for l in range(2)]
    else:
        s = s or lj_setup(N=N, n_alch=6, seed=N)
        eng = gpu_engine(_lib.RX_SYSTEM_LJ_ALCH, K, 2, N, box=tuple(s['box']), r_cutoff=s['rc'], r_switch=s['rs'],
                         use_switch=switch, softcore_c=c)
        eng.set_particles(s['sigma'], s['eps'], s['mass'], s['alch'])
        eng.set_states(temps, lambda_sterics=lambdas)
        eng.set_hmc_integrator(dts[0], n_steps)
        osys = oracle_system(s, use_switch=switch, c=c)
        ef = [ho.lj(osys, lam) for lam in lambdas]
    if dts[1] != dts[0]:
        eng.set_state_hmc_integrator(1, dts[1], n_steps)
    x0 = np.stack([s['x']] * K)
    eng.set_positions(x0); eng.set_velocities(np.zeros_like(x0))
    perm = np.array([1, 0])
    eng.set_replica_states(perm)
    eng.propagate(SEED, IT)
    xg, vg = eng.get_positions(), eng.get_velocities()
    per = [check_replica(eng, k, x0[k], s['mass'], KB * temps[perm[k]], ef[perm[k]], dts[perm[k]], n_steps, xg, vg,
                         s['box']) for k in range(K)]
    assert_exercised(per, n_steps)
    out = (xg, vg, eng.get_hmc_statistics(), eng.get_hmc_energies())
    eng.close()
    return out


@pytest.mark.parametrize('c', [4.0, 12.0])
@pytest.mark.parametrize('switch', [True, False])
def test_softcore_exponents_other_than_6(monkeypatch, c, switch):
    """The C6 = false instantiations."""
    run_lj(monkeypatch, 256, cl=1, switch=switch, c=c)


@pytest.mark.parametrize('N,cl,dts', [(1100, None, (DT_LJ, 0.04)), (2048, 2, (0.04, 0.035))])
def test_per_state_moves_at_the_compact_layout(monkeypatch, N, cl, dts):
    run_lj(monkeypatch, N, cl=cl, dts=dts)


@pytest.mark.parametrize('N,cl,dt', [(2048, 2, 0.04), (4096, 8, 0.035)])
def test_two_regions_at_the_compact_layout(monkeypatch, N, cl, dt):
    run_lj(monkeypatch, N, cl=cl, regions=True, dts=(dt, dt))


def test_per_state_moves_with_two_regions(monkeypatch):
    run_lj(monkeypatch, 256, cl=1, regions=True, dts=(DT_LJ, 0.04))


def test_4096_atoms_in_8_blocks(monkeypatch):
    run_lj(monkeypatch, 4096, cl=8, dts=(0.03, 0.03))


def test_40_atoms_without_a_list(monkeypatch):
    run_lj(monkeypatch, 40, dts=(0.06, 0.06))


def test_300_atoms_without_the_verlet_list(monkeypatch):
    run_lj(monkeypatch, 300, env=[('RX_NO_VERLET', '1')], dts=(0.055, 0.055))


DT_DENSE, N_DENSE = 0.004, 6


def test_dense_fluid_all_pairs_fallback(monkeypatch):
    """test_gpu_large_replicas' liquid-density fluid: more neighbours than a list column holds, the all-pairs loop."""
    from test_gpu_large_replicas import big
    s = big(2048, seed=31, box='cubic', reduced_density=0.6)
    run_lj(monkeypatch, 2048, s=s, dts=(DT_DENSE, DT_DENSE), n_steps=N_DENSE)


HARMONIC_DT = {33: 0.4, 1000: 0.07}


@pytest.mark.parametrize('N', [33, 1000])
def test_harmonic_warps_match_oracle(N):
    """A partial last warp (33) and 32 warps (1000)."""
    K, n_steps, dt = 2, 6, HARMONIC_DT[N]
    Ks, x0s, temps = np.array([40.0, 90.0]), np.array([[0.0, 0, 0], [0.1, 0, -0.05]]), np.array([300.0, 330.0])
    eng = harmonic_engine(K, N, Ks, x0s, temps, dt, n_steps)
    x0 = np.random.default_rng(N).normal(scale=0.1, size=(K, N, 3))
    eng.set_positions(x0); eng.set_velocities(np.zeros_like(x0))
    perm = np.array([1, 0])
    eng.set_replica_states(perm)
    eng.propagate(SEED, IT)
    xg, vg = eng.get_positions(), eng.get_velocities()
    mass = np.full(N, 39.948)
    per = [check_replica(eng, k, x0[k], mass, KB * temps[perm[k]], ho.harmonic(Ks[perm[k]], x0s[perm[k]]), dt, n_steps,
                         xg, vg, tol_x=2e-5, tol_v=2e-4) for k in range(K)]
    assert_exercised(per, n_steps)


def test_same_bits_at_every_compact_width_unsorted(monkeypatch):
    s = lj_setup(N=2048, n_alch=6, seed=3)
    K, lambdas, temps = 2, np.array([1.0, 0.4]), np.array([300.0, 330.0])
    x0 = np.stack([s['x']] * K)
    monkeypatch.setenv('RX_NO_SORT', '1')
    out = []
    for cl in (2, 4, 8):
        monkeypatch.setenv('RX_CLUSTER', str(cl))
        eng = lj_engine(s, K, lambdas, temps, 0.04, N_LJ)
        eng.set_positions(x0); eng.set_velocities(np.zeros_like(x0))
        eng.propagate(SEED, IT)
        eng.propagate(SEED, IT + 1)
        out.append((eng.get_positions(), eng.get_velocities(), eng.get_hmc_statistics(), eng.get_hmc_energies()))
        eng.close()
    for o in out[1:]:
        assert np.array_equal(o[0], out[0][0]) and np.array_equal(o[1], out[0][1])
        assert all(np.array_equal(a, b) for a, b in zip(o[2], out[0][2]))
        assert all(np.array_equal(a, b) for a, b in zip(o[3], out[0][3]))
    assert 0 < out[0][2][0].sum() < out[0][2][1].sum() == K * 2 * N_LJ


# Skins of test_gpu_large_replicas' rebuild test: the outer list is rebuilt (and the atoms re-dealt with the sorted deal)
# once an atom has moved (r_list - r_c - skin_in) / 2 = (0.09 - 0.03) / 2 = 0.03 nm from the list's reference positions.
SKINS = [('RX_SKIN', '0.09'), ('RX_SKIN_IN', '0.03')]
HALF_OUT = 0.03


@pytest.mark.parametrize('N,cl,other,dt', [(256, 1, 2, DT_LJ), (777, 4, 2, DT_LJ), (2048, 2, 4, 0.04)])
def test_rebuild_inside_a_rejected_trial(monkeypatch, N, cl, other, dt):
    """xold lives in the replica's row of global pos because a rebuild inside a trial may hand the thread another atom.
    The oracle's trajectory proves that a rejected trial moved some atom more than 2 half_out from the trial's start, so
    the list was rebuilt inside it whatever its reference positions were (they lie within half_out of the start).  The
    same launch unsorted and at another cluster width gives the same bits."""
    s = lj_setup(N=N, n_alch=6, seed=N)
    lambdas, temps = np.array([1.0, 0.4]), np.array([300.0, 330.0])
    osys = oracle_system(s)
    moved_in_rejected = []
    for l in range(2):
        g, u = ho.draws(SEED, IT, 1 - l, N, N_LJ)      # (states [1, 0]: replica 1 - l runs state l)
        x = f32(s['x'])
        for t in range(N_LJ):
            far = [0.0]
            start = x

            def on_step(y):
                far[0] = max(far[0], np.linalg.norm(min_image(y - start, s['box']), axis=1).max())
            x, _, _, _, acc = ho.trial(x, s['mass'], KB * temps[l], ho.lj(osys, lambdas[l]), g[t], u[t], dt, N_LJ,
                                       on_step=on_step)
            if not acc:
                moved_in_rejected.append(far[0])
    assert max(moved_in_rejected) > 2 * HALF_OUT, moved_in_rejected
    a = run_lj(monkeypatch, N, cl=cl, env=SKINS, dts=(dt, dt))
    b = run_lj(monkeypatch, N, cl=cl, sort=False, env=SKINS, dts=(dt, dt))
    monkeypatch.delenv('RX_NO_SORT')
    c = run_lj(monkeypatch, N, cl=other, env=SKINS, dts=(dt, dt))
    for o in (b, c):
        assert np.array_equal(o[0], a[0]) and np.array_equal(o[1], a[1])
        assert all(np.array_equal(p, q) for p, q in zip(o[2], a[2])) and all(np.array_equal(p, q) for p, q in zip(o[3], a[3]))


# ---- E. several launches, the range rule, NaN, the retry, the refusal ------------------------------------------------------
def test_three_launches_of_the_fluid_and_a_molecule(monkeypatch):
    """The statistics accumulate over launches, the energies are those of each launch's last trial, and the oracle runs on
    from its own end state (wrapped into the box between launches for the fluid, as the device wraps it)."""
    s = lj_setup(N=256, n_alch=6, seed=256)
    K, lambdas, temps = 2, np.array([1.0, 0.4]), np.array([300.0, 330.0])
    eng = lj_engine(s, K, lambdas, temps, DT_LJ, N_LJ)
    osys = oracle_system(s)
    x0 = np.stack([s['x']] * K)
    eng.set_positions(x0); eng.set_velocities(np.zeros_like(x0))
    its = (IT, IT + 1, IT + 2)
    for q in range(3):
        eng.propagate(SEED, its[q])
        xg, vg = eng.get_positions(), eng.get_velocities()
        per = [check_replica(eng, k, x0[k], s['mass'], KB * temps[k], ho.lj(osys, lambdas[k]), DT_LJ, N_LJ, xg, vg,
                             s['box'], iterations=its[:q + 1]) for k in range(K)]
    assert_exercised(per, N_LJ)
    eng.close()
    system, x = MOLECULES['mixture']()
    run_molecule(system, x, *MOLECULE_CASES['mixture'], launches=3)


def test_range_rule_rejects_every_trial_and_keeps_the_bits(monkeypatch):
    """A per-atom term at or above 2^26 kJ/mol is outside the fixed-point sum: every trial is rejected and the positions
    come back bit for bit, while a healthy replica of the same launch matches the oracle."""
    N, n_steps, dt = 4, 3, 0.05
    Ks, x0s, temps = np.array([1000.0]), np.zeros((1, 3)), np.array([300.0])
    eng = harmonic_engine(2, N, Ks, x0s, temps, dt, n_steps)
    x0 = f32(np.random.default_rng(3).normal(scale=0.05, size=(2, N, 3)))
    x0[0, 1] = [400.0, 0.0, 0.0]          # K/2 x^2 = 8e7 kJ/mol > 2^26 on one atom
    assert 0.5 * Ks[0] * 400.0 ** 2 > 2 ** 26
    eng.set_positions(x0); eng.set_velocities(np.zeros_like(x0))
    eng.set_replica_states(np.zeros(2, np.int64))
    eng.propagate(SEED, IT)
    xg, vg = eng.get_positions(), eng.get_velocities()
    acc, n = eng.get_hmc_statistics()
    assert (acc[0], n[0]) == (0, n_steps) and np.array_equal(xg[0], x0[0])
    check_replica(eng, 1, x0[1], np.full(N, 39.948), KB * 300.0, ho.harmonic(Ks[0], x0s[0]), dt, n_steps, xg, vg,
                  tol_x=2e-5, tol_v=2e-4)
    eng.close()
    # the fluid: an overlapping pair (0.05 nm apart) in replica 0
    s = lj_setup(N=256, n_alch=6, seed=256)
    eng = lj_engine(s, 2, np.array([1.0, 1.0]), np.array([300.0, 300.0]), 0.002, 3)
    x0 = np.stack([s['x']] * 2)
    x0[0, 1] = f32(x0[0, 0] + np.array([0.05, 0.0, 0.0]))
    eng.set_positions(x0); eng.set_velocities(np.zeros_like(x0))
    eng.propagate(SEED, IT)
    xg, vg = eng.get_positions(), eng.get_velocities()
    acc, n = eng.get_hmc_statistics()
    assert (acc[0], n[0]) == (0, 3) and np.array_equal(xg[0], x0[0])
    check_replica(eng, 1, x0[1], s['mass'], KB * 300.0, ho.lj(oracle_system(s), 1.0), 0.002, 3, xg, vg, s['box'])
    eng.close()


def nan_launch(eng, K, x0, bad):
    x = x0.copy()
    x[bad, 3] = np.nan
    eng.set_positions(x); eng.set_velocities(np.zeros_like(x))
    eng.set_hmc_statistics(np.zeros(K, np.int64), np.zeros(K, np.int64))
    with pytest.raises(EngineError) as e:
        eng.propagate(SEED, IT)
    assert e.value.code == _lib.RX_ERR_NAN and list(np.nonzero(e.value.nan_flags)[0]) == [bad]
    xg, vg = eng.get_positions(), eng.get_velocities()
    acc, n = eng.get_hmc_statistics()
    assert n[bad] == 0 and acc[bad] == 0
    return xg, vg, acc, n


def after_retry(eng, bad, xg, vg, acc, n):
    try:
        eng.propagate_retry(SEED, IT)
    except EngineError as e:   # the failed replica restarts from its NaN positions and fails again
        assert list(np.nonzero(e.nan_flags)[0]) == [bad]
    keep = np.arange(len(n)) != bad
    x2, v2 = eng.get_positions(), eng.get_velocities()
    acc2, n2 = eng.get_hmc_statistics()
    assert np.array_equal(x2[keep], xg[keep]) and np.array_equal(v2[keep], vg[keep])
    assert np.array_equal(acc2[keep], acc[keep]) and np.array_equal(n2[keep], n[keep])


def test_nan_replica_is_not_counted_and_the_retry_keeps_the_others():
    """NaN positions in replica 2 of 4: only its flag, its trials not counted, the others counted once and equal to the
    oracle; propagate_retry leaves the healthy replicas' bits and counts as they were."""
    K, bad = 4, 2
    s = lj_setup(N=256, n_alch=6, seed=256)
    lambdas, temps = np.linspace(1.0, 0.4, K), np.linspace(300.0, 330.0, K)
    eng = lj_engine(s, K, lambdas, temps, DT_LJ, N_LJ)
    osys = oracle_system(s)
    x0 = np.stack([s['x']] * K)
    xg, vg, acc, n = nan_launch(eng, K, x0, bad)
    for k in range(K):
        if k != bad:
            check_replica(eng, k, x0[k], s['mass'], KB * temps[k], ho.lj(osys, lambdas[k]), DT_LJ, N_LJ, xg, vg, s['box'])
    after_retry(eng, bad, xg, vg, acc, n)
    eng.close()
    system, x = MOLECULES['mixture']()
    n_steps, dt = MOLECULE_CASES['mixture']
    m = oracle_molecule(system)
    temps = np.linspace(300.0, 450.0, K)
    e = gpu_engine(_lib.RX_SYSTEM_MOLECULE, K, K, system.n_particles)
    e.set_molecule(system, constraint_tolerance=1e-10)
    e.set_states(temps, np.ones(K))
    e.set_hmc_integrator(dt, n_steps)
    x0 = np.concatenate([molecule_start(system, x, m, 2)] * 2)
    xg, vg, acc, n = nan_launch(e, K, x0, bad)
    for k in range(K):
        if k != bad:
            check_replica(e, k, x0[k], m.mass, KB * temps[k], ho.molecule(m), dt, n_steps, xg, vg, tol_x=2e-5, tol_v=1e-2,
                          cons=m.cons)
    after_retry(e, bad, xg, vg, acc, n)
    e.close()


def test_per_state_hmc_moves_on_a_molecule_are_refused():
    system, x = MOLECULES['mixture']()
    e = gpu_engine(_lib.RX_SYSTEM_MOLECULE, 2, 2, system.n_particles)
    e.set_molecule(system, constraint_tolerance=1e-10)
    e.set_states(np.array([300.0, 450.0]), np.ones(2))
    e.set_hmc_integrator(0.002, 4)
    e.set_state_hmc_integrator(1, 0.001, 4)
    e.set_positions(np.stack([x] * 2)); e.set_velocities(np.zeros((2,) + x.shape))
    with pytest.raises(EngineError) as err:
        e.propagate(SEED, IT)
    assert err.value.code == _lib.RX_ERR_UNSUPPORTED
    e.close()


# ---- F. the stationary distribution of a flexible bond ---------------------------------------------------------------------
def test_flexible_bond_samples_boltzmann_exactly():
    """<(r - r0)^2> of 128 independent chains at omega dt = 1 (omega = sqrt(k / mu)) equals the quadrature within 5 SEM +
    1 %; the molecule kernel's accept rule (f64 mol_energy, warp 0's decision shared through shared memory) is what makes
    it exact at this step.  test_hmc_variants_host.py checks the quadrature and that the same bound fails without the
    accept test."""
    system, x = flexible_hcl()
    K, T, n_steps, n_launches, dt = BOND_STATS
    kT = KB * T
    e = gpu_engine(_lib.RX_SYSTEM_MOLECULE, K, 1, 2)
    e.set_molecule(system, constraint_tolerance=1e-10)
    e.set_states(np.array([T]), np.ones(1))
    e.set_hmc_integrator(dt, n_steps)
    e.set_positions(np.stack([x] * K)); e.set_velocities(np.zeros((K, 2, 3)))
    e.set_replica_states(np.zeros(K, np.int64))
    per = []
    for it in range(n_launches):
        e.propagate(SEED, it)
        if it >= n_launches // 10:
            y = e.get_positions()
            per.append((np.linalg.norm(y[:, 0] - y[:, 1], axis=1) - BOND_R0) ** 2)
    acc, n = e.get_hmc_statistics()
    e.close()
    assert 0.5 < acc.sum() / n.sum() < 0.98   # (0.92 measured: the one vibration at omega dt = 1, the rotation nearly exact)
    ref = bond_msd_quadrature(kT)
    r = np.mean(per, axis=0) / ref
    assert abs(r.mean() - 1.0) < 5 * r.std(ddof=1) / np.sqrt(K) + 0.01, (r.mean(), r.std(ddof=1) / np.sqrt(K))


# ---- G. the sampler on a molecule ------------------------------------------------------------------------------------------
def toluene_sampler(tmp, seed=5):
    t = testsystems.TolueneImplicit()
    ref = states.ThermodynamicState(t.system, 300.0 * unit.kelvin)
    move = mcmc.SequenceMove([mcmc.MCDisplacementMove(atom_subset=None),
                              mcmc.HMCMove(timestep=1.0 * unit.femtosecond, n_steps=5)])
    s = multistate.ParallelTemperingSampler(mcmc_moves=move, number_of_iterations=6, seed=seed)
    storage = None if tmp is None else multistate.MultiStateReporter(os.path.join(str(tmp), 'run.nc'), checkpoint_interval=1)
    s.create(ref, states.SamplerState(t.positions), storage, min_temperature=300.0 * unit.kelvin,
             max_temperature=450.0 * unit.kelvin, n_temperatures=4)
    return s


def test_sampler_runs_hmc_on_toluene_fused_phase_by_phase_and_resumed(tmp_path):
    a, b = toluene_sampler(None), toluene_sampler(None)
    a.run(3)
    b._compute_energies()
    b._engine.run_iterations(3, 'swap-all', b._seed, 1)
    for f in ('get_replica_states', 'get_energies', 'get_positions', 'get_velocities', 'get_hmc_statistics'):
        ra, rb = getattr(a._engine, f)(), getattr(b._engine, f)()
        assert all(np.array_equal(p, q) for p, q in zip(ra, rb)) if isinstance(ra, tuple) else np.array_equal(ra, rb), f
    acc, n = a._engine.get_hmc_statistics()
    assert list(n) == [3 * 5] * 4 and 0 < acc.sum() <= n.sum()
    full = toluene_sampler(tmp_path / 'a')
    full.run(6)
    c = toluene_sampler(tmp_path / 'b')
    c.run(4)
    c._reporter.close()
    del c
    d = multistate.ParallelTemperingSampler.from_storage(multistate.MultiStateReporter(os.path.join(str(tmp_path / 'b'), 'run.nc')))
    assert d.iteration == 4
    d.run(2)
    assert np.array_equal(full._engine.get_positions(), d._engine.get_positions())
    assert np.array_equal(full._replica_thermodynamic_states, d._replica_thermodynamic_states)
