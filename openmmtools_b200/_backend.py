"""Glue between the reference-shaped Python objects and the CUDA engine (product code; never imports oracle/).

* :func:`engine_tables` turns a list of compatible thermodynamic states into the engine's per-state table
  (temperature, lambda_sterics, energy offset, HO parameters) -- the role of
  ``ThermodynamicState.apply_to_context`` + ``GlobalParameterState.apply_to_context``
  (/root/reference/openmmtools/states.py:1183-1233,3549-3579).
* :func:`lj_dispersion_correction` / :func:`alchemical_dispersion_correction` restate OpenMM's long-range
  corrections (SURVEY.md Appendix A) as per-state energy offsets.
* :func:`build_engine` creates and fills an :class:`Engine` for a set of replicas.
"""
import numpy as np
from . import _lib
from ._engine import Engine
from .system import MOLECULE, LJ, HARMONIC

_GL_X, _GL_W = np.polynomial.legendre.leggauss(64)


def _integrate(f, a, b):
    c, h = 0.5 * (a + b), 0.5 * (b - a)
    return h * np.sum(_GL_W * f(c + h * _GL_X))


def _switch(r, rs, rc):
    t = np.clip((r - rs) / (rc - rs), 0.0, 1.0)
    return 1.0 + t ** 3 * (-10.0 + t * (15.0 - 6.0 * t))


def _classes(sigma, eps):
    """Particle classes by (sigma, epsilon) with their multiplicities."""
    keys = {}
    for s, e in zip(sigma, eps):
        keys[(float(s), float(e))] = keys.get((float(s), float(e)), 0) + 1
    return list(keys.items())


def lj_dispersion_correction(system):
    """NonbondedForce dispersion correction (kJ/mol) for the box volume; alchemical atoms count with eps = 0
    (alchemy.py:1909).  E = 8 pi N^2/V <eps sig^12/(9 rc^9) - eps sig^6/(3 rc^3) + eps I_sw> over N(N+1)/2 class
    pairs, I_sw = int_{rs}^{rc} r^2 [(sig/r)^12 - (sig/r)^6] (1 - S(r)) dr."""
    if system.kind != LJ or not system.use_dispersion_correction:
        return 0.0
    N = system.n_particles
    eps = np.array(system.epsilon, dtype=np.float64)
    if system.alchemical_atoms:
        eps[list(system.alchemical_atoms)] = 0.0
    cls = _classes(system.sigma, eps)
    rc, rs = system.cutoff, system.switching_distance
    s1 = s2 = s3 = 0.0
    for a in range(len(cls)):
        for b in range(a, len(cls)):
            (sa, ea), na = cls[a]
            (sb, eb), nb = cls[b]
            count = 0.5 * na * (na + 1) if a == b else float(na * nb)
            sig, e = 0.5 * (sa + sb), np.sqrt(ea * eb)
            s1 += count * e * sig ** 12
            s2 += count * e * sig ** 6
            if system.use_switching_function and e != 0.0:
                s3 += count * e * _integrate(
                    lambda r: r * r * ((sig / r) ** 12 - (sig / r) ** 6) * (1.0 - _switch(r, rs, rc)), rs, rc)
    npairs = 0.5 * N * (N + 1)
    V = abs(np.linalg.det(system.box_vectors))
    return 8.0 * N * N * np.pi * (s1 / npairs / (9 * rc ** 9) - s2 / npairs / (3 * rc ** 3) + s3 / npairs) / V


def _softcore(r, sig, eps, lam, alpha, a, b, c):
    x = (alpha * (1.0 - lam) ** b + (r / sig) ** c) ** (-6.0 / c)
    return lam ** a * 4.0 * eps * x * (x - 1.0)


def alchemical_dispersion_correction(system, lambda_sterics, lambda_sterics_2=1.0):
    """CustomNonbondedForce long-range correction of the two soft-core forces (SURVEY.md Appendix A): for each
    class pair, count(pairs in the interaction group) * [int_rc^inf r^2 U dr + int_rs^rc r^2 U (1-S) dr], summed,
    divided by N(N+1)/2 and multiplied by 2 pi N^2 / V.  Depends on lambda (the cost the reference warns about,
    alchemy.py:535-540).  With two alchemical regions the two forces of each region (environment = the atoms of
    neither region, lambda_sterics of region 1, lambda_sterics_2 of region 2) are summed; no force covers the pairs
    across the regions."""
    if system.kind != LJ or not system.is_alchemical or not system.alchemical_dispersion_correction:
        return 0.0
    if getattr(system, 'alchemical_regions', None) is None:
        return _region_dispersion_correction(system, system.alchemical_mask().astype(bool),
                                             ~system.alchemical_mask().astype(bool), lambda_sterics, system.annihilate_sterics)
    ids = system.alchemical_region_ids()
    return sum(_region_dispersion_correction(system, ids == r + 1, ids == 0, lam, annihilate)
               for r, (lam, (_, _, annihilate)) in enumerate(zip((lambda_sterics, lambda_sterics_2), system.alchemical_regions)))


def _region_dispersion_correction(system, mask, env, lambda_sterics, annihilate_sterics):
    """The corrections of one region's environment x region (`mask` x `env`) and region x region forces."""
    N = system.n_particles
    sig, eps = np.asarray(system.sigma), np.asarray(system.epsilon)
    rc, rs = system.cutoff, system.switching_distance
    alpha, a, b, c = system.softcore_alpha, system.softcore_a, system.softcore_b, system.softcore_c

    def integral(sg, e, lam):
        if e == 0.0:
            return 0.0
        f = lambda r: _softcore(r, sg, e, lam, alpha, a, b, c)
        tail = _integrate(lambda t: f(1.0 / np.maximum(t, 1e-300)) / np.maximum(t, 1e-300) ** 4 * (t > 0), 0.0, 1.0 / rc)
        sw = 0.0
        if system.use_switching_function:
            sw = _integrate(lambda r: r * r * f(r) * (1.0 - _switch(r, rs, rc)), rs, rc)
        return tail + sw

    total = 0.0
    ca, ce = _classes(sig[mask], eps[mask]), _classes(sig[env], eps[env])
    # na_sterics: environment x alchemical (alchemy.py:1915)
    for (sa, ea), na in ca:
        for (se, ee), ne in ce:
            total += na * ne * integral(0.5 * (sa + se), np.sqrt(ea * ee), lambda_sterics)
    # aa_sterics: alchemical x alchemical, each unordered pair once, lambda fixed to 1 unless annihilating (:1919)
    lam_aa = lambda_sterics if annihilate_sterics else 1.0
    for i in range(len(ca)):
        for j in range(i, len(ca)):
            (si, ei), ni = ca[i]
            (sj, ej), nj = ca[j]
            count = 0.5 * ni * (ni - 1) if i == j else float(ni * nj)
            total += count * integral(0.5 * (si + sj), np.sqrt(ei * ej), lam_aa)
    V = abs(np.linalg.det(system.box_vectors))
    return 2.0 * np.pi * N * N * (total / (0.5 * N * (N + 1))) / V


def check_compatible(thermodynamic_states):
    h0 = thermodynamic_states[0]._standard_system_hash
    sys0 = thermodynamic_states[0]._standard_system
    npt = thermodynamic_states[0].pressure is not None
    scale = barostat_scale(thermodynamic_states)
    for s in thermodynamic_states[1:]:
        if (s.pressure is not None) != npt or getattr(s, '_barostat_scale', None) != scale:
            from .states import ThermodynamicsError
            raise ThermodynamicsError(ThermodynamicsError.INCOMPATIBLE_ENSEMBLE)
        if s._standard_system_hash != h0:
            so = s._standard_system
            # harmonic oscillators may differ in K/x0/U0 (global parameters in the reference)
            if not (so.kind == HARMONIC and sys0.kind == HARMONIC and np.array_equal(so.masses, sys0.masses)):
                raise NotImplementedError(
                    'all thermodynamic states must share one system (differing only in temperature, lambdas or '
                    'harmonic-oscillator parameters): the engine keeps one resident parameter set')
    return sys0


def barostat_scale(thermodynamic_states):
    """The scaled axes (x, y, z) of the states' anisotropic barostat, or None (isotropic or NVT)."""
    return getattr(thermodynamic_states[0], '_barostat_scale', None)


def engine_tables(thermodynamic_states):
    """Per-state arrays for Engine.set_states."""
    sys0 = check_compatible(thermodynamic_states)
    M = len(thermodynamic_states)
    T = np.zeros(M); lam = np.ones(M); lam_e = np.ones(M); off = np.zeros(M); hoK = np.zeros(M); hox0 = np.zeros((M, 3))
    two = sys0.kind == LJ and sys0.alchemical_regions is not None
    lam2 = np.ones(M) if two else None
    base_lrc = lj_dispersion_correction(sys0) if sys0.kind == LJ else 0.0
    cache = {}
    for l, s in enumerate(thermodynamic_states):
        p = s._engine_parameters()
        T[l] = p['temperature']
        if two:
            lam[l], lam2[l] = region_lambdas(sys0, p)
            if (lam[l], lam2[l]) not in cache:
                cache[lam[l], lam2[l]] = alchemical_dispersion_correction(sys0, lam[l], lam2[l])
            off[l] = base_lrc + cache[lam[l], lam2[l]]
        elif sys0.kind == LJ:
            lam[l] = p['lambda_sterics'] if sys0.is_alchemical else 1.0
            if lam[l] not in cache:
                cache[lam[l]] = alchemical_dispersion_correction(sys0, lam[l])
            off[l] = base_lrc + cache[lam[l]]
        elif sys0.kind == MOLECULE:
            if sys0.is_alchemical:   # (other molecules' states differ in temperature only)
                lam[l], lam_e[l] = p['lambda_sterics'], p['lambda_electrostatics']
        else:
            so = s._standard_system
            hoK[l] = so.ho_K
            hox0[l] = so.ho_x0
            off[l] = so.ho_U0
    tab = dict(temperature=T, lambda_sterics=lam, energy_offset=off, ho_K=hoK, ho_x0=hox0)
    if sys0.kind == MOLECULE and sys0.is_alchemical:
        tab['lambda_electrostatics'] = lam_e
    if two:
        tab['lambda_sterics_2'] = lam2
    return sys0, tab


def region_lambdas(system, parameters):
    """(lambda of region 1, lambda of region 2) of a two-region system from a state's _engine_parameters()."""
    return tuple(float(parameters.get(n, system.global_parameters.get(n, 1.0))) for n in system.lambda_sterics_names())


def pressure_tables(thermodynamic_states):
    """NPT states: (pressure [M] in kJ/mol/nm^3, dispersion coefficients c_l [M] in kJ/mol nm^3), or None for NVT.

    Both long-range corrections are proportional to 1/V, so c_l is the state's correction at the system's volume times
    that volume; the engine adds c_l / V_k for replica k (and the per-state offset then carries no correction)."""
    if thermodynamic_states[0].pressure is None:
        return None
    sys0 = check_compatible(thermodynamic_states)
    V0 = abs(np.linalg.det(sys0.box_vectors))
    base = lj_dispersion_correction(sys0)
    p = np.array([s._pressure_md for s in thermodynamic_states])
    cache = {}
    c = np.zeros(len(thermodynamic_states))
    for l, s in enumerate(thermodynamic_states):
        if sys0.alchemical_regions is not None:
            lam = region_lambdas(sys0, s._engine_parameters())
        else:
            lam = (s._engine_parameters()['lambda_sterics'] if sys0.is_alchemical else 1.0,)
        if lam not in cache:
            cache[lam] = (base + alchemical_dispersion_correction(sys0, *lam)) * V0
        c[l] = cache[lam]
    return p, c


def box_edges(sampler_states):
    """(K, 3) edges of the sampler states' rectangular boxes."""
    b = np.stack([np.asarray(s._box_vectors, np.float64) for s in sampler_states])
    if not np.allclose(b, np.einsum('kij,ij->kij', b, np.eye(3))):
        raise NotImplementedError('only rectangular periodic boxes are provided')
    return np.einsum('kii->ki', b).copy()


def default_device(context_cache=None):
    import os
    idx = getattr(context_cache, 'device_index', None) if context_cache is not None else None
    if idx is not None:
        return idx
    return int(os.environ.get('LOCAL_RANK', '0')) if 'LOCAL_RANK' in os.environ else 0


def build_engine(thermodynamic_states, n_replicas, device=0, rank=0, world_size=1):
    """Engine with particles and states set (positions/velocities/integrator are up to the caller)."""
    sys0, tab = engine_tables(thermodynamic_states)
    M, N = len(thermodynamic_states), sys0.n_particles
    if sys0.kind == LJ:
        bv = sys0.box_vectors
        if not np.allclose(bv, np.diag(np.diag(bv))):
            raise NotImplementedError('only rectangular periodic boxes are provided')
        eng = Engine(_lib.RX_SYSTEM_LJ_ALCH, n_replicas, M, N, device=device, rank=rank, world_size=world_size,
                     box=tuple(np.diag(bv)), r_cutoff=sys0.cutoff, r_switch=sys0.switching_distance,
                     use_switch=sys0.use_switching_function, annihilate_sterics=sys0.annihilate_sterics,
                     softcore_alpha=sys0.softcore_alpha, softcore_a=sys0.softcore_a, softcore_b=sys0.softcore_b,
                     softcore_c=sys0.softcore_c)
        eng.set_particles(sys0.sigma, sys0.epsilon, sys0.masses, sys0.alchemical_mask())
        if sys0.alchemical_regions is not None:
            eng.set_alchemical_regions(sys0.alchemical_region_ids(), *[a for _, _, a in sys0.alchemical_regions])
    elif sys0.kind == MOLECULE:
        if N > 32:
            raise NotImplementedError('molecules above 32 atoms are not provided (one lane per atom): %d atoms' % N)
        eng = Engine(_lib.RX_SYSTEM_MOLECULE, n_replicas, M, N, device=device, rank=rank, world_size=world_size,
                     softcore_alpha=sys0.softcore_alpha, softcore_a=sys0.softcore_a, softcore_b=sys0.softcore_b,
                     softcore_c=sys0.softcore_c)
        eng.set_molecule(sys0)
    else:
        eng = Engine(_lib.RX_SYSTEM_HARMONIC, n_replicas, M, N, device=device, rank=rank, world_size=world_size)
        eng.set_particles(None, None, sys0.masses, None)
    npt = pressure_tables(thermodynamic_states)
    if npt is not None:
        tab['energy_offset'] = np.zeros(M)   # (the dispersion corrections go to the engine as c_l / V)
    eng.set_states(**tab)
    if npt is not None:
        eng.set_pressures(*npt)
        if barostat_scale(thermodynamic_states) is not None:
            eng.set_anisotropic_barostat(barostat_scale(thermodynamic_states))
    return eng


def reduced_potentials(thermodynamic_states, sampler_state):
    """u_l = beta_l U_l(x) for one configuration (ThermodynamicState.reduced_potential_at_states)."""
    n = thermodynamic_states[0].n_particles
    if sampler_state.n_particles != n:
        from .states import ThermodynamicsError
        raise ThermodynamicsError(ThermodynamicsError.INCOMPATIBLE_SAMPLER_STATE)
    eng = build_engine(list(thermodynamic_states), 1, device=default_device())
    try:
        eng.set_positions(sampler_state._positions[None])
        if thermodynamic_states[0].pressure is not None:
            eng.set_boxes(box_edges([sampler_state]))
        return eng.compute_energies()[0]
    finally:
        eng.close()
