"""Shared builders for the tests: the alchemical LJ fluid of SURVEY.md section 8(d) in md units, small molecules in
vacuum (alkanes, rigid waters, a torsion probe, a mixture of cluster shapes, ions), the numpy
restatement of the device's Philox noise, and a guarded GPU-engine import."""
import os
import numpy as np

KB = 8.31446261815324e-3   # kJ/mol/K

# testsystems.LennardJonesFluid defaults (/root/reference/openmmtools/testsystems.py:1898-1909)
SIGMA = 0.34
EPSILON = 0.238 * 4.184
MASS = 39.9


# Three atom types (sigma nm, epsilon kJ/mol, mass amu) for the mixed systems: a mass ratio of about 11 and a sigma range
# wide enough that taking sigma, epsilon or 1/m from the wrong atom moves forces by tens of percent.
THREE_TYPES = ((0.30, 0.5, 12.0), (SIGMA, EPSILON, MASS), (0.40, 1.6, 131.3))
RECT = (1.0, 1.35, 0.8)


def scattered_alch(N, cluster=4):
    """Alchemical atoms spread over the whole index range: atom 0, atoms N/3 and N/2, the last atom of every block of a
    4-block cluster, an atom in the last warp, and atom N-1."""
    nq = -(-N // cluster)
    idx = {0, N // 3, N // 2, N - 1, max(N - 17, 0)}
    idx |= {min((q + 1) * nq, N) - 1 for q in range(cluster)}    # the last atom of every block of a 4-block cluster
    return np.array(sorted(i for i in idx if i < N))


def lj_setup(N=512, n_alch=10, reduced_density=0.05, seed=1, jitter=0.05, types=None, box_ratio=(1.0, 1.0, 1.0),
             alch=None, box=None):
    """Box, parameters and a jittered sub-random configuration (float32-rounded, as the reference stores it).

    types      None (every atom sigma = SIGMA, eps = EPSILON, m = MASS) or [(sigma, eps, mass), ...], dealt to the
               atoms in a seeded shuffle so that every warp and every cluster block holds a mix;
    box_ratio  edges L * r_d at the density of the cube of edge L;
    alch       explicit alchemical atom indices (default: atoms 0 .. n_alch-1);
    box        explicit edges (for N too small to fill a box of two cut-offs at the density).
    s['box'] holds the three edges, s['L'] the edge of a cubic box (None otherwise)."""
    L = (N * SIGMA ** 3 / reduced_density) ** (1.0 / 3.0)
    r = np.asarray(box_ratio, np.float64)
    edges = np.asarray(box, np.float64) if box is not None else L * r / np.prod(r) ** (1.0 / 3.0)
    rc = 3.0 * SIGMA
    rs = rc - SIGMA
    if types is None:
        sigma, eps, mass = np.full(N, SIGMA), np.full(N, EPSILON), np.full(N, MASS)
    else:
        t = np.random.default_rng(10_000 + seed).permutation(np.arange(N) % len(types))
        sigma, eps, mass = (np.array([types[q][c] for q in t]) for c in range(3))
    rng = np.random.default_rng(seed)
    rng.random((N, 3))   # (a draw earlier versions used; kept so that the configurations stay the same)
    # push apart overlapping atoms crudely: reject points closer than 0.9 sigma_ij.  Candidates are drawn in blocks
    # (the same stream as one rng.random(3) per candidate) and each is tested against all accepted points at once.
    pts = np.empty((N, 3))
    n = 0
    while n < N:
        for c in rng.random((max(N - n, 16), 3)) * edges:
            d = c - pts[:n]
            d -= edges * np.round(d / edges)
            lim = (0.9 * 0.5 * (sigma[n] + sigma[:n])) ** 2
            if not np.any(np.einsum('ij,ij->i', d, d) < lim):
                pts[n] = c
                n += 1
                if n == N:
                    break
    x = pts.astype(np.float32).astype(np.float64)
    mask = np.zeros(N, np.uint8)
    mask[np.arange(min(n_alch, N)) if alch is None else np.asarray(alch, int)] = 1
    cubic = bool(np.all(edges == edges[0]))
    return dict(N=N, L=float(edges[0]) if cubic else None, box=edges, rc=rc, rs=rs, x=x, alch=mask, sigma=sigma,
                eps=eps, mass=mass)


# ---- small molecules in vacuum (system.System of kind MOLECULE) ---------------------------------------------------------
# GAFF / TIP3P-like parameters in md units.  Bonds: (K kJ/mol/nm^2 in OpenMM's 1/2 K (r - r0)^2 convention, r0 nm); angles:
# (K kJ/mol/rad^2, theta0).  Per element: mass, sigma, epsilon.
_ELEM = {'C': (12.01, 0.339967, 0.457730), 'H': (1.008, 0.264953, 0.065689), 'N': (14.01, 0.325000, 0.711280),
         'O': (15.9994, 0.315075, 0.635968), 'Cl': (35.45, 0.440000, 0.418400), 'Na': (22.99, 0.243928, 0.365846)}
_BOND = {('C', 'C'): (259408.0, 0.1526), ('C', 'H'): (284512.0, 0.1090), ('C', 'N'): (307105.6, 0.1471),
         ('H', 'N'): (363171.2, 0.1010), ('Cl', 'H'): (250000.0, 0.1275)}
_TET = np.arccos(-1.0 / 3.0)
_ANGLE = {'CCC': (334.72, _TET), 'CCH': (418.40, _TET), 'HCH': (292.88, _TET), 'CNH': (418.40, _TET),
          'HNH': (292.88, np.deg2rad(106.4)), 'HCN': (418.40, _TET)}
# Periodic torsions (n, phase, k): C-C-C-C carries n = 1, 2, 3 with an asymmetric phase and a negative k, so that a sign
# error in the dihedral or in k does not cancel.  With one term per torsion each kind keeps its n = 3 term.
_TORS3 = {'CCCC': ((1, 0.3, 0.80), (2, np.pi, -0.25), (3, 0.0, 0.75)),
          'HCCH': ((1, 0.0, 0.10), (2, np.pi, 0.20), (3, 0.3, 0.63)),
          'CCCH': ((1, 0.0, 0.10), (2, np.pi, 0.20), (3, 0.0, 0.65)),
          'HCNH': ((3, 0.0, 0.70),)}
_TIP3P = dict(rOH=0.09572, rHH=0.15139, qO=-0.834, qH=0.417)


def _rot(rng):
    q = rng.normal(size=4)
    a, b, c, d = q / np.linalg.norm(q)
    return np.array([[a*a+b*b-c*c-d*d, 2*(b*c-a*d), 2*(b*d+a*c)], [2*(b*c+a*d), a*a-b*b+c*c-d*d, 2*(c*d-a*b)],
                     [2*(b*d-a*c), 2*(c*d+a*b), a*a-b*b-c*c+d*d]])


def _mol_system(el, x, charge, bonds, constraints_mode, torsions_per=1, extra_constraints=(), rigid=(), remove_cm=True,
                impropers=(), torsion_terms=None, shuffle=None, jitter_seed=0, jitter=0.005):
    """Assemble a System from elements, a bond graph and positions.

    Angles, proper torsions, 1-2/1-3 exclusions and 1-4 exceptions (charge product / 1.2, epsilon / 2) follow from the bond
    graph; `constraints_mode` 'HBonds' turns bonds to hydrogen into constraints (their bond terms dropped, as
    AmberPrmtopFile.createSystem does), 'AllBonds' every bond, None none.  `rigid`: triangles (a, b, c) constrained on all
    three edges with no bonded terms (rigid water).  The positions are jittered and then every constraint is put back at
    its length by walking each constraint tree from its heaviest atom; rigid triangles move as rigid bodies instead."""
    from openmmtools_b200.system import System, MOLECULE
    n = len(el)
    x = np.array(x, np.float64)
    rng = np.random.default_rng(jitter_seed)
    mass = np.array([_ELEM[e][0] for e in el]); sig = np.array([_ELEM[e][1] for e in el]); eps = np.array([_ELEM[e][2] for e in el])
    nbr = [set() for _ in range(n)]
    for i, j in bonds:
        nbr[i].add(j); nbr[j].add(i)
    key = lambda *a: ''.join(el[q] for q in a)
    cons, btab = [], []
    for i, j in bonds:
        K, r0 = _BOND[tuple(sorted((el[i], el[j])))]
        if constraints_mode == 'AllBonds' or (constraints_mode == 'HBonds' and 'H' in (el[i], el[j])):
            cons.append((i, j, r0))
        else:
            btab.append((i, j, K, r0))
    for a, b, c in rigid:
        for i, j in ((a, b), (a, c), (b, c)):
            cons.append((i, j, _TIP3P['rHH'] if el[i] == el[j] == 'H' else _TIP3P['rOH']))
    cons += list(extra_constraints)
    angles = []
    for j in range(n):
        for i in sorted(nbr[j]):
            for k in sorted(nbr[j]):
                if i < k:
                    kk = key(i, j, k) if key(i, j, k) in _ANGLE else key(k, j, i)
                    angles.append((i, j, k) + _ANGLE[kk])
    tors = []
    for j, k in bonds:
        for i in sorted(nbr[j] - {k}):
            for l in sorted(nbr[k] - {j, i}):
                kind = key(i, j, k, l)
                kind = kind if kind in _TORS3 else key(l, k, j, i)
                terms = torsion_terms[kind] if torsion_terms else _TORS3[kind]
                if torsions_per == 1:
                    terms = [t for t in terms if t[0] == 3] or terms[-1:]
                tors += [(i, j, k, l) + tuple(t) for t in terms]
    tors += list(impropers)
    excl, one4 = set(), set()
    for i in range(n):
        for j in nbr[i]:
            excl.add((min(i, j), max(i, j)))
            for k in nbr[j] - {i}:
                excl.add((min(i, k), max(i, k)))
    for a, b, c in rigid:
        excl |= {(min(a, b), max(a, b)), (min(a, c), max(a, c)), (min(b, c), max(b, c))}
    for i in range(n):
        for j in nbr[i]:
            for k in nbr[j] - {i}:
                for l in nbr[k] - {i, j}:
                    p = (min(i, l), max(i, l))
                    if p not in excl:
                        one4.add(p)
    exc = [(i, j, charge[i] * charge[j] / 1.2, 0.5 * (sig[i] + sig[j]), np.sqrt(eps[i] * eps[j]) / 2.0) for i, j in sorted(one4)]
    # jitter, then restore every constraint exactly
    groups = {q for t in rigid for q in t}
    for a, b, c in rigid:
        cen = x[[a, b, c]].mean(0)
        R = _rot(rng) if jitter else np.eye(3)
        x[[a, b, c]] = (x[[a, b, c]] - cen) @ R.T + cen + rng.normal(0, jitter, 3)
    free = [q for q in range(n) if q not in groups]
    x[free] += rng.normal(0, jitter, (len(free), 3))
    cadj = [[] for _ in range(n)]
    for i, j, d in cons:
        if i in groups:
            continue
        cadj[i].append((j, d)); cadj[j].append((i, d))
    seen = set()
    for root in sorted(range(n), key=lambda q: -mass[q]):
        if root in seen or not cadj[root]:
            continue
        seen.add(root)
        stack = [root]
        while stack:
            a = stack.pop()
            for b, d in cadj[a]:
                if b not in seen:
                    u = x[b] - x[a]
                    x[b] = x[a] + d * u / np.linalg.norm(u)
                    seen.add(b); stack.append(b)
    cons = [(int(i), int(j), float(d)) for i, j, d in cons]
    if shuffle is not None:
        el, x, mass, sig, eps, charge, btab, angles, tors, excl, exc, cons = _shuffle(
            shuffle, el, x, mass, sig, eps, np.asarray(charge, float), btab, angles, tors, sorted(excl), exc, cons)
    s = System(MOLECULE, mass)
    s.charge = np.asarray(charge, np.float64); s.sigma = sig; s.epsilon = eps
    s.bonds = np.array(btab, np.float64).reshape(-1, 4)
    s.angles = np.array(angles, np.float64).reshape(-1, 5)
    s.torsions = np.array(tors, np.float64).reshape(-1, 7)
    s.exclusions = np.array(sorted(excl) if shuffle is None else excl, np.int64).reshape(-1, 2)
    s.exceptions = np.array(exc, np.float64).reshape(-1, 5)
    s.constraints = np.array(cons, np.float64).reshape(-1, 3)
    s.remove_cm_motion = remove_cm
    return s, np.ascontiguousarray(x)


def constraint_clusters(cons, n):
    """Connected components of the constraint graph: lists of constraint rows, each in list order."""
    parent = list(range(n))

    def find(a):
        while parent[a] != a:
            a = parent[a]
        return a
    for i, j, _ in cons:
        parent[find(int(i))] = find(int(j))
    out = {}
    for c in cons:
        out.setdefault(find(int(c[0])), []).append(tuple(c))
    return list(out.values())


def _shuffle(seed, el, x, mass, sig, eps, charge, btab, angles, tors, excl, exc, cons):
    """Renumber the atoms (hydrogens first, each group in a seeded random order), write every constraint with i > j, let the
    constraints of different clusters alternate in the list, and swap the ends of some bonds, exclusions and exceptions."""
    rng = np.random.default_rng(seed)
    n = len(el)
    hs = [q for q in range(n) if el[q] == 'H']
    heavy = [q for q in range(n) if el[q] != 'H']
    order = list(rng.permutation(hs)) + list(rng.permutation(heavy))     # order[new] = old
    new = np.empty(n, int)
    new[order] = np.arange(n)
    P = lambda a: int(new[int(a)])
    flip = lambda i, j: (j, i) if rng.random() < 0.5 else (i, j)
    btab = [flip(P(b[0]), P(b[1])) + tuple(b[2:]) for b in btab]
    angles = [(P(a[0]), P(a[1]), P(a[2])) + tuple(a[3:]) for a in angles]
    tors = [tuple(P(t[q]) for q in range(4)) + tuple(t[4:]) for t in tors]
    excl = [flip(P(i), P(j)) for i, j in excl]
    exc = [flip(P(e[0]), P(e[1])) + tuple(e[2:]) for e in exc]
    cl = constraint_clusters([(max(P(i), P(j)), min(P(i), P(j)), d) for i, j, d in cons], n)
    cl = [list(c) for c in cl]
    rng.shuffle(cl)
    for c in cl:
        rng.shuffle(c)
    inter = []
    while any(cl):
        for c in cl:
            if c:
                inter.append(c.pop())
    pick = lambda a: np.asarray(a)[order]
    return ([el[q] for q in order], pick(x), pick(mass), pick(sig), pick(eps), pick(charge), btab, angles, tors, excl, exc,
            inter)


def _alkane_geometry(hcount):
    """A zig-zag carbon chain in the xy plane with tetrahedral hydrogens; hcount[c] hydrogens on carbon c."""
    nc = len(hcount)
    el, x, bonds = [], [], []
    half = 0.5 * _TET
    cpos = [np.array([c * 0.1526 * np.sin(half), (c % 2) * 0.1526 * np.cos(half), 0.0]) for c in range(nc)]
    cidx = []
    for c in range(nc):
        cidx.append(len(el)); el.append('C'); x.append(cpos[c])
        if c:
            bonds.append((cidx[c - 1], cidx[c]))
    for c in range(nc):
        nb = [cpos[q] for q in (c - 1, c + 1) if 0 <= q < nc]
        if not nb:
            dirs = [np.array(v, float) / np.sqrt(3) for v in ((1, 1, 1), (1, -1, -1), (-1, 1, -1), (-1, -1, 1))]
        else:
            u = [(p - cpos[c]) / np.linalg.norm(p - cpos[c]) for p in nb]
            b = -np.sum(u, 0); b /= np.linalg.norm(b)
            if len(u) == 1:       # three hydrogens at the tetrahedral angle to the C-C bond
                e1 = np.cross(u[0], [0, 0, 1.0]); e1 /= np.linalg.norm(e1); e2 = np.cross(u[0], e1)
                dirs = [np.cos(_TET) * u[0] + np.sin(_TET) * (np.cos(t) * e1 + np.sin(t) * e2)
                        for t in (0, 2 * np.pi / 3, 4 * np.pi / 3)]
            else:
                w = np.cross(u[0], u[1]); w /= np.linalg.norm(w)
                dirs = [b * np.cos(0.5 * _TET) + w * np.sin(0.5 * _TET), b * np.cos(0.5 * _TET) - w * np.sin(0.5 * _TET)]
        for h in range(hcount[c]):
            el.append('H'); x.append(cpos[c] + 0.1090 * dirs[h] / np.linalg.norm(dirs[h]))
            bonds.append((cidx[c], len(el) - 1))
    return el, np.array(x), bonds


def _alkane_charges(el, bonds):
    nh = {}
    for i, j in bonds:
        if el[i] == 'C' and el[j] == 'H':
            nh[i] = nh.get(i, 0) + 1
    return np.array([0.06 if e == 'H' else -0.06 * nh.get(q, 0) for q, e in enumerate(el)])


def alkane(n_carbons, terms_per_torsion=1, constraints='HBonds', shuffle=None, seed=0, hydrogens=None):
    """CnH(2n+2) (n_carbons = 10: decane, 32 atoms; 1: methane, one cluster of 4 constraints; 3 with 'AllBonds': propane as
    one cluster of 10 constraints).  `hydrogens`: per-carbon hydrogen counts instead of the saturated chain (fragments).
    Charges -0.06 per attached hydrogen on carbon, +0.06 on hydrogen (neutral); mass ratio C/H 11.9."""
    hc = hydrogens if hydrogens is not None else ([4] if n_carbons == 1 else [3] + [2] * (n_carbons - 2) + [3])
    el, x, bonds = _alkane_geometry(hc)
    return _mol_system(el, x, _alkane_charges(el, bonds), bonds, constraints, torsions_per=terms_per_torsion,
                       shuffle=shuffle, jitter_seed=seed)


def waters(n, ions=0, shuffle=None, seed=0):
    """n rigid TIP3P waters (three constraints over three atoms each: a cycle) on a 0.31 nm grid, random orientations,
    plus `ions` sodium/chloride ions alternating; centre-of-mass motion kept (remove_cm_motion = False)."""
    rOH, rHH = _TIP3P['rOH'], _TIP3P['rHH']
    h = np.sqrt(rOH ** 2 - (rHH / 2) ** 2)
    w = np.array([[0.0, 0.0, 0.0], [rHH / 2, h, 0.0], [-rHH / 2, h, 0.0]])
    g = int(np.ceil((n + ions) ** (1 / 3)))
    sites = [0.31 * np.array([a, b, c], float) for a in range(g) for b in range(g) for c in range(g)][:n + ions]
    el, x, q, rigid = [], [], [], []
    for m in range(n):
        rigid.append((len(el), len(el) + 1, len(el) + 2))
        el += ['O', 'H', 'H']; x += list(w + sites[m]); q += [_TIP3P['qO'], _TIP3P['qH'], _TIP3P['qH']]
    for m in range(ions):
        el.append('Na' if m % 2 == 0 else 'Cl'); x.append(sites[n + m]); q.append(1.0 if m % 2 == 0 else -1.0)
    s, x = _mol_system(el, x, np.array(q), [], None, rigid=rigid, remove_cm=False, shuffle=shuffle, jitter_seed=seed,
                       jitter=0.02)
    hyd = s.masses < 1.1
    s.epsilon[hyd] = 0.0; s.sigma[hyd] = 0.1             # TIP3P hydrogens carry no Lennard-Jones term
    return s, x


def torsion_probe(n, phase, k, phi=np.deg2rad(70.0), shuffle=None):
    """Five atoms: the proper torsion 0-1-2-3 (periodicity n, phase, k) at the IUPAC dihedral `phi` -- j = 0,
    k = 0.15 z, i = 0.1 x, l = (0.1 cos phi, 0.1 sin phi, 0.15) up to a shift -- and an improper 1-3-2-4 centred on atom 2
    (n = 2, phase pi).  Flexible bonds, no charges on the torsion ends."""
    x = np.array([[0.1, 0.0, 0.0], [0.0, 0.0, 0.0], [0.0, 0.0, 0.15], [0.1 * np.cos(phi), 0.1 * np.sin(phi), 0.15],
                  [-0.08, -0.06, 0.21]]) + np.array([0.3, -0.2, 0.1])
    el = ['C', 'C', 'C', 'C', 'H']
    tt = {'CCCC': ((int(n), float(phase), float(k)),), 'CCCH': ((3, 0.0, 0.0),)}
    s, x = _mol_system(el, x, np.array([0.0, 0.1, -0.15, 0.0, 0.05]), [(0, 1), (1, 2), (2, 3), (2, 4)], None,
                       torsions_per=3, impropers=[(1, 3, 2, 4, 2, np.pi, 4.6)], torsion_terms=tt, shuffle=shuffle,
                       jitter=0.0)
    keep = s.torsions[:, 6] != 0.0            # (the C-C-C-H proper carries no energy: dropped)
    s.torsions = s.torsions[keep]
    return s, x


def mixture(shuffle=None, seed=0):
    """Methylamine (clusters of 3 and 2 constraints), methane (4) and HCl (1) in one System, 14 atoms: every cluster size
    of k_propagate_mol<false> at once.  Mass ratio Cl/H 35."""
    el, x, bonds = [], [], []
    # methylamine: C, N, 3 H on C, 2 H on N
    cx, nx = np.zeros(3), np.array([0.1471, 0.0, 0.0])
    el += ['C', 'N']; x += [cx, nx]; bonds.append((0, 1))
    ring = lambda t, a: np.array([np.cos(t), np.sin(t) * np.cos(a), np.sin(t) * np.sin(a)])
    for t in range(3):        # at the tetrahedral angle to C->N (+x)
        el.append('H'); x.append(cx + 0.1090 * ring(_TET, 2 * np.pi * t / 3)); bonds.append((0, len(el) - 1))
    for t in range(2):        # at 110 degrees to N->C (-x)
        d = ring(np.deg2rad(110.0), np.pi / 2 + np.pi * t) * np.array([-1.0, 1.0, 1.0])
        el.append('H'); x.append(nx + 0.1010 * d); bonds.append((1, len(el) - 1))
    # methane at 0.45 nm
    mc = np.array([0.1, 0.45, 0.0]); c0 = len(el)
    el.append('C'); x.append(mc)
    for v in ((1, 1, 1), (1, -1, -1), (-1, 1, -1), (-1, -1, 1)):
        el.append('H'); x.append(mc + 0.1090 * np.array(v, float) / np.sqrt(3)); bonds.append((c0, len(el) - 1))
    # HCl at 0.45 nm the other way
    hc = np.array([0.05, -0.42, 0.1]); h0 = len(el)
    el += ['Cl', 'H']; x += [hc, hc + np.array([0.0, -0.1275, 0.0])]; bonds.append((h0, h0 + 1))
    q = np.array([0.0, -0.90, 0.06, 0.06, 0.06, 0.36, 0.36, -0.24, 0.06, 0.06, 0.06, 0.06, -0.20, 0.20])
    return _mol_system(el, np.array(x), q, bonds, 'HBonds', shuffle=shuffle, jitter_seed=seed)


def ion(n_ions=1):
    """Sodium ions in vacuum (n = 1: no interaction at all); remove_cm_motion = False."""
    x = np.array([[0.1, 0.2, 0.3], [0.45, 0.2, 0.3]])[:n_ions]
    return _mol_system(['Na'] * n_ions, x, np.ones(n_ions), [], None, remove_cm=False, jitter=0.0)


def diatomic():
    """HCl with its bond constrained: n = 2, one cluster of one constraint."""
    return _mol_system(['Cl', 'H'], np.array([[0.0, 0.0, 0.0], [0.1275, 0.0, 0.0]]), np.array([-0.2, 0.2]), [(0, 1)],
                       'HBonds', jitter=0.003)


def wrap(x, box):
    return x - box * np.floor(x / box)


def min_image(d, box):
    return d - box * np.round(d / box)


def oracle_system(s, annihilate=False, alpha=0.5, a=1.0, b=1.0, c=6.0, use_switch=True):
    from oracle import oracle
    return oracle.LJSystem(s['sigma'], s['eps'], s['mass'], s['alch'], tuple(s['box']), s['rc'], s['rs'],
                           use_switch=use_switch, alpha=alpha, a=a, b=b, c=c, annihilate_sterics=annihilate)


def gpu_engine(*args, **kw):
    from openmmtools_b200._engine import Engine
    return Engine(*args, **kw)


# ---- Philox4x32-10 + Box-Muller exactly as openmmtools_b200/csrc/rx_dynamics.cu -------------------------
def philox4x32_10(ctr, key):
    """ctr: uint32 array [..., 4]; key: (k0, k1). Vectorised."""
    c = [ctr[..., i].astype(np.uint64) for i in range(4)]
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
    mask = np.uint64(0xFFFFFFFF)
    for _ in range(10):
        p0 = M0 * c[0]
        p1 = M1 * c[2]
        n0 = ((p1 >> np.uint64(32)) ^ c[1] ^ k0) & mask
        n1 = p1 & mask
        n2 = ((p0 >> np.uint64(32)) ^ c[3] ^ k1) & mask
        n3 = p0 & mask
        c = [n0, n1, n2, n3]
        k0 = (k0 + np.uint64(0x9E3779B9)) & mask
        k1 = (k1 + np.uint64(0xBB67AE85)) & mask
    return np.stack(c, axis=-1).astype(np.uint32)


def philox_normal3(r):
    u = ((r >> 8).astype(np.float64) + 0.5) / 16777216.0
    ra = np.sqrt(-2.0 * np.log(u[..., 0]))
    rb = np.sqrt(-2.0 * np.log(u[..., 2]))
    return np.stack([ra * np.cos(2 * np.pi * u[..., 1]), ra * np.sin(2 * np.pi * u[..., 1]),
                     rb * np.cos(2 * np.pi * u[..., 3])], axis=-1)


def device_noise(seed, iteration, replica, N, n_osteps):
    """Standard normals the device uses for replica `replica`: [n_osteps, N, 3]."""
    key = (seed & 0xFFFFFFFF, ((seed >> 32) ^ (iteration >> 32)) & 0xFFFFFFFF)
    ctr = np.zeros((n_osteps, N, 4), np.uint32)
    ctr[..., 0] = np.arange(N)[None, :]
    ctr[..., 1] = np.arange(n_osteps)[:, None]
    ctr[..., 2] = replica
    ctr[..., 3] = iteration & 0xFFFFFFFF
    return philox_normal3(philox4x32_10(ctr, key))


def device_reassign_noise(seed, iteration, replica, N):
    key = (seed & 0xFFFFFFFF, ((seed >> 32) ^ (iteration >> 32)) & 0xFFFFFFFF)
    ctr = np.zeros((N, 4), np.uint32)
    ctr[:, 0] = np.arange(N); ctr[:, 1] = 0x80000000; ctr[:, 2] = replica; ctr[:, 3] = iteration & 0xFFFFFFFF
    return philox_normal3(philox4x32_10(ctr, key))


def device_randomize_noise(seed, replica, N, stream=0):
    """Standard normals of rx_randomize_velocities for replica `replica`: [N, 3]."""
    key = (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    ctr = np.zeros((N, 4), np.uint32)
    ctr[:, 0] = np.arange(N); ctr[:, 1] = 0xC0000000; ctr[:, 2] = replica; ctr[:, 3] = stream & 0xFFFFFFFF
    return philox_normal3(philox4x32_10(ctr, key))
