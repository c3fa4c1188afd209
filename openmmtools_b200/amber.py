"""AMBER prmtop / inpcrd reader for the small-molecule systems of the replica-exchange path (AlanineDipeptideVacuum,
/root/reference/openmmtools/testsystems.py:3352-3388, which calls openmm.app.AmberPrmtopFile.createSystem(
implicitSolvent=None, constraints=HBonds, nonbondedCutoff=None)).

What createSystem does with the file -- restated here from the AMBER file-format specification (ambermd.org/FileFormats.php)
and OpenMM's documented conventions, NOT taken from OpenMM's source (which is not available in this environment):
  * units: lengths Angstrom -> nm, energies kcal/mol -> kJ/mol (x 4.184), charges are stored x 18.2223;
  * bonds      E = k (r - r0)^2        -> HarmonicBondForce  1/2 K (r - r0)^2 with K = 2 k (kJ/mol/nm^2);
  * angles     E = k (t - t0)^2        -> HarmonicAngleForce 1/2 K (t - t0)^2 with K = 2 k (kJ/mol/rad^2);
  * dihedrals  E = k (1 + cos(n phi - phase))  -> PeriodicTorsionForce (n = |periodicity|);
    a negative THIRD atom index marks a torsion whose end atoms do not get a 1-4 interaction, a negative FOURTH an improper;
  * Lennard-Jones: per-atom sigma / epsilon from the diagonal A, B coefficients (A = eps rmin^12, B = 2 eps rmin^6,
    rmin_ii = 2 R_i), Lorentz-Berthelot combination; 1-4 pairs: Coulomb / 1.2 (SCEE), LJ epsilon / 2 (SCNB) with the pair's
    own A, B; 1-2 and 1-3 pairs (EXCLUDED_ATOMS_LIST) excluded;
  * constraints=HBonds: every bond that involves a hydrogen becomes a distance constraint at r0 and its bond term is dropped;
  * no cutoff: plain sums over all non-excluded pairs; Coulomb constant 138.935456 kJ nm / (mol e^2);
  * implicitSolvent=OBC1 / OBC2: the generalized Born model of GBSAOBCForce with the file's RADII (Angstrom -> nm) and
    SCREEN factors (RADIUS_SET names the radius set), solute / solvent dielectric 1 / 78.5, the ACE non-polar term
    (2.25936 kJ/mol/nm^2, probe radius 0.14 nm), no salt (see obc_parameters).
"""
import numpy as np

KCAL = 4.184
AMBER_CHARGE = 18.2223


def _sections(text):
    out, name, fmt, buf = {}, None, None, []
    for line in text.splitlines():
        if line.startswith('%FLAG'):
            if name is not None:
                out[name] = (fmt, buf)
            name, fmt, buf = line.split()[1], None, []
        elif line.startswith('%FORMAT'):
            fmt = line[line.index('(') + 1:line.index(')')]
        elif line.startswith('%'):
            continue
        elif name is not None:
            buf.append(line)
    if name is not None:
        out[name] = (fmt, buf)
    return out


def _values(section):
    fmt, lines = section
    f = fmt.upper()
    kind = 'a' if 'A' in f else ('i' if 'I' in f else 'e')
    width = int(f.split('A' if kind == 'a' else ('I' if kind == 'i' else 'E'))[1].split('.')[0])
    vals = []
    for line in lines:
        line = line.rstrip('\n')
        for c in range(0, len(line), width):
            tok = line[c:c + width]
            if tok.strip() == '' and kind != 'a':
                continue
            vals.append(tok if kind == 'a' else (int(tok) if kind == 'i' else float(tok)))
    return vals


def read_prmtop(path):
    """Raw prmtop arrays in md units plus the derived exclusion / 1-4 structure."""
    sec = _sections(open(path).read())
    get = lambda n: _values(sec[n])
    ptr = get('POINTERS')
    natom, ntypes = ptr[0], ptr[1]
    charge = np.array(get('CHARGE')) / AMBER_CHARGE
    mass = np.array(get('MASS'))
    names = [s.strip() for s in get('ATOM_NAME')][:natom]
    type_index = np.array(get('ATOM_TYPE_INDEX')) - 1
    nb_index = np.array(get('NONBONDED_PARM_INDEX')).reshape(ntypes, ntypes) - 1
    acoef, bcoef = np.array(get('LENNARD_JONES_ACOEF')), np.array(get('LENNARD_JONES_BCOEF'))

    def lj_pair(ti, tj):
        """(sigma nm, epsilon kJ/mol) of a type pair from its A, B."""
        a, b = acoef[nb_index[ti, tj]], bcoef[nb_index[ti, tj]]
        if a == 0.0 or b == 0.0:
            return 1.0 * 0.1, 0.0
        rmin = (2.0 * a / b) ** (1.0 / 6.0)
        eps = 0.25 * b * b / a
        return rmin * 0.1 / 2.0 ** (1.0 / 6.0), eps * KCAL

    sigma = np.zeros(natom); epsilon = np.zeros(natom)
    for i in range(natom):
        sigma[i], epsilon[i] = lj_pair(type_index[i], type_index[i])

    bk, br = np.array(get('BOND_FORCE_CONSTANT')), np.array(get('BOND_EQUIL_VALUE'))
    ak, at = np.array(get('ANGLE_FORCE_CONSTANT')), np.array(get('ANGLE_EQUIL_VALUE'))
    dk, dn, dp = np.array(get('DIHEDRAL_FORCE_CONSTANT')), np.array(get('DIHEDRAL_PERIODICITY')), np.array(get('DIHEDRAL_PHASE'))

    def bonds(flag, with_h):
        v = get(flag)
        return [(v[q] // 3, v[q + 1] // 3, 2.0 * bk[v[q + 2] - 1] * KCAL * 100.0, br[v[q + 2] - 1] * 0.1, with_h)
                for q in range(0, len(v), 3)]

    def angles(flag):
        v = get(flag)
        return [(v[q] // 3, v[q + 1] // 3, v[q + 2] // 3, 2.0 * ak[v[q + 3] - 1] * KCAL, at[v[q + 3] - 1])
                for q in range(0, len(v), 4)]

    torsions, pairs14 = [], []
    for flag in ('DIHEDRALS_INC_HYDROGEN', 'DIHEDRALS_WITHOUT_HYDROGEN'):
        v = get(flag)
        for q in range(0, len(v), 5):
            i, j, k, l, t = v[q], v[q + 1], v[q + 2], v[q + 3], v[q + 4] - 1
            ai, aj, akk, al = abs(i) // 3, abs(j) // 3, abs(k) // 3, abs(l) // 3
            if dk[t] != 0.0:
                torsions.append((ai, aj, akk, al, int(round(abs(dn[t]))), float(dp[t]), float(dk[t]) * KCAL))
            if k >= 0 and l >= 0:
                pairs14.append((min(ai, al), max(ai, al)))
    pairs14 = sorted(set(pairs14))

    nexcl = get('NUMBER_EXCLUDED_ATOMS')
    exlist = get('EXCLUDED_ATOMS_LIST')
    excluded, pos = set(), 0
    for i in range(natom):
        for q in range(nexcl[i]):
            j = exlist[pos + q] - 1
            if j >= 0:
                excluded.add((min(i, j), max(i, j)))
        pos += nexcl[i]

    all_bonds = bonds('BONDS_INC_HYDROGEN', True) + bonds('BONDS_WITHOUT_HYDROGEN', False)
    exceptions = []
    for (i, j) in pairs14:
        s_ij, e_ij = lj_pair(type_index[i], type_index[j])
        exceptions.append((i, j, charge[i] * charge[j] / 1.2, s_ij, e_ij / 2.0))
    full = sorted(excluded - set(pairs14))
    return dict(names=names, mass=mass, charge=charge, sigma=sigma, epsilon=epsilon, bonds=all_bonds,
                angles=angles('ANGLES_INC_HYDROGEN') + angles('ANGLES_WITHOUT_HYDROGEN'), torsions=torsions,
                exclusions=full, exceptions=exceptions,
                radii=np.array(get('RADII')) * 0.1 if 'RADII' in sec else None,
                screen=np.array(get('SCREEN')) if 'SCREEN' in sec else None,
                radius_set=''.join(get('RADIUS_SET')).strip() if 'RADIUS_SET' in sec else None)


# (alpha, beta, gamma) of the OBC models (Onufriev, Bashford, Case 2004: OBC1 = AMBER igb=2, OBC2 = igb=5)
OBC_MODELS = {'OBC1': (0.8, 0.0, 2.909125), 'OBC2': (1.0, 0.8, 4.85)}


def obc_parameters(implicitSolvent='OBC1', implicitSolventKappa=None, implicitSolventSaltConc=None, soluteDielectric=1.0,
                   solventDielectric=78.5, gbsaModel='ACE', nonbondedCutoff=None, nonbondedMethod=None):
    """system.System.gb_parameters for createSystem(implicitSolvent=...): (alpha, beta, gamma, offset, solute dielectric,
    solvent dielectric, surface-area energy, probe radius).  Salt screening, cutoffs and the HCT / GBn / GBn2 models are
    not provided: they raise NotImplementedError."""
    name = getattr(implicitSolvent, '__name__', implicitSolvent)
    if name not in OBC_MODELS:
        raise NotImplementedError('implicitSolvent=%r is not provided: OBC1 and OBC2 only (HCT, GBn and GBn2 are not)' % (name,))
    for v, what in ((implicitSolventKappa, 'implicitSolventKappa'), (implicitSolventSaltConc, 'implicitSolventSaltConc')):
        if v is not None and float(getattr(v, '_value', v)) != 0.0:
            raise NotImplementedError('%s: salt screening of the GB model is not provided' % what)
    method = getattr(nonbondedMethod, '__name__', nonbondedMethod)
    if nonbondedCutoff is not None or method not in (None, 'NoCutoff'):
        raise NotImplementedError('implicit solvent molecules are all-pairs (nonbondedMethod=NoCutoff, nonbondedCutoff=None)')
    model = getattr(gbsaModel, '__name__', gbsaModel)
    if model not in ('ACE', None):
        raise NotImplementedError("gbsaModel must be 'ACE' or None")
    sa = 2.25936 if model == 'ACE' else 0.0
    eps_in, eps_out = (float(getattr(v, '_value', v)) for v in (soluteDielectric, solventDielectric))
    return OBC_MODELS[name] + (0.009, eps_in, eps_out, sa, 0.14)


def read_inpcrd(path):
    """Positions (nm) of an AMBER coordinate file (title, atom count, 6F12.7 coordinates)."""
    lines = open(path).read().splitlines()
    n = int(lines[1].split()[0])
    vals = []
    for line in lines[2:]:
        for c in range(0, len(line), 12):
            tok = line[c:c + 12]
            if tok.strip():
                vals.append(float(tok))
        if len(vals) >= 3 * n:
            break
    return np.array(vals[:3 * n]).reshape(n, 3) * 0.1
