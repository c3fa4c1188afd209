"""Float64 restatement of an alchemically modified small molecule (vacuum, OBC1, OBC2): energy and forces at
(lambda_sterics, lambda_electrostatics), written from the reference's energy expressions (openmmtools/alchemy/alchemy.py):

* pairs and 1-4 exceptions with one alchemical atom (:1380-1450, 1840-1880, NoCutoff so reff_electrostatics = r):
    U = lambda_e 138.935456 qq / r + lambda_s^a 4 eps x (x - 1),  x = (sigma / reff)^6,
    reff = sigma (alpha (1 - lambda_s)^b + (r/sigma)^c)^(1/c)
  pairs with two alchemical atoms the same with each lambda replaced by 1 unless annihilate_sterics/_electrostatics;
* OBC (w_i = lambda_e alch_i + 1 - alch_i): I_i = sum_j w_j I_ij, self term w_i P q_i^2 / (2 B_i), ACE w_i ace_i
  (rho_i / B_i)^6, pair term P w_i q_i w_j q_j / f_ij.  OBC1 (the rewriting rules of :2223-2300) keeps the constants of the
  unmodified model; OBC2 (:2144-2221) uses 138.935485, 28.3919551 (rho + 0.14)^2 and the engulfment term C.

Bonds, angles, torsions and the pairs no lambda reaches are oracle.Molecule's (rx_oracle_mol.c), evaluated on a copy of the
system whose lambda-controlled pairs are exclusions.  TEST INFRASTRUCTURE ONLY: the product package never imports it.
"""
import numpy as np
from . import oracle

ONE_4PI_EPS0 = 138.935456
OBC2_COULOMB, OBC2_ACE = 138.935485, 28.3919551


def _pairs(system, annihilate_sterics, annihilate_electrostatics):
    """(i, j, qq, sigma, epsilon, follows lambda_s, follows lambda_e) of every lambda-controlled pair or exception."""
    n = system.n_particles
    alch = np.zeros(n, bool)
    alch[list(system.alchemical_atoms)] = True
    skip = {tuple(sorted((int(i), int(j)))) for i, j in np.asarray(system.exclusions).reshape(-1, 2)}
    exc = {tuple(sorted((int(e[0]), int(e[1])))): e for e in np.asarray(system.exceptions).reshape(-1, 5)}
    out = []

    def add(i, j, qq, sig, eps):
        na = int(alch[i]) + int(alch[j])
        ls, le = na == 1 or (na == 2 and annihilate_sterics), na == 1 or (na == 2 and annihilate_electrostatics)
        if ls or le:
            out.append((i, j, qq, sig, eps, ls, le))
    for i in range(n):
        for j in range(i + 1, n):
            if (i, j) in skip:
                continue
            if (i, j) in exc:
                e = exc[(i, j)]
                add(i, j, e[2], e[3], e[4])
            else:
                add(i, j, system.charge[i] * system.charge[j], 0.5 * (system.sigma[i] + system.sigma[j]),
                    np.sqrt(system.epsilon[i] * system.epsilon[j]))
    return out


class AlchemicalMolecule:
    """`system`: an alchemically modified System of kind 'molecule' (AbsoluteAlchemicalFactory), with or without OBC."""

    def __init__(self, system):
        if not system.is_alchemical:
            raise ValueError('the system is not alchemically modified')
        self.system = system
        self.pairs = _pairs(system, system.annihilate_sterics, system.annihilate_electrostatics)
        rest = system.copy()
        rest.alchemical_atoms = None
        rest.gb_radius = None
        extra = np.array([(p[0], p[1]) for p in self.pairs], np.int64).reshape(-1, 2)
        keep = [e for e in np.asarray(system.exceptions).reshape(-1, 5)
                if not any({int(e[0]), int(e[1])} == {p[0], p[1]} for p in self.pairs)]
        rest.exceptions = np.array(keep, np.float64).reshape(-1, 5)
        rest.exclusions = np.concatenate([np.asarray(system.exclusions, np.int64).reshape(-1, 2), extra])
        self.rest = oracle.Molecule(rest)
        self.alch = system.alchemical_mask().astype(np.float64)

    # -- the lambda-controlled pairs
    def pair_energy(self, x, lambda_sterics, lambda_electrostatics, forces=False):
        s = self.system
        al, a, b, c = s.softcore_alpha, s.softcore_a, s.softcore_b, s.softcore_c
        E, F = 0.0, np.zeros_like(x)
        for i, j, qq, sig, eps, ls, le in self.pairs:
            lam_s = lambda_sterics if ls else 1.0
            lam_e = lambda_electrostatics if le else 1.0
            d = x[i] - x[j]
            r = np.sqrt(d @ d)
            ob = al * (1.0 - lam_s) ** b
            reff = sig * (ob + (r / sig) ** c) ** (1.0 / c)
            xx = (sig / reff) ** 6
            la = lam_s ** a
            E += lam_e * ONE_4PI_EPS0 * qq / r + la * 4.0 * eps * xx * (xx - 1.0)
            if forces:
                u = (r / sig) ** c
                dreff = reff * u / ((ob + u) * r)   # d reff / d r
                dxx = -6.0 * xx / reff * dreff
                dU = -lam_e * ONE_4PI_EPS0 * qq / r ** 2 + la * 4.0 * eps * (2.0 * xx - 1.0) * dxx
                F[i] -= dU * d / r
                F[j] += dU * d / r
        return (E, F) if forces else E

    # -- OBC
    def gb_energy(self, x, lambda_electrostatics, forces=False):
        s = self.system
        alpha, beta, gamma, offset, e_in, e_out, sa, probe = s.gb_parameters
        obc2 = s.alchemical_obc2
        rho = np.asarray(s.gb_radius, np.float64)
        rt = rho - offset
        sr = np.asarray(s.gb_scale) * rt
        q = np.asarray(s.charge, np.float64)
        w = lambda_electrostatics * self.alch + (1.0 - self.alch)
        pre = -(OBC2_COULOMB if obc2 else ONE_4PI_EPS0) * (1.0 / e_in - 1.0 / e_out)
        ace = OBC2_ACE * (rho + 0.14) ** 2 if obc2 else 4.0 * np.pi * sa * (rho + probe) ** 2
        n = len(q)
        d = x[:, None, :] - x[None, :, :]
        r = np.sqrt((d ** 2).sum(-1)) + np.eye(n)
        I = np.zeros((n, n)); dI = np.zeros((n, n))
        for i in range(n):
            for j in range(n):
                if i == j or not (r[i, j] + sr[j] > rt[i]):
                    continue
                rr, S, R = r[i, j], sr[j], rt[i]
                U = rr + S
                L = max(R, abs(rr - S))
                dL = 0.0 if abs(rr - S) <= R else np.sign(rr - S)
                v = 0.5 * (1 / L - 1 / U + 0.25 * (rr - S * S / rr) * (1 / U ** 2 - 1 / L ** 2) + 0.5 * np.log(L / U) / rr)
                dv = 0.5 * (-dL / L ** 2 + 1 / U ** 2 + 0.25 * (1 + S * S / rr ** 2) * (1 / U ** 2 - 1 / L ** 2)
                            + 0.25 * (rr - S * S / rr) * (-2 / U ** 3 + 2 * dL / L ** 3)
                            + 0.5 * (dL / L - 1 / U) / rr - 0.5 * np.log(L / U) / rr ** 2)
                if obc2 and S - rr > R:       # 1/2 C
                    v += 1 / R - 1 / L
                    dv += dL / L ** 2
                I[i, j], dI[i, j] = w[j] * v, w[j] * dv
        Isum = I.sum(1)
        psi = Isum * rt
        th = np.tanh(alpha * psi - beta * psi ** 2 + gamma * psi ** 3)
        B = 1.0 / (1.0 / rt - th / rho)
        dBdI = B ** 2 * (1 - th ** 2) / rho * (alpha - 2 * beta * psi + 3 * gamma * psi ** 2) * rt
        wq = w * q
        E = np.sum(w * (0.5 * pre * q ** 2 / B + ace * (rho / B) ** 6))
        dEdB = w * (-0.5 * pre * q ** 2 / B ** 2 - 6.0 * ace * (rho / B) ** 6 / B)
        F = np.zeros_like(x)
        for i in range(n):
            for j in range(i + 1, n):
                r2, D = r[i, j] ** 2, B[i] * B[j]
                ex = np.exp(-r2 / (4 * D))
                f = np.sqrt(r2 + D * ex)
                e = pre * wq[i] * wq[j] / f
                E += e
                if forces:
                    dfd = -e / f                        # dE/df
                    df_dr = (2 * r[i, j] - 0.5 * r[i, j] * ex) / (2 * f)
                    df_dD = ex * (1 + r2 / (4 * D)) / (2 * f)
                    dEdB[i] += dfd * df_dD * B[j]
                    dEdB[j] += dfd * df_dD * B[i]
                    g = dfd * df_dr * d[i, j] / r[i, j]
                    F[i] -= g; F[j] += g
        if forces:
            C = dEdB * dBdI
            for i in range(n):
                for j in range(n):
                    if i != j:
                        g = C[i] * dI[i, j] * d[i, j] / r[i, j]   # dE/dx_i through I_i(r_ij)
                        F[i] -= g; F[j] += g
        return (E, F) if forces else E

    def energy(self, x, lambda_sterics=1.0, lambda_electrostatics=1.0, forces=False):
        x = np.ascontiguousarray(x, np.float64)
        E, F = self.rest.energy(x, forces=True)
        F = np.array(F, np.float64)
        e, f = self.pair_energy(x, lambda_sterics, lambda_electrostatics, forces=True)
        E += e; F += f
        if self.system.gb_radius is not None:
            e, f = self.gb_energy(x, lambda_electrostatics, forces=True)
            E += e; F += f
        return (E, F) if forces else E
