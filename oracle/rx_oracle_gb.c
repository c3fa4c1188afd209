/* rx_oracle_gb.c -- CPU restatement (f64) of a small molecule in OBC implicit solvent: the vacuum force field and the
 * constrained Langevin steps of rx_oracle_mol.c plus the generalized Born model below.
 *
 * TEST INFRASTRUCTURE ONLY, like rx_oracle_mol.c: used by tests/ and tools/, never by the product.  Built as its own library,
 * liborc_gb.so (oracle/implicit.py), from this file alone: rx_oracle_mol.c is included so that the vacuum terms, SHAKE,
 * RATTLE and the centre-of-mass removal are the very code the vacuum oracle runs.
 * Parity: pinned against AMBER 9 sander for OBC1 without the ACE term (the T4-lysozyme L99A ligand, tests/test_oracle_implicit.py);
 * OBC2, the ACE term and engulfed pairs are unpinned (DESIGN.md section 2). */
#include "rx_oracle_mol.c"

/* OBC generalized Born (AmberPrmtopFile.createSystem(implicitSolvent=OBC1|OBC2), no cutoff, no salt), restated from the
 * published model (Onufriev, Bashford, Case 2004; OpenMM's GBSAOBCForce documentation).  For atom i: rho_i the radius,
 * rt_i = rho_i - offset, sr_i = scale_i rt_i.
 *   I_i = sum_{j != i} I_ij over every pair,  I_ij = 1/2 [1/L - 1/U + 1/4 (r - sr_j^2/r)(1/U^2 - 1/L^2) + 1/2 ln(L/U)/r]
 *         when r + sr_j > rt_i (else 0),  U = r + sr_j,  L = max(rt_i, |r - sr_j|)   (no engulfment term)
 *   B_i = 1 / (1/rt_i - tanh(alpha psi_i - beta psi_i^2 + gamma psi_i^3) / rho_i),  psi_i = I_i rt_i
 *   E   = sum_i 1/2 P q_i^2 / B_i + sum_{i<j} P q_i q_j / f_ij,  f_ij = sqrt(r^2 + B_i B_j exp(-r^2 / (4 B_i B_j)))
 *         + sum_i 4 pi sa_energy (rho_i + probe)^2 (rho_i / B_i)^6   (ACE non-polar term)
 *   P   = -ONE_4PI_EPS0 (1/solute_dielectric - 1/solvent_dielectric). */
typedef struct orc_gb {
    const double *radius, *scale;   /* [n_atoms] nm, dimensionless */
    double alpha, beta, gamma, offset, solute_dielectric, solvent_dielectric, sa_energy, probe_radius;
} orc_gb;

/* I_ij of atom i (offset radius rt) descreened by j (scaled radius sr) at distance r, and dI_ij/dr. */
static double descreen(double r, double rt, double sr, double *dIdr) {
    *dIdr = 0.0;
    if (r + sr <= rt) return 0.0;
    const double U = r + sr;
    double L = rt, dL = 0.0;
    if (fabs(r - sr) > rt) { L = fabs(r - sr); dL = r > sr ? 1.0 : -1.0; }
    const double a = r - sr * sr / r, b = 1.0 / (U * U) - 1.0 / (L * L);
    const double I = 0.5 * (1.0 / L - 1.0 / U + 0.25 * a * b + 0.5 * log(L / U) / r);
    const double da = 1.0 + sr * sr / (r * r), db = -2.0 / (U * U * U) + 2.0 * dL / (L * L * L);
    *dIdr = 0.5 * (-dL / (L * L) + 1.0 / (U * U) + 0.25 * (da * b + a * db) + 0.5 * ((dL / L - 1.0 / U) / r - log(L / U) / (r * r)));
    return I;
}

/* The OBC energy; f (may be NULL) accumulates its forces. */
static double gb_energy(const orc_mol *m, const orc_gb *g, const double *x, double *f) {
    const int n = m->n_atoms;
    const double P = -ONE_4PI_EPS0 * (1.0 / g->solute_dielectric - 1.0 / g->solvent_dielectric);
    double *B = (double *)calloc((size_t)n, sizeof(double)), *dB = (double *)calloc((size_t)n, sizeof(double));
    double *dE = (double *)calloc((size_t)n, sizeof(double));
    double E = 0.0;
    for (int i = 0; i < n; i++) {
        const double rho = g->radius[i], rt = rho - g->offset;
        double I = 0.0, dI;
        for (int j = 0; j < n; j++) {
            if (j == i) continue;
            double d[3] = {x[3 * i] - x[3 * j], x[3 * i + 1] - x[3 * j + 1], x[3 * i + 2] - x[3 * j + 2]};
            I += descreen(sqrt(dot(d, d)), rt, g->scale[j] * (g->radius[j] - g->offset), &dI);
        }
        const double psi = I * rt, z = g->alpha * psi - g->beta * psi * psi + g->gamma * psi * psi * psi, th = tanh(z);
        B[i] = 1.0 / (1.0 / rt - th / rho);
        dB[i] = B[i] * B[i] * (1.0 - th * th) / rho * (g->alpha - 2.0 * g->beta * psi + 3.0 * g->gamma * psi * psi) * rt;
    }
    for (int i = 0; i < n; i++) {
        const double q = m->charge[i], rho = g->radius[i];
        const double self = 0.5 * P * q * q / B[i], ace = 4.0 * M_PI * g->sa_energy * pow(rho + g->probe_radius, 2.0) * pow(rho / B[i], 6.0);
        E += self + ace;
        dE[i] += -self / B[i] - 6.0 * ace / B[i];
        for (int j = i + 1; j < n; j++) {
            double d[3] = {x[3 * i] - x[3 * j], x[3 * i + 1] - x[3 * j + 1], x[3 * i + 2] - x[3 * j + 2]};
            const double r2 = dot(d, d), D = B[i] * B[j], ex = exp(-r2 / (4.0 * D)), fij = sqrt(r2 + D * ex);
            const double e = P * q * m->charge[j] / fij;
            E += e;
            /* dE/d(f^2) = -e / (2 f^2);  d(f^2)/dr = r (2 - ex/2);  d(f^2)/dB_i = B_j ex (1 + r^2/(4 D)) */
            const double c = -0.5 * e / (fij * fij);
            dE[i] += c * B[j] * ex * (1.0 + r2 / (4.0 * D));
            dE[j] += c * B[i] * ex * (1.0 + r2 / (4.0 * D));
            if (f) {
                const double fr = -c * (2.0 - 0.5 * ex);   /* -dE/dr / r */
                for (int k = 0; k < 3; k++) { f[3 * i + k] += fr * d[k]; f[3 * j + k] -= fr * d[k]; }
            }
        }
    }
    if (f)   /* through the Born radii: dE/dB_i dB_i/dI_i dI_ij/dr_ij */
        for (int i = 0; i < n; i++) {
            const double rt = g->radius[i] - g->offset, ci = dE[i] * dB[i];
            for (int j = 0; j < n; j++) {
                if (j == i) continue;
                double d[3] = {x[3 * i] - x[3 * j], x[3 * i + 1] - x[3 * j + 1], x[3 * i + 2] - x[3 * j + 2]}, dI;
                const double r = sqrt(dot(d, d));
                descreen(r, rt, g->scale[j] * (g->radius[j] - g->offset), &dI);
                for (int k = 0; k < 3; k++) { f[3 * i + k] -= ci * dI * d[k] / r; f[3 * j + k] += ci * dI * d[k] / r; }
            }
        }
    free(B); free(dB); free(dE);
    return E;
}

/* The OBC energy alone; f (may be NULL) receives its forces. */
ORC_API double orc_gb_energy(const orc_mol *m, const orc_gb *g, const double *x, double *f) {
    if (f) memset(f, 0, sizeof(double) * 3 * (size_t)m->n_atoms);
    return gb_energy(m, g, x, f);
}

/* The potential energy in implicit solvent: the vacuum force field plus the OBC energy; f (may be NULL) the forces. */
ORC_API double orc_gb_mol_energy(const orc_mol *m, const orc_gb *g, const double *x, double *f) {
    const double U = orc_mol_energy(m, x, f);
    return U + gb_energy(m, g, x, f);
}

/* Born radii (nm) into B; returns the number of pairs with sr_j - r > rt_i ("engulfed", outside the model above). */
ORC_API int orc_gb_born_radii(const orc_mol *m, const orc_gb *g, const double *x, double *B) {
    int engulfed = 0;
    for (int i = 0; i < m->n_atoms; i++) {
        const double rho = g->radius[i], rt = rho - g->offset;
        double I = 0.0, dI;
        for (int j = 0; j < m->n_atoms; j++) {
            if (j == i) continue;
            double d[3] = {x[3 * i] - x[3 * j], x[3 * i + 1] - x[3 * j + 1], x[3 * i + 2] - x[3 * j + 2]};
            const double r = sqrt(dot(d, d)), sr = g->scale[j] * (g->radius[j] - g->offset);
            if (sr - r > rt) engulfed++;
            I += descreen(r, rt, sr, &dI);
        }
        const double psi = I * rt;
        B[i] = 1.0 / (1.0 / rt - tanh(g->alpha * psi - g->beta * psi * psi + g->gamma * psi * psi * psi) / rho);
    }
    return engulfed;
}

/* orc_mol_langevin in implicit solvent: n_steps of the splitting `program` (characters V, R, O) with injected standard normals noise[n_steps*nO][n][3]. */
ORC_API double orc_gb_langevin(const orc_mol *m, const orc_gb *g, double *x, double *v, const double *noise, double kT, double dt, double gamma,
                              int n_steps, const char *program, double tol) {
    const int n = m->n_atoms;
    int nV = 0, nR = 0, nO = 0;
    for (const char *q = program; *q; q++) { if (*q == 'V') nV++; else if (*q == 'R') nR++; else if (*q == 'O') nO++; }
    const double hO = dt / (nO > 0 ? nO : 1);
    const double a = exp(-gamma * hO), b = sqrt(1.0 - exp(-2.0 * gamma * hO));
    double *f = (double *)malloc(sizeof(double) * 3 * n), *x1 = (double *)malloc(sizeof(double) * 3 * n);
    int f_valid = 0;
    long oc = 0;
    for (int s = 0; s < n_steps; s++) {
        if (m->remove_cm) remove_cm(m, v);
        for (const char *q = program; *q; q++) {
            if (*q == 'V') {
                if (!f_valid) { orc_gb_mol_energy(m, g, x, f); f_valid = 1; }
                const double h = dt / nV;
                for (int i = 0; i < n; i++) for (int c = 0; c < 3; c++) v[3 * i + c] += h * f[3 * i + c] / m->mass[i];
                if (m->n_cons) rattle(m, x, v, tol);
            } else if (*q == 'R') {
                const double h = dt / nR;
                memcpy(x1, x, sizeof(double) * 3 * n);           /* bond vectors before the move (SHAKE directions) */
                for (int i = 0; i < 3 * n; i++) x[i] += h * v[i];
                if (m->n_cons) {
                    double *xu = (double *)malloc(sizeof(double) * 3 * n);
                    memcpy(xu, x, sizeof(double) * 3 * n);       /* "x1" of integrators.py:1415: the unconstrained positions */
                    shake(m, x1, x, tol);
                    for (int i = 0; i < 3 * n; i++) v[i] += (x[i] - xu[i]) / h;
                    free(xu);
                    rattle(m, x, v, tol);
                }
                f_valid = 0;
            } else if (*q == 'O') {
                for (int i = 0; i < n; i++) {
                    const double sg = sqrt(kT / m->mass[i]);
                    for (int c = 0; c < 3; c++) v[3 * i + c] = a * v[3 * i + c] + b * sg * noise[(oc * n + i) * 3 + c];
                }
                oc++;
                if (m->n_cons) rattle(m, x, v, tol);
            }
        }
    }
    const double U = orc_gb_mol_energy(m, g, x, NULL);
    free(f); free(x1);
    return U;
}

