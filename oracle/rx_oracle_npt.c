/* rx_oracle_npt.c -- CPU restatement (f64) of the alchemical LJ fluid at constant pressure: the energy matrix with a box per
 * replica and the pV term, and the Monte Carlo barostat step.
 *
 * TEST INFRASTRUCTURE ONLY, like rx_oracle.c: used by tests/, never by the product.  Built as its own library, liborc_npt.so
 * (oracle/npt.py), from this file alone: rx_oracle.c is included so that the pair energies, forces and Langevin steps are the
 * very code the NVT oracle runs.
 *
 * The barostat follows OpenMM's documented MonteCarloBarostat (isotropic, every atom its own molecule):
 *   propose V' = V + dV, dV = volume_scale (2 u1 - 1); scale positions about the origin by s = (V'/V)^(1/3);
 *   w = U(s x, s L) - U(x, L) + c (1/V' - 1/V) + p dV - N kT ln(V'/V); accept when w <= 0 or u2 < exp(-w/kT);
 *   after every 10 attempts: acceptance < 0.25 -> volume_scale / 1.1, > 0.75 -> min(volume_scale * 1.1, 0.3 V), counters reset.
 * The uniforms u1, u2 are inputs, so that tests can feed the device's.  A proposal with a box edge below min_edge (twice the
 * cutoff) is refused and counted as an attempt (OpenMM raises instead).  Velocities are not scaled. */
#include "rx_oracle.c"

typedef struct orc_barostat {
    double volume_scale;
    int32_t step, n_attempted, n_accepted, reserved;
} orc_barostat;

static double lj_energy_at(const orc_lj_params *p, const double *box, const double *sigma, const double *eps,
                           const uint8_t *alch, const double *x, double lam, double *f) {
    orc_lj_params q = *p;
    for (int d = 0; d < 3; d++) q.box[d] = box[d];
    return orc_lj_energy(&q, sigma, eps, alch, x, lam, NULL, f);
}

/* u[k][l] = beta_l (U_l(x_k; box_k) + offset_l + dispersion_l / V_k + pressure_l V_k); boxes [count][3]. */
ORC_API void orc_npt_energy_matrix(const orc_lj_params *p, const double *sigma, const double *eps, const uint8_t *alch,
                                   int count, const double *x, const double *boxes, int M, const double *lambdas,
                                   const double *betas, const double *offsets, const double *pressure,
                                   const double *dispersion, double *u) {
    const int N = p->n_atoms;
#pragma omp parallel for schedule(dynamic)
    for (int k = 0; k < count; k++) {
        const double *b = boxes + 3 * k;
        const double V = b[0] * b[1] * b[2];
        for (int l = 0; l < M; l++) {
            const double U = lj_energy_at(p, b, sigma, eps, alch, x + (size_t)3 * N * k, lambdas[l], NULL);
            u[(size_t)k * M + l] = betas[l] * (U + (offsets ? offsets[l] : 0.0) + dispersion[l] / V + pressure[l] * V);
        }
    }
}

/* One barostat attempt on x [N][3] and box [3] (both updated on acceptance).  Returns 1 accepted, 0 rejected, -1 refused
 * (box edge below min_edge); *w_out (may be NULL) gets w when an energy was taken. */
ORC_API int orc_npt_barostat_step(const orc_lj_params *p, const double *sigma, const double *eps, const uint8_t *alch,
                                  double lam, double kT, double pressure, double dispersion, double min_edge, double *x,
                                  double *box, orc_barostat *st, double u1, double u2, double *w_out) {
    const int N = p->n_atoms;
    const double V = box[0] * box[1] * box[2];
    const double dV = st->volume_scale * (2.0 * u1 - 1.0), V1 = V + dV;
    const double s = V1 > 0.0 ? cbrt(V1 / V) : 0.0;
    int result = -1;
    st->n_attempted++;
    if (box[0] * s >= min_edge && box[1] * s >= min_edge && box[2] * s >= min_edge) {
        double *y = (double *)malloc(sizeof(double) * 3 * N);
        const double nb[3] = {box[0] * s, box[1] * s, box[2] * s};
        for (int i = 0; i < 3 * N; i++) y[i] = x[i] * s;
        const double U0 = lj_energy_at(p, box, sigma, eps, alch, x, lam, NULL);
        const double U1 = lj_energy_at(p, nb, sigma, eps, alch, y, lam, NULL);
        const double w = U1 - U0 + dispersion * (1.0 / V1 - 1.0 / V) + pressure * dV - N * kT * log(V1 / V);
        if (w_out) *w_out = w;
        result = (w <= 0.0 || u2 < exp(-w / kT)) ? 1 : 0;
        if (result) {
            memcpy(x, y, sizeof(double) * 3 * N);
            for (int d = 0; d < 3; d++) box[d] = nb[d];
            st->n_accepted++;
        }
        free(y);
    }
    if (st->n_attempted >= 10) {
        if (st->n_accepted < 0.25 * st->n_attempted) { st->volume_scale /= 1.1; st->n_attempted = st->n_accepted = 0; }
        else if (st->n_accepted > 0.75 * st->n_attempted) {
            st->volume_scale = fmin(st->volume_scale * 1.1, 0.3 * V);
            st->n_attempted = st->n_accepted = 0;
        }
    }
    return result;
}

/* n_steps Langevin steps (program, noise as orc_langevin_steps) with a barostat attempt at the start of every step whose
 * counter st->step reaches 25; uniforms [2 * attempts] are consumed in order, decisions[attempts] receive the results. */
ORC_API int orc_npt_langevin(const orc_lj_params *p, const orc_dyn_params *d, const char *program, const double *sigma,
                             const double *eps, const uint8_t *alch, const double *mass, double *x, double *v,
                             const double *noise, double *box, orc_barostat *st, double pressure, double dispersion,
                             double min_edge, const double *uniforms, int max_attempts, int *decisions, double *potential_out) {
    const int N = p->n_atoms;
    int nO = 0;
    for (const char *c = program; *c; c++) nO += *c == 'O';
    orc_dyn_params one = *d;
    one.n_steps = 1;
    int n_att = 0;
    double U = 0.0;
    for (int s = 0; s < d->n_steps; s++) {
        if (++st->step >= 25) {
            st->step = 0;
            if (n_att >= max_attempts) return -3;
            decisions[n_att] = orc_npt_barostat_step(p, sigma, eps, alch, d->lambda, d->kT, pressure, dispersion, min_edge, x,
                                                     box, st, uniforms[2 * n_att], uniforms[2 * n_att + 1], NULL);
            n_att++;
        }
        orc_lj_params q = *p;
        for (int k = 0; k < 3; k++) q.box[k] = box[k];
        const int r = orc_langevin_steps(&q, &one, program, sigma, eps, alch, mass, x, v, noise + (size_t)s * nO * 3 * N, &U);
        if (r) return r;
    }
    if (potential_out) *potential_out = U + dispersion / (box[0] * box[1] * box[2]);
    return n_att;
}
