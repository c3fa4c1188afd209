/* rx_oracle_npt_aniso.c -- CPU restatement (f64) of the anisotropic Monte Carlo barostat on the alchemical LJ fluid.
 *
 * TEST INFRASTRUCTURE ONLY, like rx_oracle_npt.c: used by tests/, never by the product.  Built as its own library,
 * liborc_npt_aniso.so (oracle/npt_aniso.py), from this file alone: rx_oracle_npt.c (and through it rx_oracle.c) is included,
 * so that the pair energies, forces and Langevin steps are the very code the isotropic NPT oracle runs.
 *
 * OpenMM's MonteCarloAnisotropicBarostat with every atom its own molecule and one pressure on the scaled axes: an attempt on
 * axis `axis` (an input, as the uniforms are) proposes dV = volume_scale[axis] (2 u1 - 1) and scales that box edge and that
 * coordinate of every atom by s = V'/V; w = U(s x, s L) - U(x, L) + c (1/V' - 1/V) + p dV - N kT ln(V'/V), accepted when
 * w <= 0 or u2 < exp(-w/kT).  Only the scaled edge is held at min_edge (a shorter one is refused and counted as an
 * attempt).  Each axis counts its own attempts and, after every 10 of them, adapts its own volume_scale by the isotropic
 * rule: acceptance < 0.25 -> / 1.1, > 0.75 -> min(* 1.1, 0.3 V), counters reset.  Velocities are not scaled. */
#include "rx_oracle_npt.c"

typedef struct orc_aniso_barostat {
    double volume_scale[3];
    int32_t n_attempted[3], n_accepted[3], step, scale_mask;
} orc_aniso_barostat;

/* One attempt on `axis`; x [N][3], box [3] and st are updated.  Returns 1 accepted, 0 rejected, -1 refused; *w_out (may
 * be NULL) gets w when an energy was taken. */
ORC_API int orc_npt_aniso_barostat_step(const orc_lj_params *p, const double *sigma, const double *eps, const uint8_t *alch,
                                        double lam, double kT, double pressure, double dispersion, double min_edge, double *x,
                                        double *box, orc_aniso_barostat *st, int axis, double u1, double u2, double *w_out) {
    const int N = p->n_atoms;
    const double V = box[0] * box[1] * box[2];
    const double dV = st->volume_scale[axis] * (2.0 * u1 - 1.0), V1 = V + dV, s = V1 / V;
    int result = -1;
    st->n_attempted[axis]++;
    if (box[axis] * s >= min_edge) {
        double *y = (double *)malloc(sizeof(double) * 3 * N);
        double nb[3] = {box[0], box[1], box[2]};
        nb[axis] *= s;
        memcpy(y, x, sizeof(double) * 3 * N);
        for (int i = 0; i < N; i++) y[3 * i + axis] *= s;
        const double U0 = lj_energy_at(p, box, sigma, eps, alch, x, lam, NULL);
        const double U1 = lj_energy_at(p, nb, sigma, eps, alch, y, lam, NULL);
        const double w = U1 - U0 + dispersion * (1.0 / V1 - 1.0 / V) + pressure * dV - N * kT * log(V1 / V);
        if (w_out) *w_out = w;
        result = (w <= 0.0 || u2 < exp(-w / kT)) ? 1 : 0;
        if (result) {
            memcpy(x, y, sizeof(double) * 3 * N);
            box[axis] = nb[axis];
            st->n_accepted[axis]++;
        }
        free(y);
    }
    if (st->n_attempted[axis] >= 10) {
        if (st->n_accepted[axis] < 0.25 * st->n_attempted[axis]) {
            st->volume_scale[axis] /= 1.1;
            st->n_attempted[axis] = st->n_accepted[axis] = 0;
        } else if (st->n_accepted[axis] > 0.75 * st->n_attempted[axis]) {
            st->volume_scale[axis] = fmin(st->volume_scale[axis] * 1.1, 0.3 * V);
            st->n_attempted[axis] = st->n_accepted[axis] = 0;
        }
    }
    return result;
}

/* orc_npt_langevin with the anisotropic barostat: n_steps steps with an attempt at the start of every step whose counter
 * st->step reaches 25; attempt i takes axes[i] and uniforms[2 i], [2 i + 1], decisions[i] receives its result. */
ORC_API int orc_npt_aniso_langevin(const orc_lj_params *p, const orc_dyn_params *d, const char *program, const double *sigma,
                                   const double *eps, const uint8_t *alch, const double *mass, double *x, double *v,
                                   const double *noise, double *box, orc_aniso_barostat *st, double pressure,
                                   double dispersion, double min_edge, const int *axes, const double *uniforms,
                                   int max_attempts, int *decisions, double *potential_out) {
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
            decisions[n_att] = orc_npt_aniso_barostat_step(p, sigma, eps, alch, d->lambda, d->kT, pressure, dispersion, min_edge,
                                                           x, box, st, axes[n_att], uniforms[2 * n_att],
                                                           uniforms[2 * n_att + 1], NULL);
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
