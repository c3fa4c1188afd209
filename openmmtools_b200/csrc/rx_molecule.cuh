// rx_molecule.cuh -- a small molecule in vacuum per replica (included at the end of rx_dynamics.cu).
//
// The system testsystems.AlanineDipeptideVacuum builds (/root/reference/openmmtools/testsystems.py:3352-3388:
// AmberPrmtopFile.createSystem(implicitSolvent=None, constraints=HBonds, nonbondedCutoff=None)) propagated by the constrained
// Langevin splitting of /root/reference/openmmtools/integrators.py:1404-1460:
//   R  x1 = x + (dt/nR) v;  x = constrain(x1);  v += (x - x1) / (dt/nR);  constrain velocities      (:1404-1422)
//   V  v += (dt/nV) f / m;  constrain velocities                                                    (:1424-1447)
//   O  v = a v + b sqrt(kT/m) xi;  constrain velocities                                             (:1449-1460)
// with the centre-of-mass velocity removed at the start of every step (CMMotionRemover through addUpdateContextState).
//
// k_propagate_mol: one block of four warps per replica, the state (x, v in f64) on chip for all steps.  Warp 0 integrates --
// one lane per atom (N <= 32), one lane per constraint cluster -- and all 128 threads evaluate the force terms in f32 on the
// f64 positions: every bond / angle / torsion / pair ONCE, by whichever thread its index falls to, into fixed shared-memory
// slots that each atom then adds up in slot order (no atomics: the same bits every run, whatever the thread count).
// Constraints are solved cluster by cluster (connected components of the constraint graph, e.g. a CH3 group) by the lane that
// owns the cluster.  Clusters of <= 3 constraints (every H-bond cluster) take the MolStar path: register copies of the
// cluster's <= 4 atoms, the RATTLE matrix inverted once per position update in closed form, SHAKE as chord iterations on that
// inverse (k_propagate_mol<true>); larger clusters a Newton M-SHAKE (<= 4 constraints) or Gauss-Seidel sweeps
// (k_propagate_mol<false>).  All of them reach the constrained point of oracle/rx_oracle_mol.c's sweeps to the tolerance.
// The energy kernel (k_energy_mol) and the minimiser (k_minimize_mol) use one warp per replica and the same term list packed
// in f64 (mol_terms<double, .>); the energy a launch of k_propagate_mol reports is k_energy_mol's function (mol_energy).
#pragma once

#define MOL_MAX_ATOMS 32
#define MOL_ONE_4PI_EPS0 138.935456

struct MolCons { int i, j; double d; };

// The term list of a molecule, packed in the precision T of its evaluation: rx_set_molecule packs it twice in one layout, f32
// for the dynamics' forces and f64 for the energies and the minimiser.  Every bond / angle / torsion / interacting pair is
// evaluated ONCE, by whichever thread its index falls to; its contributions go to fixed slots of a shared-memory array and
// every atom then adds up ITS slots in slot order -- no atomics, the same bits every run whatever the thread count.
template <typename T> struct TBond { short i, j, si, sj; T K, r0; };
template <typename T> struct TAngle { short i, j, k, si, sj, sk; T K, t0; };
template <typename T> struct TTors { short i, j, k, l, si, sj, sk, sl; T n, phase, kk; };
template <typename T> struct TPair { short i, j, si, sj; T qq, sig, eps; };   // qq = 138.935456 q_i q_j (exceptions: their own values)
// An alchemical pair (rx_set_molecule with an alchemical mask; alchemy.py:1380-1450, NoCutoff): a pair or 1-4 exception with
// an alchemical atom whose soft-core sterics follow the state's lambda_sterics (ls = 1; ls = 0: lambda 1, an alchemical/
// alchemical pair without annihilate_sterics) and whose Coulomb term is scaled by lambda_electrostatics (le = 1; le = 0: by 1).
//   U = le_factor qq / r + la 4 eps x (x - 1),  x = (ob + (r/sig)^c)^(-6/c),  la = lambda^a, ob = alpha (1 - lambda)^b
template <typename T> struct TAPair { short i, j, si, sj, ls, le, pad[2]; T qq, sig, eps; };
struct MolTerms {      // one contiguous blob: header, then the arrays (offsets in bytes from the blob's start)
    int o_bond, o_angle, o_tors, o_pair, o_goff, o_apair, pad[2];   // goff (at o_goff): atom a's slots are [goff[a], goff[a + 1])
};

struct MolDev {
    int n, n_clusters, remove_cm, max_cluster;   // max_cluster: constraints in the largest cluster
    double tol;
    const double *mass, *charge;
    const int *c_off;
    const MolCons *cons;
    const MolTerms *terms32, *terms64;   // the term list in f32 and in f64 (bytes32, bytes64: multiples of 16)
    int bytes32, bytes64, n_tb, n_ta, n_tt, n_tp, n_slots;
    // alchemical molecules only (the ALCH instantiations read them): the alchemical pairs, the region as a bit mask of atoms,
    // the soft-core exponent c (c6: c == 6)
    int n_tap, c6;
    unsigned alch;
    double sc_c;
};

// OBC generalized Born implicit solvent (rx_set_implicit_solvent), passed to the kernels as a trailing argument so that the
// vacuum instantiations (GB = false) keep their argument layout.  All in f64.  For atom i: rho_i the radius, rt_i = rho_i -
// offset, sr_i = scale_i rt_i.
//   I_i = sum_{j != i} I_ij,  I_ij = 1/2 [1/L - 1/U + 1/4 (r - sr_j^2/r)(1/U^2 - 1/L^2) + 1/2 ln(L/U) / r]  if r + sr_j > rt_i
//         (U = r + sr_j, L = max(rt_i, |r - sr_j|); no engulfment term),
//   B_i = 1 / (1/rt_i - tanh(alpha psi - beta psi^2 + gamma psi^3) / rho_i),  psi = I_i rt_i,
//   E = sum_i [1/2 pre q_i^2 / B_i + ace_i (rho_i / B_i)^6] + sum_{i<j} pre q_i q_j / sqrt(r^2 + B_i B_j exp(-r^2 / (4 B_i B_j)))
// with pre = -138.935456 (1/eps_solute - 1/eps_solvent) and ace_i = 4 pi sa_energy (rho_i + probe)^2.
struct MolGB {
    const double *atom;   // [n][4]: rt, sr, rho, ace
    double alpha, beta, gamma, pre;
    int on;               // (0: vacuum; the GB = true kernels are only launched with 1)
    int prop_bytes;       // the arrays of MolGBArrays, behind the slots (mol_gb_at)
    int engulf;           // the alchemical OBC2 expression's engulfment term C (alchemy.py:2188-2193; ALCH kernels only)
};

// The weight of atom i's charge and descreening in an alchemical state: w_i = lambda_e alch_i + (1 - alch_i)
// (alchemy.py:2188-2203 and the rewriting rules of :2223-2300).
__device__ __forceinline__ double mol_w(const MolDev &m, int i, double le) { return ((m.alch >> i) & 1u) ? le : 1.0; }

// Dynamic shared memory of the molecule kernels: the staged term table (f32: k_propagate_mol, f64: k_energy_mol and
// k_minimize_mol), then one double[3] per slot (k_propagate_mol: the float[3] forces of its steps, then the energy slots of
// its final energy), then with GB the arrays of MolGBArrays.
__host__ __device__ inline int mol_slots_at(const MolDev &m, bool f32) { return f32 ? m.bytes32 : m.bytes64; }
__host__ __device__ inline int mol_gb_at(const MolDev &m, bool f32) { return mol_slots_at(m, f32) + 24 * m.n_slots; }

// I_ij at distance r of atom i (offset radius rt) descreened by j (scaled radius sr); *dIdr its derivative.
// engulf: with the engulfment term 1/2 C, C = 2 (1/rt - 1/L) step(sr - r - rt) (the alchemical OBC2 expression).
__device__ __forceinline__ double gb_descreen(double r, double rt, double sr, double *dIdr, bool engulf = false) {
    if (!(r + sr > rt)) { *dIdr = 0.0; return 0.0; }
    const double U = r + sr, d = r - sr, ad = fabs(d);
    const bool far = ad > rt;
    const double L = far ? ad : rt, dL = far ? (d > 0.0 ? 1.0 : -1.0) : 0.0;
    const double iL = 1.0 / L, iU = 1.0 / U, ir = 1.0 / r, iL2 = iL * iL, iU2 = iU * iU, q = sr * sr * ir, lg = log(L * iU);
    *dIdr = 0.5 * (-dL * iL2 + iU2 + 0.25 * (1.0 + q * ir) * (iU2 - iL2) + 0.5 * (r - q) * (dL * iL2 * iL - iU2 * iU) +
                   0.5 * ((dL * iL - iU) - lg * ir) * ir);
    const double I = 0.5 * (iL - iU + 0.25 * (r - q) * (iU2 - iL2) + 0.5 * lg * ir);
    if (engulf && sr - r > rt) { *dIdr += dL * iL2; return I + (1.0 / rt - iL); }
    return I;
}

// Born radius from the descreening sum; *dBdI its derivative.
__device__ __forceinline__ double gb_born(const MolGB &g, double I, double rt, double rho, double *dBdI) {
    const double psi = I * rt, th = tanh(psi * (g.alpha + psi * (-g.beta + psi * g.gamma)));
    const double B = 1.0 / (1.0 / rt - th / rho);
    *dBdI = B * B * (1.0 - th * th) / rho * (g.alpha + psi * (-2.0 * g.beta + 3.0 * g.gamma * psi)) * rt;
    return B;
}

// The pair term pqq / f (pqq = pre q_i q_j); *dr: dE/dr / r; *dbi, *dbj: dE/dB_i, dE/dB_j.
__device__ __forceinline__ double gb_pair(double r2, double Bi, double Bj, double pqq, double *dr, double *dbi, double *dbj) {
    const double D = Bi * Bj, ex = exp(-0.25 * r2 / D), f2 = r2 + D * ex, E = pqq / sqrt(f2), c = -0.5 * E / f2;
    const double cb = c * ex * (1.0 + 0.25 * r2 / D);
    *dr = c * (2.0 - 0.5 * ex); *dbi = cb * Bj; *dbj = cb * Bi;
    return E;
}

// The self and ACE terms of atom a; *dB: their dE/dB.
__device__ __forceinline__ double gb_self(const MolGB &g, double q, double B, double rho, double ace, double *dB) {
    const double es = 0.5 * g.pre * q * q / B, t = rho / B, t3 = t * t * t, ea = ace * t3 * t3;
    *dB = -(es + 6.0 * ea) / B;
    return es + ea;
}

__device__ __forceinline__ double gb_dist(const double (*X)[3], int i, int j, double *d) {
    d[0] = X[i][0] - X[j][0]; d[1] = X[i][1] - X[j][1]; d[2] = X[i][2] - X[j][2];
    return sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
}

__device__ __forceinline__ void mol_cross(const double *a, const double *b, double *c) {
    c[0] = a[1] * b[2] - a[2] * b[1]; c[1] = a[2] * b[0] - a[0] * b[2]; c[2] = a[0] * b[1] - a[1] * b[0];
}
__device__ __forceinline__ double mol_dot(const double *a, const double *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

__device__ __forceinline__ double mol_warp_sum(double v) {   // fixed tree: bit-reproducible
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// The f32 and f64 forms of the math of mol_terms (the f32 ones are those the dynamics has always used).
__device__ __forceinline__ float mol_sqrt(float x) { return sqrtf(x); }
__device__ __forceinline__ double mol_sqrt(double x) { return sqrt(x); }
__device__ __forceinline__ float mol_rsqrt(float x) { return rsqrtf(x); }
__device__ __forceinline__ double mol_rsqrt(double x) { return 1.0 / sqrt(x); }
__device__ __forceinline__ float mol_clamp1(float x) { return fminf(1.f, fmaxf(-1.f, x)); }
__device__ __forceinline__ double mol_clamp1(double x) { return x > 1.0 ? 1.0 : (x < -1.0 ? -1.0 : x); }
__device__ __forceinline__ float mol_acos(float x) { return acosf(x); }
__device__ __forceinline__ double mol_acos(double x) { return acos(x); }
__device__ __forceinline__ float mol_atan2(float y, float x) { return atan2f(y, x); }
__device__ __forceinline__ double mol_atan2(double y, double x) { return atan2(y, x); }
__device__ __forceinline__ void mol_sincos(float x, float *s, float *c) { sincosf(x, s, c); }
__device__ __forceinline__ void mol_sincos(double x, double *s, double *c) { sincos(x, s, c); }

// Stage a term table (bytes: a multiple of 16) into shared memory; every thread of the block.
__device__ __forceinline__ void mol_stage(unsigned char *dst, const MolTerms *src, int bytes) {
    for (int q = threadIdx.x * 8; q < bytes; q += blockDim.x * 8) *(unsigned long long *)(dst + q) = *(const unsigned long long *)((const unsigned char *)src + q);
}

// All terms of the table tb, each once, by every thread of the block (the f64 table: T = double).  Forces: S[slot] = the
// term's force on that atom.  ENERGY (T = double): the term's energy goes to the slot of its owner -- the smaller atom index
// of a bond or pair, role 0 of an angle or torsion -- as the two factors x, y of its last product, so that the owner's sum
// e = fma(x, y, e) over its slots in slot order (mol_energy) rounds as one fused multiply-add per term; its other slots get 0.
// One alchemical pair at state st: *e its energy, *c = -dU/dr / r.
template <typename T>
__device__ __forceinline__ void mol_apair(const MolDev &m, const TAPair<T> &p, const double (*X)[3], const StateDev &st, T *e, T *c) {
    const T d[3] = {(T)(X[p.i][0] - X[p.j][0]), (T)(X[p.i][1] - X[p.j][1]), (T)(X[p.i][2] - X[p.j][2])};
    const T r2 = d[0] * d[0] + d[1] * d[1] + d[2] * d[2], ir2 = T(1) / r2, ir = mol_sqrt(ir2);
    const T la = p.ls ? (T)st.la : T(1), ob = p.ls ? (T)st.ob : T(0), le = p.le ? (T)st.lambda_e : T(1);
    const T u2 = r2 / (p.sig * p.sig);                                      // (r/sig)^2
    const T s = m.c6 ? u2 * u2 * u2 : (T)pow((double)u2, 0.5 * m.sc_c);   // (r/sig)^c
    const T x = m.c6 ? T(1) / (ob + s) : (T)pow((double)(ob + s), -6.0 / m.sc_c);
    const T qe = le * p.qq * ir, lj = la * T(4) * p.eps;
    *e = qe + lj * x * (x - T(1));
    *c = (qe + T(6) * lj * (T(2) * x - T(1)) * x * s / (ob + s)) * ir2;
}

// ALCH: the alchemical pairs too, at the state st (forces; ENERGY: their slots get 0, mol_alch_energy has their energy).
template <typename T, bool ENERGY, bool ALCH = false>
__device__ __forceinline__ void mol_terms(const MolDev &m, const unsigned char *tb, const double (*X)[3], T (*S)[3],
                                          const StateDev *st = nullptr) {
    const MolTerms *h = (const MolTerms *)tb;
    const int lane = threadIdx.x, nth = blockDim.x;   // (k_propagate_mol: all warps of the block; the other kernels: one warp)
    auto energy = [&](int s, bool own, T x, T y) { S[s][0] = own ? x : T(0); S[s][1] = own ? y : T(0); };
    const TBond<T> *B = (const TBond<T> *)(tb + h->o_bond);
    // (which thread evaluates a term does not matter for the result -- fixed slots; the four kinds start at different threads so
    // that no thread gets a torsion AND an angle AND two pairs: the evaluation is as long as its busiest thread)
    for (int t = (lane + nth / 2) % nth; t < m.n_tb; t += nth) {
        const TBond<T> b = B[t];
        const T d[3] = {(T)(X[b.i][0] - X[b.j][0]), (T)(X[b.i][1] - X[b.j][1]), (T)(X[b.i][2] - X[b.j][2])};
        const T r = mol_sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
        if (ENERGY) {
            const T dr = r - b.r0;
            energy(b.si, b.i < b.j, T(0.5) * b.K * dr, dr); energy(b.sj, b.j < b.i, T(0.5) * b.K * dr, dr);
        } else {
            const T c = -b.K * (r - b.r0) / r;
            for (int q = 0; q < 3; q++) { S[b.si][q] = c * d[q]; S[b.sj][q] = -c * d[q]; }
        }
    }
    const TAngle<T> *A = (const TAngle<T> *)(tb + h->o_angle);
    for (int t = nth - 1 - lane; t < m.n_ta; t += nth) {
        const TAngle<T> g = A[t];
        T u[3], v[3];
        for (int c = 0; c < 3; c++) { u[c] = (T)(X[g.i][c] - X[g.j][c]); v[c] = (T)(X[g.k][c] - X[g.j][c]); }
        const T ru2 = u[0] * u[0] + u[1] * u[1] + u[2] * u[2], rv2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
        const T iruv = mol_rsqrt(ru2 * rv2);
        const T cs = mol_clamp1((u[0] * v[0] + u[1] * v[1] + u[2] * v[2]) * iruv);
        const T dt = mol_acos(cs) - g.t0;
        if (ENERGY) {
            energy(g.si, true, T(0.5) * g.K * dt, dt); energy(g.sj, false, 0, 0); energy(g.sk, false, 0, 0);
        } else {
            const T sn = mol_sqrt(T(1) - cs * cs);
            const T gg = (sn > T(1e-6)) ? g.K * dt / sn : T(0);
            for (int c = 0; c < 3; c++) {
                const T fi = gg * (v[c] * iruv - cs * u[c] / ru2), fk = gg * (u[c] * iruv - cs * v[c] / rv2);
                S[g.si][c] = fi; S[g.sk][c] = fk; S[g.sj][c] = -(fi + fk);
            }
        }
    }
    const TTors<T> *W = (const TTors<T> *)(tb + h->o_tors);
    for (int t = lane; t < m.n_tt; t += nth) {
        const TTors<T> w = W[t];
        T rij[3], rkj[3], rkl[3], mm[3], nn[3];
        for (int c = 0; c < 3; c++) { rij[c] = (T)(X[w.i][c] - X[w.j][c]); rkj[c] = (T)(X[w.k][c] - X[w.j][c]); rkl[c] = (T)(X[w.k][c] - X[w.l][c]); }
        mm[0] = rij[1] * rkj[2] - rij[2] * rkj[1]; mm[1] = rij[2] * rkj[0] - rij[0] * rkj[2]; mm[2] = rij[0] * rkj[1] - rij[1] * rkj[0];
        nn[0] = rkj[1] * rkl[2] - rkj[2] * rkl[1]; nn[1] = rkj[2] * rkl[0] - rkj[0] * rkl[2]; nn[2] = rkj[0] * rkl[1] - rkj[1] * rkl[0];
        const T rkj2 = rkj[0] * rkj[0] + rkj[1] * rkj[1] + rkj[2] * rkj[2], nrkj = mol_sqrt(rkj2);
        const T phi = mol_atan2(nrkj * (rij[0] * nn[0] + rij[1] * nn[1] + rij[2] * nn[2]), mm[0] * nn[0] + mm[1] * nn[1] + mm[2] * nn[2]);
        T sn, cs;
        mol_sincos(w.n * phi - w.phase, &sn, &cs);
        if (ENERGY) {
            energy(w.si, true, w.kk, T(1) + cs); energy(w.sj, false, 0, 0); energy(w.sk, false, 0, 0); energy(w.sl, false, 0, 0);
        } else {
            const T dU = -w.kk * w.n * sn;
            const T m2 = mm[0] * mm[0] + mm[1] * mm[1] + mm[2] * mm[2], n2 = nn[0] * nn[0] + nn[1] * nn[1] + nn[2] * nn[2];
            const T pp = (rij[0] * rkj[0] + rij[1] * rkj[1] + rij[2] * rkj[2]) / rkj2, qq = (rkl[0] * rkj[0] + rkl[1] * rkj[1] + rkl[2] * rkj[2]) / rkj2;
            const T ci = -dU * nrkj / m2, cl = dU * nrkj / n2;
            for (int c = 0; c < 3; c++) {
                const T fi = ci * mm[c], fl = cl * nn[c], sv = pp * fi - qq * fl;
                S[w.si][c] = fi; S[w.sj][c] = sv - fi; S[w.sk][c] = -sv - fl; S[w.sl][c] = fl;
            }
        }
    }
    const TPair<T> *P = (const TPair<T> *)(tb + h->o_pair);
    for (int t = ((lane - m.n_tt) % nth + nth) % nth; t < m.n_tp; t += nth) {
        const TPair<T> p = P[t];
        const T d[3] = {(T)(X[p.i][0] - X[p.j][0]), (T)(X[p.i][1] - X[p.j][1]), (T)(X[p.i][2] - X[p.j][2])};
        const T ir2 = T(1) / (d[0] * d[0] + d[1] * d[1] + d[2] * d[2]), ir = mol_sqrt(ir2);
        const T s2 = p.sig * p.sig * ir2, s6 = s2 * s2 * s2;
        if (ENERGY) {
            const T e = p.qq * ir + T(4) * p.eps * (s6 * s6 - s6);
            energy(p.si, p.i < p.j, e, 1); energy(p.sj, p.j < p.i, e, 1);
        } else {
            const T c = (p.qq * ir + T(24) * p.eps * (T(2) * s6 * s6 - s6)) * ir2;
            for (int q = 0; q < 3; q++) { S[p.si][q] = c * d[q]; S[p.sj][q] = -c * d[q]; }
        }
    }
    if (!ALCH) return;
    const TAPair<T> *AP = (const TAPair<T> *)(tb + h->o_apair);
    for (int t = lane; t < m.n_tap; t += nth) {
        const TAPair<T> p = AP[t];
        if (ENERGY) { energy(p.si, false, 0, 0); energy(p.sj, false, 0, 0); continue; }
        T e, c;
        mol_apair<T>(m, p, X, *st, &e, &c);
        const T d[3] = {(T)(X[p.i][0] - X[p.j][0]), (T)(X[p.i][1] - X[p.j][1]), (T)(X[p.i][2] - X[p.j][2])};
        for (int q = 0; q < 3; q++) { S[p.si][q] = c * d[q]; S[p.sj][q] = -c * d[q]; }
    }
}

// The alchemical pairs' energy at state st, summed by each warp over its lanes in a fixed order (every warp gets the same
// bits, whatever the block size).
__device__ __forceinline__ double mol_alch_energy(const MolDev &m, const unsigned char *t64, const double (*X)[3],
                                                  const StateDev &st) {
    const TAPair<double> *AP = (const TAPair<double> *)(t64 + ((const MolTerms *)t64)->o_apair);
    double e = 0.0;
    for (int t = threadIdx.x & 31; t < m.n_tap; t += 32) {
        double et, c;
        mol_apair<double>(m, AP[t], X, st, &et, &c);
        e += et;
    }
    return mol_warp_sum(e);
}

// Constraints are solved per cluster (connected component of the constraint graph) by ONE lane.  Clusters of up to
// MOL_MAXC constraints (a CH3 group has three) are solved as a whole: the velocity conditions are a linear system in the
// multipliers (one solve), the position conditions are solved by Newton iterations on the same coupled system
// (M-SHAKE: converges quadratically, 2-3 iterations where Gauss-Seidel sweeps need ~10).  Larger clusters fall back to
// Gauss-Seidel sweeps.  Both reach the same constrained point to the tolerance (the oracle uses sweeps).
#define MOL_MAXC 4

struct MolCluster {       // one lane's cluster, in registers / local memory for the whole kernel
    int nc;
    int i[MOL_MAXC], j[MOL_MAXC];
    double d2[MOL_MAXC], wi[MOL_MAXC], wj[MOL_MAXC];
    double coup[MOL_MAXC][MOL_MAXC];   // mass coupling of constraints c and d (see mol_load_cluster)
};

__device__ __forceinline__ void mol_load_cluster(const MolDev &m, int c, MolCluster &k) {
    const int q0 = m.c_off[c];
    k.nc = m.c_off[c + 1] - q0;
    // (static indices only, so that the whole record lives in registers)
#pragma unroll
    for (int a = 0; a < MOL_MAXC; a++) {
        const bool on = a < k.nc && k.nc <= MOL_MAXC;
        const MolCons s = on ? m.cons[q0 + a] : MolCons{0, 0, 1.0};
        k.i[a] = s.i; k.j[a] = s.j; k.d2[a] = s.d * s.d;
        k.wi[a] = on ? 1.0 / m.mass[s.i] : 0.0; k.wj[a] = on ? 1.0 / m.mass[s.j] : 0.0;
    }
    // a unit multiplier on constraint d moves x_i(d) by +w r_d and x_j(d) by -w r_d: its effect on the bond vector of c
#pragma unroll
    for (int a = 0; a < MOL_MAXC; a++)
#pragma unroll
        for (int b = 0; b < MOL_MAXC; b++) {
            double v = 0.0;
            if (k.i[a] == k.i[b]) v += k.wi[a];
            if (k.i[a] == k.j[b]) v -= k.wi[a];
            if (k.j[a] == k.i[b]) v -= k.wj[a];
            if (k.j[a] == k.j[b]) v += k.wj[a];
            k.coup[a][b] = v;
        }
}

// solve A g = b in place (A: NC x NC, diagonally dominant here), result in b; fully unrolled: everything stays in registers
template <int NC>
__device__ __forceinline__ void mol_solve(double (*A)[MOL_MAXC], double *b) {
#pragma unroll
    for (int p = 0; p < NC; p++) {
        const double ip = 1.0 / A[p][p];
#pragma unroll
        for (int r = p + 1; r < NC; r++) {
            const double f = A[r][p] * ip;
#pragma unroll
            for (int c = p; c < NC; c++) A[r][c] -= f * A[p][c];
            b[r] -= f * b[p];
        }
    }
#pragma unroll
    for (int p = NC - 1; p >= 0; p--) {
        double v = b[p];
#pragma unroll
        for (int c = p + 1; c < NC; c++) v -= A[p][c] * b[c];
        b[p] = v / A[p][p];
    }
}

// SHAKE on a cluster of NC constraints: Newton iterations on the coupled system (M-SHAKE).
template <int NC>
__device__ __forceinline__ void mol_shake_n(const MolDev &m, const MolCluster &k, const double (*XO)[3], double (*X)[3]) {
    double r0[MOL_MAXC][3];
#pragma unroll
    for (int a = 0; a < NC; a++)
#pragma unroll
        for (int q = 0; q < 3; q++) r0[a][q] = XO[k.i[a]][q] - XO[k.j[a]][q];
    for (int it = 0; it < 50; it++) {
        double A[MOL_MAXC][MOL_MAXC], g[MOL_MAXC], r[MOL_MAXC][3];
        bool done = true;
#pragma unroll
        for (int a = 0; a < NC; a++) {
#pragma unroll
            for (int q = 0; q < 3; q++) r[a][q] = X[k.i[a]][q] - X[k.j[a]][q];
            g[a] = k.d2[a] - mol_dot(r[a], r[a]);
            if (fabs(g[a]) > m.tol * k.d2[a]) done = false;
        }
        if (done) break;
#pragma unroll
        for (int a = 0; a < NC; a++)
#pragma unroll
            for (int b = 0; b < NC; b++) A[a][b] = 2.0 * k.coup[a][b] * mol_dot(r[a], r0[b]);
        mol_solve<NC>(A, g);
#pragma unroll
        for (int b = 0; b < NC; b++)
#pragma unroll
            for (int q = 0; q < 3; q++) { X[k.i[b]][q] += g[b] * k.wi[b] * r0[b][q]; X[k.j[b]][q] -= g[b] * k.wj[b] * r0[b][q]; }
    }
}

// RATTLE on a cluster of NC constraints: one linear solve.
template <int NC>
__device__ __forceinline__ void mol_rattle_n(const MolCluster &k, const double (*X)[3], double (*V)[3]) {
    double A[MOL_MAXC][MOL_MAXC], g[MOL_MAXC], r[MOL_MAXC][3];
#pragma unroll
    for (int a = 0; a < NC; a++) {
        double dv[3];
#pragma unroll
        for (int q = 0; q < 3; q++) { r[a][q] = X[k.i[a]][q] - X[k.j[a]][q]; dv[q] = V[k.i[a]][q] - V[k.j[a]][q]; }
        g[a] = mol_dot(r[a], dv);
    }
#pragma unroll
    for (int a = 0; a < NC; a++)
#pragma unroll
        for (int b = 0; b < NC; b++) A[a][b] = k.coup[a][b] * mol_dot(r[a], r[b]);
    mol_solve<NC>(A, g);
#pragma unroll
    for (int b = 0; b < NC; b++)
#pragma unroll
        for (int q = 0; q < 3; q++) { V[k.i[b]][q] -= g[b] * k.wi[b] * r[b][q]; V[k.j[b]][q] += g[b] * k.wj[b] * r[b][q]; }
}

// SHAKE on one cluster: positions X moved so that its constraints have their lengths, along the bond vectors of XO.
__device__ __forceinline__ void mol_shake_cluster(const MolDev &m, int c, const MolCluster &k, const double (*XO)[3], double (*X)[3]) {
    switch (k.nc) {
        case 1: mol_shake_n<1>(m, k, XO, X); return;
        case 2: mol_shake_n<2>(m, k, XO, X); return;
        case 3: mol_shake_n<3>(m, k, XO, X); return;
        case 4: mol_shake_n<4>(m, k, XO, X); return;
        default: break;
    }
    for (int it = 0; it < 500; it++) {
        bool done = true;
        for (int q = m.c_off[c]; q < m.c_off[c + 1]; q++) {
            const MolCons s = m.cons[q];
            const double d2 = s.d * s.d;
            double r[3], r0[3];
            for (int a = 0; a < 3; a++) { r[a] = X[s.i][a] - X[s.j][a]; r0[a] = XO[s.i][a] - XO[s.j][a]; }
            const double diff = d2 - mol_dot(r, r);
            if (fabs(diff) > m.tol * d2) {
                done = false;
                const double wi = 1.0 / m.mass[s.i], wj = 1.0 / m.mass[s.j];
                const double g = diff / (2.0 * (wi + wj) * mol_dot(r, r0));
                for (int a = 0; a < 3; a++) { X[s.i][a] += g * wi * r0[a]; X[s.j][a] -= g * wj * r0[a]; }
            }
        }
        if (done) break;
    }
}

// RATTLE on one cluster: the velocity components along its constraints are removed.  unit: unit weights instead of 1/m
// (the minimiser's projection; clusters of <= MOL_MAXC constraints carry their weights in k).
__device__ __forceinline__ void mol_rattle_cluster(const MolDev &m, int c, const MolCluster &k, const double (*X)[3], double (*V)[3],
                                                   bool unit = false) {
    switch (k.nc) {
        case 1: mol_rattle_n<1>(k, X, V); return;
        case 2: mol_rattle_n<2>(k, X, V); return;
        case 3: mol_rattle_n<3>(k, X, V); return;
        case 4: mol_rattle_n<4>(k, X, V); return;
        default: break;
    }
    for (int it = 0; it < 500; it++) {
        bool done = true;
        for (int q = m.c_off[c]; q < m.c_off[c + 1]; q++) {
            const MolCons s = m.cons[q];
            double r[3], dv[3];
            for (int a = 0; a < 3; a++) { r[a] = X[s.i][a] - X[s.j][a]; dv[a] = V[s.i][a] - V[s.j][a]; }
            const double rv = mol_dot(r, dv), r2 = mol_dot(r, r);
            if (fabs(rv) > m.tol * r2) {
                done = false;
                const double wi = unit ? 1.0 : 1.0 / m.mass[s.i], wj = unit ? 1.0 : 1.0 / m.mass[s.j];
                const double g = rv / ((wi + wj) * r2);
                for (int a = 0; a < 3; a++) { V[s.i][a] -= g * wi * r[a]; V[s.j][a] += g * wj * r[a]; }
            }
        }
        if (done) break;
    }
}

// --- k_propagate_mol's constraint path for clusters of up to three constraints (every H-bond cluster: XH, XH2, XH3; a rigid
// water) ------------------------------------------------------------------------------------------------------------------
// A connected cluster of nc <= 3 constraints has at most 4 atoms: the lane that owns the cluster works on register copies of
// those atoms -- one load and one store per atom and call, nothing read back from shared memory in between (the coupled
// updates of the shared heavy atom were three dependent read-modify-writes per component before).  The geometry is two small
// coefficient tables: E[b][n] (+1, -1, 0: bond vector of constraint b = sum_n E x_n) and S[n][b] (+1/m_i, -1/m_j, 0: a unit
// multiplier on constraint b moves atom n by S r_b).
// The RATTLE matrix A = coup o (r r^T), coup = E S, depends on the positions only, and positions change in the R operations
// only: its inverse is formed ONCE per position update (closed form, one reciprocal) and serves the two to three velocity
// projections that follow as a matrix-vector product -- no pivoting, no division on the step's critical path.  SHAKE iterates
// with the same inverse (the Jacobian at the previous constrained positions is 2 A: a chord iteration; the bond vectors turn
// by about 1e-2 per R operation, so every iteration gains 1.5-2 digits), entirely in registers: 3 dot products and a 3x3
// product per iteration instead of a Newton solve.  Clusters with fewer constraints / atoms are padded (zero coefficients,
// unit diagonal): one instruction stream for all lanes.  Same constrained point as mol_shake_n / the oracle's sweeps to the
// tolerance.
struct MolStar {
    int nc, na;
    int idx[4];          // the cluster's atoms (padded with its first atom: read, never written)
    double S[4][3];
    float E[3][4];
    double d2[3];
    double coup[3][3];
    double r[3][3];      // bond vectors at the last constrained positions
    double Ai[3][3];     // inverse of coup o (r r^T)
};

__device__ __forceinline__ void mol_star_load(const MolDev &m, int c, MolStar &k) {
    const int q0 = m.c_off[c];
    k.nc = m.c_off[c + 1] - q0;
    int ci[3], cj[3], at[4] = {-1, -1, -1, -1}, na = 0;
    double wi[3], wj[3];
    // (static indices only, so that the whole record lives in registers)
#pragma unroll
    for (int a = 0; a < 3; a++) {
        const bool on = a < k.nc;
        const MolCons s = on ? m.cons[q0 + a] : MolCons{-1, -1, 1.0};
        ci[a] = s.i; cj[a] = s.j; k.d2[a] = s.d * s.d;
        wi[a] = on ? 1.0 / m.mass[s.i] : 0.0; wj[a] = on ? 1.0 / m.mass[s.j] : 0.0;
    }
#pragma unroll
    for (int a = 0; a < 3; a++)
#pragma unroll
        for (int e = 0; e < 2; e++) {
            const int atom = e ? cj[a] : ci[a];
            bool found = atom < 0;
#pragma unroll
            for (int n = 0; n < 4; n++) found |= at[n] == atom;
            if (!found) {
#pragma unroll
                for (int n = 0; n < 4; n++) if (n == na) at[n] = atom;
                na++;
            }
        }
    k.na = na;
#pragma unroll
    for (int n = 0; n < 4; n++) {
        k.idx[n] = n < na ? at[n] : at[0];
#pragma unroll
        for (int b = 0; b < 3; b++) {
            const bool is_i = at[n] >= 0 && at[n] == ci[b], is_j = at[n] >= 0 && at[n] == cj[b];
            k.S[n][b] = (is_i ? wi[b] : 0.0) - (is_j ? wj[b] : 0.0);
            k.E[b][n] = (float)((int)is_i - (int)is_j);
        }
    }
#pragma unroll
    for (int a = 0; a < 3; a++)
#pragma unroll
        for (int b = 0; b < 3; b++) {
            double v = 0.0;
#pragma unroll
            for (int n = 0; n < 4; n++) v += (double)k.E[a][n] * k.S[n][b];
            k.coup[a][b] = v;
        }
}

__device__ __forceinline__ void mol_star_invert(MolStar &k) {
    double A[3][3];
#pragma unroll
    for (int a = 0; a < 3; a++)
#pragma unroll
        for (int b = 0; b < 3; b++) A[a][b] = (a == b && a >= k.nc) ? 1.0 : k.coup[a][b] * mol_dot(k.r[a], k.r[b]);
    const double c00 = A[1][1] * A[2][2] - A[1][2] * A[2][1], c01 = A[1][0] * A[2][2] - A[1][2] * A[2][0],
                 c02 = A[1][0] * A[2][1] - A[1][1] * A[2][0];
    const double id = 1.0 / (A[0][0] * c00 - A[0][1] * c01 + A[0][2] * c02);
    k.Ai[0][0] = c00 * id;
    k.Ai[0][1] = (A[0][2] * A[2][1] - A[0][1] * A[2][2]) * id;
    k.Ai[0][2] = (A[0][1] * A[1][2] - A[0][2] * A[1][1]) * id;
    k.Ai[1][0] = -c01 * id;
    k.Ai[1][1] = (A[0][0] * A[2][2] - A[0][2] * A[2][0]) * id;
    k.Ai[1][2] = (A[0][2] * A[1][0] - A[0][0] * A[1][2]) * id;
    k.Ai[2][0] = c02 * id;
    k.Ai[2][1] = (A[0][1] * A[2][0] - A[0][0] * A[2][1]) * id;
    k.Ai[2][2] = (A[0][0] * A[1][1] - A[0][1] * A[1][0]) * id;
}

// bond vectors of the cluster's constraints from register copies of its atoms
__device__ __forceinline__ void mol_star_bonds(const MolStar &k, const double (*x)[3], double (*rb)[3]) {
#pragma unroll
    for (int a = 0; a < 3; a++)
#pragma unroll
        for (int q = 0; q < 3; q++) {
            double v = 0.0;
#pragma unroll
            for (int n = 0; n < 4; n++) v += (double)k.E[a][n] * x[n][q];
            rb[a][q] = v;
        }
}

__device__ __forceinline__ void mol_star_init(MolStar &k, const double (*X)[3]) {
    double x[4][3];
#pragma unroll
    for (int n = 0; n < 4; n++)
#pragma unroll
        for (int q = 0; q < 3; q++) x[n][q] = X[k.idx[n]][q];
    mol_star_bonds(k, x, k.r);
    mol_star_invert(k);
}

__device__ __forceinline__ void mol_star_rattle(const MolStar &k, double (*V)[3]) {
    double v[4][3], dv[3][3], g[3], lam[3];
#pragma unroll
    for (int n = 0; n < 4; n++)
#pragma unroll
        for (int q = 0; q < 3; q++) v[n][q] = V[k.idx[n]][q];
    mol_star_bonds(k, v, dv);
#pragma unroll
    for (int a = 0; a < 3; a++) g[a] = mol_dot(k.r[a], dv[a]);
#pragma unroll
    for (int b = 0; b < 3; b++) lam[b] = k.Ai[b][0] * g[0] + k.Ai[b][1] * g[1] + k.Ai[b][2] * g[2];
#pragma unroll
    for (int n = 0; n < 4; n++)
        if (n < k.na) {
#pragma unroll
            for (int q = 0; q < 3; q++)
                V[k.idx[n]][q] = v[n][q] - (k.S[n][0] * lam[0] * k.r[0][q] + k.S[n][1] * lam[1] * k.r[1][q] + k.S[n][2] * lam[2] * k.r[2][q]);
        }
}

// positions X (moved from the constrained positions the cache was built at) back onto the constraints, along the cached bond
// vectors; the cache is rebuilt at the result.
__device__ __forceinline__ void mol_star_shake(const MolDev &m, MolStar &k, double (*X)[3]) {
    double x[4][3], rc[3][3];
#pragma unroll
    for (int n = 0; n < 4; n++)
#pragma unroll
        for (int q = 0; q < 3; q++) x[n][q] = X[k.idx[n]][q];
    for (int it = 0; it < 60; it++) {
        double g[3], lam[3];
        bool done = true;
        mol_star_bonds(k, x, rc);
#pragma unroll
        for (int a = 0; a < 3; a++) {
            g[a] = a < k.nc ? k.d2[a] - mol_dot(rc[a], rc[a]) : 0.0;
            if (fabs(g[a]) > m.tol * k.d2[a]) done = false;
        }
        if (done) break;
#pragma unroll
        for (int b = 0; b < 3; b++) lam[b] = 0.5 * (k.Ai[b][0] * g[0] + k.Ai[b][1] * g[1] + k.Ai[b][2] * g[2]);
#pragma unroll
        for (int n = 0; n < 4; n++)
#pragma unroll
            for (int q = 0; q < 3; q++)
                x[n][q] += k.S[n][0] * lam[0] * k.r[0][q] + k.S[n][1] * lam[1] * k.r[1][q] + k.S[n][2] * lam[2] * k.r[2][q];
    }
#pragma unroll
    for (int n = 0; n < 4; n++)
        if (n < k.na) {
#pragma unroll
            for (int q = 0; q < 3; q++) X[k.idx[n]][q] = x[n][q];
        }
#pragma unroll
    for (int a = 0; a < 3; a++)
#pragma unroll
        for (int q = 0; q < 3; q++) k.r[a][q] = rc[a][q];
    mol_star_invert(k);
}

// The GB terms, pair-parallel over the block, in the arrays of MolGB::prop_bytes: n x n matrices I_ij, dI_ij/dr, the pair's
// dE/dr / r (symmetric; ENERGY: the pair's energy for j > i) and dE_pair/dB_i, then B_i, dB_i/dI_i and C_i = dE/dB_i dB_i/dI_i.
// Every entry is written by one thread and every atom adds up its row in index order: no atomics, the same bits whatever the
// thread count.
struct MolGBArrays {
    double *I, *D, *P, *EB, *B, *dB, *C;
    __device__ MolGBArrays(double *s, int n) : I(s), D(s + n * n), P(s + 2 * n * n), EB(s + 3 * n * n), B(s + 4 * n * n), dB(B + n), C(dB + n) {}
};

// phase 1 (before the barrier that ends the term evaluation): the descreening integrals of the ordered pairs.  ALCH: at
// lambda_electrostatics le of the alchemical molecule m, j's descreening of i weighted by w_j (I and dI/dr alike).
template <bool ENERGY, bool ALCH = false>
__device__ __forceinline__ void mol_gb_integrals(const MolGB &g, const double (*X)[3], int n, const MolGBArrays &s,
                                                 const MolDev *m = nullptr, double le = 1.0) {
    for (int t = threadIdx.x; t < n * n; t += blockDim.x) {
        const int i = t / n, j = t - i * n;
        double d[3], dI = 0.0, I = 0.0;
        if (i != j) I = gb_descreen(gb_dist(X, i, j, d), g.atom[4 * i], g.atom[4 * j + 1], &dI, ALCH && g.engulf);
        if (ALCH) { const double w = mol_w(*m, j, le); I *= w; dI *= w; }
        s.I[t] = I;
        if (!ENERGY) s.D[t] = dI;
    }
}

// phases 2 and 3 (after it; every thread of the block): Born radii, the pair terms, then the chain-rule factors C_i or, ENERGY,
// the GB energy atom a < n owns (returned): its self and ACE terms, then its pairs with larger partners in index order.
// ALCH: the pair term with charges w_i q_i, w_j q_j, the self and ACE terms of atom a scaled by w_a.
template <bool ENERGY, bool ALCH = false>
__device__ __forceinline__ double mol_gb_radii_pairs(const MolGB &g, const double (*X)[3], const double *q, int n, const MolGBArrays &s,
                                                     const MolDev *m = nullptr, double le = 1.0) {
    const int a = threadIdx.x;
    if (a < n) {
        double I = 0.0, dB;
        for (int j = 0; j < n; j++) I += s.I[a * n + j];
        s.B[a] = gb_born(g, I, g.atom[4 * a], g.atom[4 * a + 2], &dB);
        if (!ENERGY) s.dB[a] = dB;
    }
    __syncthreads();
    for (int t = threadIdx.x; t < n * n; t += blockDim.x) {
        const int i = t / n, j = t - i * n;
        if (j <= i) continue;
        double d[3], dr, dbi, dbj;
        const double r = gb_dist(X, i, j, d);
        const double pqq = ALCH ? g.pre * (mol_w(*m, i, le) * q[i]) * (mol_w(*m, j, le) * q[j]) : g.pre * q[i] * q[j];
        const double e = gb_pair(r * r, s.B[i], s.B[j], pqq, &dr, &dbi, &dbj);
        if (ENERGY) s.P[t] = e;
        else { s.P[t] = s.P[j * n + i] = dr; s.EB[t] = dbi; s.EB[j * n + i] = dbj; }
    }
    __syncthreads();
    double e = 0.0;
    if (a < n) {
        double dEdB;
        e = gb_self(g, q[a], s.B[a], g.atom[4 * a + 2], g.atom[4 * a + 3], &dEdB);
        if (ALCH) { const double w = mol_w(*m, a, le); e *= w; dEdB *= w; }
        if (ENERGY) {
            for (int j = a + 1; j < n; j++) e += s.P[a * n + j];
        } else {
            for (int j = 0; j < n; j++) if (j != a) dEdB += s.EB[a * n + j];
            s.C[a] = dEdB * s.dB[a];
        }
    }
    __syncwarp();
    return e;
}

// the GB force on atom a (warp 0, after mol_gb_radii_pairs)
__device__ __forceinline__ void mol_gb_force(const double (*X)[3], int a, int n, const MolGBArrays &s, double *f) {
    for (int j = 0; j < n; j++) {
        if (j == a) continue;
        double d[3];
        const double r = gb_dist(X, a, j, d);
        const double c = s.P[a * n + j] + (s.C[a] * s.D[a * n + j] + s.C[j] * s.D[j * n + a]) / r;
        for (int q = 0; q < 3; q++) f[q] -= c * d[q];
    }
}

// The lambda-independent part of an alchemical molecule's U: every term of the table but the alchemical pairs.  Every thread
// of the block, after a block barrier; the result is warp 0's.
__device__ __forceinline__ double mol_energy_fixed(const MolDev &m, const unsigned char *t64, const double (*X)[3], double (*S)[3]) {
    mol_terms<double, true, true>(m, t64, X, S);
    __syncthreads();
    const int a = threadIdx.x, *goff = (const int *)(t64 + ((const MolTerms *)t64)->o_goff);
    double e = 0.0;
    if (a < m.n)
        for (int q = goff[a]; q < goff[a + 1]; q++) e = fma(S[q][0], S[q][1], e);
    return mol_warp_sum(a < m.n ? e : 0.0);
}

// The alchemical OBC energy at lambda_electrostatics le (every thread of the block; warp 0's result).
__device__ __forceinline__ double mol_energy_gb(const MolDev &m, const MolGB &g, const double (*X)[3], const MolGBArrays &gs, double le) {
    __syncthreads();   // (the arrays may still be read by the previous evaluation)
    mol_gb_integrals<true, true>(g, X, m.n, gs, &m, le);
    __syncthreads();
    const double e = mol_gb_radii_pairs<true, true>(g, X, m.charge, m.n, gs, &m, le);
    return mol_warp_sum(threadIdx.x < m.n ? e : 0.0);
}

// U of the molecule at X from the f64 term table t64, in k_energy_mol and at the end of k_propagate_mol (the same function:
// the same bits).  Every thread of the block calls it after a block barrier; S: double[n_slots][3] with, GB, the arrays of gs
// behind them.  The result is warp 0's.
// ALCH: U at the state st, mol_energy_fixed + (mol_energy_gb + mol_alch_energy) -- k_energy_mol evaluates the same functions
// and adds them in the same order, re-evaluating only the lambda-dependent ones per state.
template <bool GB, bool ALCH = false>
__device__ __forceinline__ double mol_energy(const MolDev &m, const MolGB &g, const unsigned char *t64, const double (*X)[3],
                                             double (*S)[3], const MolGBArrays &gs, const StateDev *st = nullptr) {
    if (ALCH) {
        const double u0 = mol_energy_fixed(m, t64, X, S);
        return u0 + ((GB ? mol_energy_gb(m, g, X, gs, st->lambda_e) : 0.0) + mol_alch_energy(m, t64, X, *st));
    }
    mol_terms<double, true>(m, t64, X, S);
    if (GB) mol_gb_integrals<true>(g, X, m.n, gs);
    __syncthreads();
    const double e_gb = GB ? mol_gb_radii_pairs<true>(g, X, m.charge, m.n, gs) : 0.0;
    const int a = threadIdx.x, *goff = (const int *)(t64 + ((const MolTerms *)t64)->o_goff);
    double e = 0.0;
    if (a < m.n)
        for (int q = goff[a]; q < goff[a + 1]; q++) e = fma(S[q][0], S[q][1], e);
    return mol_warp_sum(a < m.n ? (GB ? e + e_gb : e) : 0.0);
}

// One block of MOL_WARPS warps per owned replica.  Warp 0 integrates (one lane per atom, one lane per constraint cluster);
// all warps evaluate the force terms (each term once, by whichever thread its index falls to, into its fixed slots: the
// per-atom sums in slot order do not depend on the number of threads -- the same bits as with one warp), between two block
// barriers per force evaluation.  Every warp runs the same control flow (steps, program, lazy force flag); warps 1.. only take
// part in the force evaluations.  pos / vel: double[kloc][n][3].
#define MOL_WARPS 4
// STAR: every constraint cluster has at most three constraints (MolDev::max_cluster): the MolStar path.
// GB: OBC implicit solvent (g), three phases per force evaluation: the descreening integrals with the other terms, then
// (a block barrier) Born radii, (barrier) pair terms, (barrier) chain-rule factors, then each atom's sum.
// mv: the move, __grid_constant__ so that the program is indexed in the parameter bank (a plain by-value struct of this
// size is copied to local memory).  `reassign` stays an argument: read from mv, it costs this kernel 40-250 instructions.
// ALCH: an alchemical molecule (MolDev::n_tap, alch) at the lambdas of the replica's state.
template <bool STAR, bool GB, bool ALCH>
__global__ void __launch_bounds__(32 * MOL_WARPS) k_propagate_mol(MolDev m, const __grid_constant__ MoveDev mv, const StateDev *__restrict__ states,
                                                      const int *__restrict__ perm, double *__restrict__ pos,
                                                      double *__restrict__ vel, int k0, uint2 key, uint32_t iteration,
                                                      int reassign, double *__restrict__ pot, double *__restrict__ kin,
                                                      int *__restrict__ nan_flag, const int *__restrict__ only, MolGB g) {
    __shared__ double X[MOL_MAX_ATOMS][3], XO[MOL_MAX_ATOMS][3], V[MOL_MAX_ATOMS][3];
    extern __shared__ unsigned long long mol_tab[];
    const int r = blockIdx.x, k = k0 + r, a = threadIdx.x, n = m.n;
    if (only && !only[k]) return;
    // the f32 term table and the slots of its force contributions
    unsigned char *tb = (unsigned char *)mol_tab;
    mol_stage(tb, m.terms32, m.bytes32);
    float (*FS)[3] = (float (*)[3])(tb + mol_slots_at(m, true));
    const MolGBArrays gs((double *)(tb + mol_gb_at(m, true)), n);
    __syncthreads();
    const int *g_off = (const int *)(tb + ((const MolTerms *)tb)->o_goff);
    const bool active = a < n;
    const StateDev st = states[perm[k]];
    const double mass = active ? m.mass[a] : 1.0, sg = sqrt(st.kT / mass);
    const double inv_mt = 1.0 / mol_warp_sum(active ? mass : 0.0);
    if (active) {
        for (int c = 0; c < 3; c++) { X[a][c] = pos[((size_t)r * n + a) * 3 + c]; V[a][c] = vel[((size_t)r * n + a) * 3 + c]; }
        if (reassign) {   // context.setVelocitiesToTemperature, mcmc.py:711
            const float3 g = philox_normal3(philox4x32_10(make_uint4(a, 0x80000000u, k, iteration), key));
            V[a][0] = sg * g.x; V[a][1] = sg * g.y; V[a][2] = sg * g.z;
        }
    }
    MolCluster kc;
    MolStar ks;
    kc.nc = 0;
    const bool has_c = a < m.n_clusters;
    if (has_c) { if (STAR) mol_star_load(m, a, ks); else mol_load_cluster(m, a, kc); }
    __syncwarp();
    // incoming velocities obey the constraints
    if (has_c) { if (STAR) { mol_star_init(ks, X); mol_star_rattle(ks, V); } else mol_rattle_cluster(m, a, kc, X, V); }
    __syncwarp();
    const double inv_mass = 1.0 / mass;
    // (the program is interpreted, so the compiler does not hoist these out of the step loop: two f64 divisions per R)
    const double hm = mv.dt_d / mv.nV * inv_mass, h = mv.dt_d / mv.nR, inv_h = 1.0 / h;
    double f[3] = {0, 0, 0};
    bool f_valid = false;
    uint32_t ocount = 0;
    for (int s = 0; s < mv.n_steps; s++) {
        if (m.remove_cm) {
            double px = mol_warp_sum(active ? mass * V[a][0] : 0.0), py = mol_warp_sum(active ? mass * V[a][1] : 0.0),
                   pz = mol_warp_sum(active ? mass * V[a][2] : 0.0);
            if (active) { V[a][0] -= px * inv_mt; V[a][1] -= py * inv_mt; V[a][2] -= pz * inv_mt; }
            __syncwarp();
        }
        for (int q = 0; q < mv.n_prog; q++) {
            const char op = mv.prog[q];
            if (op == 'V') {
                if (!f_valid) {
                    __syncthreads();   // warp 0's positions are in shared memory
                    mol_terms<float, false, ALCH>(m, tb, X, FS, &st);
                    if (GB) mol_gb_integrals<false, ALCH>(g, X, n, gs, &m, st.lambda_e);
                    __syncthreads();   // every term's contributions are in their slots
                    if (GB) mol_gb_radii_pairs<false, ALCH>(g, X, m.charge, n, gs, &m, st.lambda_e);
                    if (active) {   // this atom's slots, in slot order
                        float fx = 0.f, fy = 0.f, fz = 0.f;
                        for (int q = g_off[a]; q < g_off[a + 1]; q++) { fx += FS[q][0]; fy += FS[q][1]; fz += FS[q][2]; }
                        f[0] = fx; f[1] = fy; f[2] = fz;
                        if (GB) mol_gb_force(X, a, n, gs, f);
                    }
                    __syncwarp();
                    f_valid = true;
                }
                if (active) for (int c = 0; c < 3; c++) V[a][c] += hm * f[c];
                __syncwarp();
                if (has_c) { if (STAR) mol_star_rattle(ks, V); else mol_rattle_cluster(m, a, kc, X, V); }
                __syncwarp();
            } else if (op == 'R') {
                double xu[3] = {0, 0, 0};
                if (active) for (int c = 0; c < 3; c++) { XO[a][c] = X[a][c]; X[a][c] += h * V[a][c]; xu[c] = X[a][c]; }
                __syncwarp();
                if (m.n_clusters) {
                    if (has_c) { if (STAR) mol_star_shake(m, ks, X); else mol_shake_cluster(m, a, kc, XO, X); }
                    __syncwarp();
                    if (active) for (int c = 0; c < 3; c++) V[a][c] += (X[a][c] - xu[c]) * inv_h;
                    __syncwarp();
                    if (has_c) { if (STAR) mol_star_rattle(ks, V); else mol_rattle_cluster(m, a, kc, X, V); }
                    __syncwarp();
                }
                f_valid = false;
            } else {   // 'O'
                if (active) {
                    const float3 g = philox_normal3(philox4x32_10(make_uint4(a, ocount, k, iteration), key));
                    V[a][0] = mv.a_d * V[a][0] + mv.b_d * sg * (double)g.x;
                    V[a][1] = mv.a_d * V[a][1] + mv.b_d * sg * (double)g.y;
                    V[a][2] = mv.a_d * V[a][2] + mv.b_d * sg * (double)g.z;
                }
                ocount++;
                __syncwarp();
                if (has_c) { if (STAR) mol_star_rattle(ks, V); else mol_rattle_cluster(m, a, kc, X, V); }
                __syncwarp();
            }
        }
    }
    __syncthreads();   // warp 0's final positions; the force slots are free for the energy's
    const double U = mol_energy<GB, ALCH>(m, g, (const unsigned char *)m.terms64, X, (double (*)[3])FS, gs, &st);
    const double KE = mol_warp_sum(active ? 0.5 * mass * (V[a][0] * V[a][0] + V[a][1] * V[a][1] + V[a][2] * V[a][2]) : 0.0);
    const bool bad = active && !(isfinite(X[a][0]) && isfinite(X[a][1]) && isfinite(X[a][2]) && isfinite(V[a][0]) &&
                                 isfinite(V[a][1]) && isfinite(V[a][2]));
    const unsigned any_bad = __ballot_sync(0xffffffffu, bad);
    // (the offset read again: kept in registers across the steps, it costs k_propagate_mol<false, true> a spill)
    if (a == 0) { pot[k] = U + states[perm[k]].offset; kin[k] = KE; nan_flag[k] = (any_bad || !isfinite(U)) ? 1 : 0; }
    if (active)
        for (int c = 0; c < 3; c++) { pos[((size_t)r * n + a) * 3 + c] = X[a][c]; vel[((size_t)r * n + a) * 3 + c] = V[a][c]; }
}

// Hybrid Monte Carlo on a molecule (rx_set_hmc_integrator; HMCIntegrator, integrators.py:959-997): the block of
// k_propagate_mol, mv.n_steps trials of mv.n_steps constrained velocity-Verlet steps.  Per trial: v = sqrt(kT/m) g (Philox
// counter (atom, 0x90000000 + trial, k, iteration)), constrain velocities; Eold = KE + U; xold = x; n_steps x {v += dt/2 f/m;
// x1 = x + dt v; x = constrain(x1); v += dt/2 f(x)/m + (x - x1)/dt; constrain velocities}; Enew = KE + U; accept iff
// u <= exp(-(Enew - Eold)/kT) (u: counter (trial, 0xB0000000, k, iteration)), else x = x*0 + xold.  U is mol_energy's (f64,
// the same function as the energy rows), KE a fixed-tree warp sum in f64, the forces those of k_propagate_mol (f32 terms).
// No CM-motion removal: the reference removes it before the velocity draw, where it has no effect.  stats[r] += (accepted,
// trials) of a launch that ends finite; energy[r] = (Eold, Enew) of the last trial.
template <bool STAR, bool GB, bool ALCH>
__global__ void __launch_bounds__(32 * MOL_WARPS) k_propagate_mol_hmc(MolDev m, const __grid_constant__ MoveDev mv,
                                                          const StateDev *__restrict__ states, const int *__restrict__ perm,
                                                          double *__restrict__ pos, double *__restrict__ vel, int k0, uint2 key,
                                                          uint32_t iteration, double *__restrict__ pot, double *__restrict__ kin,
                                                          int *__restrict__ nan_flag, const int *__restrict__ only, MolGB g,
                                                          ulonglong2 *__restrict__ stats, double2 *__restrict__ energy) {
    __shared__ double X[MOL_MAX_ATOMS][3], XO[MOL_MAX_ATOMS][3], V[MOL_MAX_ATOMS][3];
    __shared__ int s_accept;
    extern __shared__ unsigned long long mol_tab[];
    const int r = blockIdx.x, k = k0 + r, a = threadIdx.x, n = m.n;
    if (only && !only[k]) return;
    unsigned char *tb = (unsigned char *)mol_tab;
    mol_stage(tb, m.terms32, m.bytes32);
    float (*FS)[3] = (float (*)[3])(tb + mol_slots_at(m, true));
    const MolGBArrays gs((double *)(tb + mol_gb_at(m, true)), n);
    __syncthreads();
    const int *g_off = (const int *)(tb + ((const MolTerms *)tb)->o_goff);
    const bool active = a < n;
    const StateDev st = states[perm[k]];
    const double mass = active ? m.mass[a] : 1.0, sg = sqrt(st.kT / mass), inv_mass = 1.0 / mass;
    if (active) for (int c = 0; c < 3; c++) { X[a][c] = pos[((size_t)r * n + a) * 3 + c]; V[a][c] = vel[((size_t)r * n + a) * 3 + c]; }
    MolCluster kc;
    MolStar ks;
    kc.nc = 0;
    const bool has_c = a < m.n_clusters;
    if (has_c) { if (STAR) mol_star_load(m, a, ks); else mol_load_cluster(m, a, kc); }
    __syncwarp();
    if (has_c && STAR) mol_star_init(ks, X);
    __syncwarp();
    auto rattle = [&]() {
        __syncwarp();
        if (has_c) { if (STAR) mol_star_rattle(ks, V); else mol_rattle_cluster(m, a, kc, X, V); }
        __syncwarp();
    };
    double f[3] = {0, 0, 0};
    auto forces = [&]() {   // every thread of the block (as in k_propagate_mol)
        __syncthreads();
        mol_terms<float, false, ALCH>(m, tb, X, FS, &st);
        if (GB) mol_gb_integrals<false, ALCH>(g, X, n, gs, &m, st.lambda_e);
        __syncthreads();
        if (GB) mol_gb_radii_pairs<false, ALCH>(g, X, m.charge, n, gs, &m, st.lambda_e);
        if (active) {
            float fx = 0.f, fy = 0.f, fz = 0.f;
            for (int q = g_off[a]; q < g_off[a + 1]; q++) { fx += FS[q][0]; fy += FS[q][1]; fz += FS[q][2]; }
            f[0] = fx; f[1] = fy; f[2] = fz;
            if (GB) mol_gb_force(X, a, n, gs, f);
        }
        __syncwarp();
    };
    auto total = [&]() {   // KE + U (warp 0's; every thread of the block calls it)
        __syncthreads();
        const double U = mol_energy<GB, ALCH>(m, g, (const unsigned char *)m.terms64, X, (double (*)[3])FS, gs, &st);
        return U + mol_warp_sum(active ? 0.5 * mass * (V[a][0] * V[a][0] + V[a][1] * V[a][1] + V[a][2] * V[a][2]) : 0.0);
    };
    const double dt = mv.dt_d, hdt = 0.5 * dt, inv_dt = 1.0 / dt;
    const int n_steps = mv.n_steps;
    unsigned long long n_acc = 0;
    double e_old = __longlong_as_double(0x7ff8000000000000ll), e_new = e_old;
    bool f_valid = false;
    for (int s = 0; s < n_steps; s++) {
        if (active) {
            const float3 gv = philox_normal3(philox4x32_10(make_uint4(a, 0x90000000u + (uint32_t)s, k, iteration), key));
            V[a][0] = sg * gv.x; V[a][1] = sg * gv.y; V[a][2] = sg * gv.z;
        }
        rattle();
        e_old = total();
        double xold[3] = {0, 0, 0};
        if (active) for (int c = 0; c < 3; c++) xold[c] = X[a][c];
        if (!f_valid) forces();
        for (int j = 0; j < n_steps; j++) {
            double xu[3] = {0, 0, 0};
            if (active)
                for (int c = 0; c < 3; c++) { V[a][c] += hdt * f[c] * inv_mass; XO[a][c] = X[a][c]; X[a][c] += dt * V[a][c]; xu[c] = X[a][c]; }
            __syncwarp();
            if (has_c) { if (STAR) mol_star_shake(m, ks, X); else mol_shake_cluster(m, a, kc, XO, X); }
            forces();
            if (active) for (int c = 0; c < 3; c++) V[a][c] += hdt * f[c] * inv_mass + (X[a][c] - xu[c]) * inv_dt;
            rattle();
        }
        f_valid = true;
        e_new = total();
        if (a == 0) {   // warp 0's energies decide; every warp takes the decision (the force evaluations are block-wide)
            const uint4 rr = philox4x32_10(make_uint4((uint32_t)s, 0xB0000000u, k, iteration), key);
            const double u = ((double)rr.x + 0.5) * 2.3283064365386963e-10;
            s_accept = u <= exp(-(e_new - e_old) / st.kT);   // (NaN: rejected)
        }
        __syncthreads();
        if (s_accept) {
            n_acc++;
        } else {
            if (active) for (int c = 0; c < 3; c++) X[a][c] = isfinite(X[a][c]) ? xold[c] : X[a][c] * 0.0;
            __syncwarp();
            if (has_c && STAR) mol_star_init(ks, X);   // (the SHAKE cache is that of the constrained start)
            f_valid = false;
        }
    }
    __syncthreads();
    const double U = mol_energy<GB, ALCH>(m, g, (const unsigned char *)m.terms64, X, (double (*)[3])FS, gs, &st);
    const double KE = mol_warp_sum(active ? 0.5 * mass * (V[a][0] * V[a][0] + V[a][1] * V[a][1] + V[a][2] * V[a][2]) : 0.0);
    const bool bad = active && !(isfinite(X[a][0]) && isfinite(X[a][1]) && isfinite(X[a][2]) && isfinite(V[a][0]) &&
                                 isfinite(V[a][1]) && isfinite(V[a][2]));
    const unsigned any_bad = __ballot_sync(0xffffffffu, bad);
    if (a == 0) {
        pot[k] = U + states[perm[k]].offset; kin[k] = KE;
        nan_flag[k] = (any_bad || !isfinite(U)) ? 1 : 0;
        if (!nan_flag[k]) { const ulonglong2 c = stats[r]; stats[r] = make_ulonglong2(c.x + n_acc, c.y + (unsigned)n_steps); }
        energy[r] = make_double2(e_old, e_new);
    }
    if (active)
        for (int c = 0; c < 3; c++) { pos[((size_t)r * n + a) * 3 + c] = X[a][c]; vel[((size_t)r * n + a) * 3 + c] = V[a][c]; }
}

// MultiStateSampler.minimize (multistatesampler.py:611-647) for a molecule: FIRE descent on the constraint manifold.  The
// force is projected onto the manifold (components along the constrained bonds removed: the RATTLE solve with unit
// weights, unit-weight sweeps for clusters of more than MOL_MAXC constraints), the move is followed by SHAKE, the FIRE
// velocity is kept tangent.  Converged when the RMS of the projected force
// falls below tol_rms (kJ/mol/nm); f64 throughout.  (OpenMM's L-BFGS is not reproduced, as for the other systems.)
// GB: the OBC force of g added to each atom's (mol_gb_radii_pairs, mol_gb_force).
// ALCH: at the lambdas of the replica's state (states[perm[k]]).
template <bool GB, bool ALCH>
__global__ void __launch_bounds__(32) k_minimize_mol(MolDev m, double *__restrict__ pos, int k0, double tol_rms, int max_iter,
                                                     double *__restrict__ rms_out, int *__restrict__ iters_out, MolGB g,
                                                     const StateDev *__restrict__ states, const int *__restrict__ perm) {
    __shared__ double X[MOL_MAX_ATOMS][3], XO[MOL_MAX_ATOMS][3], V[MOL_MAX_ATOMS][3], F[MOL_MAX_ATOMS][3];
    extern __shared__ unsigned long long mol_tab[];
    const int r = blockIdx.x, k = k0 + r, a = threadIdx.x, n = m.n;
    const bool active = a < n;
    StateDev st;
    if (ALCH) st = states[perm[k]];
    unsigned char *tb = (unsigned char *)mol_tab;
    mol_stage(tb, m.terms64, m.bytes64);
    double (*FS)[3] = (double (*)[3])(tb + mol_slots_at(m, false));
    const MolGBArrays gs((double *)(tb + mol_gb_at(m, false)), n);
    const int *goff = (const int *)(tb + ((const MolTerms *)tb)->o_goff);
    MolCluster kc, ku;   // the cluster with its masses (SHAKE) and with unit weights (projections)
    kc.nc = ku.nc = 0;
    if (a < m.n_clusters) {
        mol_load_cluster(m, a, kc);
        ku = kc;
#pragma unroll
        for (int c = 0; c < MOL_MAXC; c++) { const bool on = c < ku.nc; ku.wi[c] = on ? 1.0 : 0.0; ku.wj[c] = on ? 1.0 : 0.0; }
#pragma unroll
        for (int c = 0; c < MOL_MAXC; c++)
#pragma unroll
            for (int d = 0; d < MOL_MAXC; d++) {
                double v = 0.0;
                if (ku.i[c] == ku.i[d]) v += ku.wi[c];
                if (ku.i[c] == ku.j[d]) v -= ku.wi[c];
                if (ku.j[c] == ku.i[d]) v -= ku.wj[c];
                if (ku.j[c] == ku.j[d]) v += ku.wj[c];
                ku.coup[c][d] = v;
            }
    }
    if (active) for (int c = 0; c < 3; c++) { X[a][c] = pos[((size_t)r * n + a) * 3 + c]; V[a][c] = 0.0; }
    __syncwarp();
    const double dt0 = 0.001, dt_max = 0.010, alpha0 = 0.1, max_move = 0.01;   // (as k_minimize)
    double dt = dt0, alpha = alpha0, rms = 0.0;
    int n_pos = 0, it = 0;
    for (;; it++) {
        double f[3] = {0, 0, 0};
        mol_terms<double, false, ALCH>(m, tb, X, FS, &st);
        if (GB) mol_gb_integrals<false, ALCH>(g, X, n, gs, &m, st.lambda_e);
        __syncwarp();   // every term's contributions are in their slots
        if (GB) mol_gb_radii_pairs<false, ALCH>(g, X, m.charge, n, gs, &m, st.lambda_e);
        if (active) {   // this atom's slots, in slot order
            for (int q = goff[a]; q < goff[a + 1]; q++) for (int c = 0; c < 3; c++) f[c] += FS[q][c];
            if (GB) mol_gb_force(X, a, n, gs, f);
        }
        if (active) for (int c = 0; c < 3; c++) F[a][c] = f[c];
        __syncwarp();
        if (a < m.n_clusters) mol_rattle_cluster(m, a, ku, X, F, true);   // projected force
        __syncwarp();
        if (active) for (int c = 0; c < 3; c++) f[c] = F[a][c];
        const double FF = mol_warp_sum(active ? f[0] * f[0] + f[1] * f[1] + f[2] * f[2] : 0.0);
        rms = sqrt(FF / (3.0 * n));
        if (!(rms > tol_rms) || it >= max_iter) break;   // converged, out of iterations, or NaN
        double v[3] = {active ? V[a][0] : 0.0, active ? V[a][1] : 0.0, active ? V[a][2] : 0.0};
        const double P = mol_warp_sum(f[0] * v[0] + f[1] * v[1] + f[2] * v[2]);
        const double VV = mol_warp_sum(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
        if (P > 0.0) {
            const double mix = alpha * sqrt(VV / fmax(FF, 1e-300));
            for (int c = 0; c < 3; c++) v[c] = (1.0 - alpha) * v[c] + mix * f[c];
            if (++n_pos > 5) { dt = fmin(dt * 1.1, dt_max); alpha *= 0.99; }
        } else {
            v[0] = v[1] = v[2] = 0.0; dt *= 0.5; alpha = alpha0; n_pos = 0;
        }
        const double inv_m = active ? 1.0 / m.mass[a] : 0.0;
        for (int c = 0; c < 3; c++) v[c] += dt * f[c] * inv_m;
        double mv[3] = {dt * v[0], dt * v[1], dt * v[2]};
        const double m2 = mv[0] * mv[0] + mv[1] * mv[1] + mv[2] * mv[2];
        if (m2 > max_move * max_move) {   // displacement cap: rescale this atom's velocity
            const double sc = max_move / sqrt(m2);
            for (int c = 0; c < 3; c++) { v[c] *= sc; mv[c] *= sc; }
        }
        if (active) for (int c = 0; c < 3; c++) { XO[a][c] = X[a][c]; X[a][c] += mv[c]; V[a][c] = v[c]; }
        __syncwarp();
        if (a < m.n_clusters) mol_shake_cluster(m, a, kc, XO, X);
        __syncwarp();
        if (a < m.n_clusters) mol_rattle_cluster(m, a, ku, X, V, true);   // velocity stays tangent
        __syncwarp();
    }
    if (a == 0) { rms_out[k] = rms; iters_out[k] = it; }
    if (active) for (int c = 0; c < 3; c++) pos[((size_t)r * n + a) * 3 + c] = X[a][c];
}

// u[k][l] = beta_l (U(x_k) + offset_l): the states of a molecule differ in temperature only (parallel tempering,
// paralleltempering.py:175-237: one potential evaluation per replica, scaled by beta_l).
// GB: with the OBC energy of g.
// ALCH: u[k][l] = beta_l (U_l(x_k) + offset_l) of an alchemical molecule: the lambda-independent part once per replica, the
// OBC energy again only where lambda_electrostatics differs from the previous state's, the alchemical pairs only where
// (lambda_sterics, lambda_electrostatics) does -- the functions and the order of additions of mol_energy<GB, true>.
template <bool GB, bool ALCH>
__global__ void __launch_bounds__(32) k_energy_mol(MolDev m, const StateDev *__restrict__ states, int n_states,
                                                   const double *__restrict__ pos, int k0, double *__restrict__ u_out, MolGB g) {
    __shared__ double X[MOL_MAX_ATOMS][3];
    extern __shared__ unsigned long long mol_tab[];
    const int r = blockIdx.x, k = k0 + r, a = threadIdx.x, n = m.n;
    unsigned char *tb = (unsigned char *)mol_tab;
    mol_stage(tb, m.terms64, m.bytes64);
    if (a < n) for (int c = 0; c < 3; c++) X[a][c] = pos[((size_t)r * n + a) * 3 + c];
    __syncthreads();
    double (*S)[3] = (double (*)[3])(tb + mol_slots_at(m, false));
    const MolGBArrays gs((double *)(tb + mol_gb_at(m, false)), n);
    if (!ALCH) {
        const double U = mol_energy<GB>(m, g, tb, X, S, gs);
        for (int l = a; l < n_states; l += 32) u_out[(size_t)k * n_states + l] = states[l].beta * (U + states[l].offset);
        return;
    }
    const double u0 = mol_energy_fixed(m, tb, X, S);
    double e_gb = 0.0, e_ap = 0.0;
    for (int l = 0; l < n_states; l++) {
        const StateDev st = states[l];
        const bool new_e = l == 0 || st.lambda_e != states[l - 1].lambda_e;
        if (GB && new_e) e_gb = mol_energy_gb(m, g, X, gs, st.lambda_e);
        if (new_e || st.la != states[l - 1].la || st.ob != states[l - 1].ob) e_ap = mol_alch_energy(m, tb, X, st);
        if (a == 0) u_out[(size_t)k * n_states + l] = st.beta * ((u0 + (e_gb + e_ap)) + st.offset);
    }
}

__global__ void k_randomize_velocities_mol(MolDev m, const StateDev *__restrict__ states, const int *__restrict__ perm,
                                           double *__restrict__ vel, int k0, uint2 key, uint32_t stream_id) {
    const int r = blockIdx.x, k = k0 + r, a = threadIdx.x;
    if (a >= m.n) return;
    const StateDev st = states[perm[k]];
    const double sv = sqrt(st.kT / m.mass[a]);
    const float3 g = philox_normal3(philox4x32_10(make_uint4(a, 0xC0000000u, k, stream_id), key));
    vel[((size_t)r * m.n + a) * 3 + 0] = sv * g.x;
    vel[((size_t)r * m.n + a) * 3 + 1] = sv * g.y;
    vel[((size_t)r * m.n + a) * 3 + 2] = sv * g.z;
}

