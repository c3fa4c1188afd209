// rx_mc.cuh -- Monte Carlo rigid-body moves (included at the end of rx_dynamics.cu, after rx_molecule.cuh).
//
// MCDisplacementMove and MCRotationMove as MetropolizedMove.apply runs them (/root/reference/openmmtools/mcmc.py:810-970,
// 1704-1911), for every owned replica at once: rxi_mc_moves makes one launch per move slot j, in which replica k applies move
// j of the state it is in (perm[k]) or does nothing.  The proposal and the acceptance uniform are Philox blocks keyed as the
// propagation noise, with counters (j, 0xE0000000, k, iteration) and (j, 0xE0000001, k, iteration): the O step's counters
// stay far below that tag, and 0x80000000 / 0xA0000000 / 0xC0000000 belong to the velocity reassignment, the barostat and
// k_randomize_velocities.  The energy change is f64; positions keep their storage precision (f32, a molecule's f64), and the
// energy is that of the stored proposal, so that it is the difference of two rows of rx_compute_energies.
//
// k_mc_move      LJ fluid (one block per replica, N <= 4096): dU over the pairs with an atom in the subset, by
//                k_energy_rows' pair rules at the replica's own state (soft core, switch, two regions, the replica's box
//                under NPT), summed in a fixed order; proposed positions are rounded to f32 and wrapped into the box as
//                k_propagate wraps them (wrap_into), and dU is that of the wrapped f32 positions.  Harmonic systems: dU of
//                the subset's K/2 |x - x0|^2.
// k_mc_move_mol  small molecules in vacuum or OBC solvent (one warp per replica): the whole energy (mol_energy) before and
//                after, GB being many-body.
// Both kernels write the dU of every proposal to du[r][slot] (NaN when a rotation was rejected before any energy), so that it
// can be checked against rows of rx_compute_energies (rx_get_mc_energy_changes).
#pragma once

__device__ __forceinline__ double mc_u32(uint32_t w) { return ((double)w + 0.5) * (1.0 / 4294967296.0); }
// numpy's random_sample from two words: (a >> 5, b >> 6) as a 53-bit fraction
__device__ __forceinline__ double mc_u53(uint4 w) {
    return ((double)(w.x >> 5) * 67108864.0 + (double)(w.y >> 6)) * (1.0 / 9007199254740992.0);
}

// The proposal of move `mv` from the Philox block w: T[0..2] the displacement (sigma times three Box-Muller normals), or T[0..8]
// the rotation matrix (row major) of Shoemake's uniform quaternion (mcmc.py:1869-1906).
__device__ __forceinline__ void mc_proposal(const rx_mc_move &mv, uint4 w, double *T) {
    const double two_pi = 6.283185307179586;
    if (mv.kind == RX_MC_DISPLACEMENT) {
        const double ra = sqrt(-2.0 * log(mc_u32(w.x))), rb = sqrt(-2.0 * log(mc_u32(w.z)));
        T[0] = mv.sigma_nm * (ra * cos(two_pi * mc_u32(w.y)));
        T[1] = mv.sigma_nm * (ra * sin(two_pi * mc_u32(w.y)));
        T[2] = mv.sigma_nm * (rb * cos(two_pi * mc_u32(w.w)));
        return;
    }
    const double u0 = mc_u32(w.x), u1 = mc_u32(w.y), u2 = mc_u32(w.z);
    const double qw = sqrt(1.0 - u0) * sin(two_pi * u1), qx = sqrt(1.0 - u0) * cos(two_pi * u1);
    const double qy = sqrt(u0) * sin(two_pi * u2), qz = sqrt(u0) * cos(two_pi * u2);
    const double Nq = qw * qw + qx * qx + qy * qy + qz * qz;
    const double s = Nq > 0.0 ? 2.0 / Nq : 0.0;
    const double X = qx * s, Y = qy * s, Z = qz * s;
    const double wX = qw * X, wY = qw * Y, wZ = qw * Z, xX = qx * X, xY = qx * Y, xZ = qx * Z, yY = qy * Y, yZ = qy * Z, zZ = qz * Z;
    T[0] = 1.0 - (yY + zZ); T[1] = xY - wZ;          T[2] = xZ + wY;
    T[3] = xY + wZ;         T[4] = 1.0 - (xX + zZ);  T[5] = yZ - wX;
    T[6] = xZ - wY;         T[7] = yZ + wX;          T[8] = 1.0 - (xX + yY);
}

__device__ __forceinline__ void mc_rotate(const double *R, const double *v, double *out) {
    for (int a = 0; a < 3; a++) out[a] = R[3 * a] * v[0] + R[3 * a + 1] * v[1] + R[3 * a + 2] * v[2];
}

// The Metropolis test of mcmc.py:930-937 with the replica's beta, u from block (slot, 0xE0000001, k, iteration); counted.
__device__ __forceinline__ bool mc_accept(bool ok, double dU, double beta, int slot, int k, uint32_t iteration, uint2 key,
                                          unsigned long long *acc, unsigned long long *prop) {
    const double u = mc_u53(philox4x32_10(make_uint4((uint32_t)slot, 0xE0000001u, (uint32_t)k, iteration), key));
    const double bdu = beta * dU;
    const bool yes = ok && isfinite(dU) && (bdu <= 0.0 || u < exp(-bdu));
    atomicAdd(prop, 1ull);
    if (yes) atomicAdd(acc, 1ull);
    return yes;
}

// One pair's energy by the rules of k_energy_rows at state st (d: the raw displacement; minimum image here).
template <bool REG>
__device__ __forceinline__ double mc_pair_energy(const EnParams &p, const StateDev &st, const double4 &ai, const double4 &aj,
                                                 double dx, double dy, double dz) {
    dx = min_image_d(dx, p.Lx); dy = min_image_d(dy, p.Ly); dz = min_image_d(dz, p.Lz);
    const double r2 = dx * dx + dy * dy + dz * dz;
    if (r2 >= p.rc2) return 0.0;
    const double sig = 0.5 * (ai.x + aj.x), eps = sqrt(ai.y * aj.y);
    bool soft;
    double la = st.la, ob = st.ob;
    if constexpr (REG) {
        const int ri = (int)ai.w, rj = (int)aj.w, rr = ri | rj;
        if (rr == 3) return 0.0;   // across the two regions: no interaction
        soft = ri != rj || (((p.annihilate << 1) >> ri) & 1);
        if (rr >= 2) { la = st.la2; ob = st.ob2; }
    } else {
        const bool alch_i = ai.w != 0.0, alch_j = aj.w != 0.0;
        soft = (alch_i != alch_j) || (alch_i && alch_j && p.annihilate);
    }
    if (!soft) {
        const double s2 = sig * sig / r2, s6 = s2 * s2 * s2;
        return 4.0 * eps * (s6 * s6 - s6) * switch_d(p, sqrt(r2));
    }
    const double q = r2 / (sig * sig);
    const double rsc = p.c_is_6 ? q * q * q : pow(q, 0.5 * p.sc_c);
    const double D = ob + rsc;
    const double x = p.c_is_6 ? 1.0 / D : pow(D, -6.0 / p.sc_c);
    return la * (4.0 * eps * switch_d(p, sqrt(r2))) * x * (x - 1.0);
}

// Shared memory: old and proposed positions of every atom (float4 each), then a byte per atom: 1 in the subset.
__host__ __device__ inline size_t mc_smem_bytes(int N) { return (size_t)2 * N * sizeof(float4) + (((size_t)N + 15) & ~(size_t)15); }

template <bool NPT, bool REG>
__global__ void __launch_bounds__(256) k_mc_move(EnParams p, const double4 *__restrict__ atom_d, const StateDev *__restrict__ states,
                                                 const int *__restrict__ perm, const rx_mc_move *__restrict__ moves,
                                                 const int32_t *__restrict__ atoms, float4 *__restrict__ pos, int k0, int slot,
                                                 uint2 key, uint32_t iteration, const double4 *__restrict__ box,
                                                 unsigned long long *__restrict__ n_acc, unsigned long long *__restrict__ n_prop,
                                                 double *__restrict__ du) {
    extern __shared__ float4 s_mc[];
    float4 *s_old = s_mc, *s_new = s_mc + p.N;
    unsigned char *s_in = (unsigned char *)(s_new + p.N);
    __shared__ double s_red[32];
    __shared__ double s_T[12];   // the proposal (mc_proposal), then the rotation's centre
    __shared__ int s_ok;
    const int r = blockIdx.x, k = k0 + r, t = threadIdx.x, nt = blockDim.x;
    const int l = perm[k];
    const rx_mc_move mv = moves[l * RX_MAX_MC_MOVES + slot];
    if (mv.kind < 0) {
        if (t == 0) du[r * RX_MAX_MC_MOVES + slot] = __longlong_as_double(0x7ff8000000000000ll);
        return;
    }
    if constexpr (NPT) { const double4 b = box[r]; p.Lx = b.x; p.Ly = b.y; p.Lz = b.z; }
    const StateDev st = states[l];
    const bool lj = p.kind == RX_SYSTEM_LJ_ALCH;
    float4 *x = pos + (size_t)r * p.N;
    for (int q = t; q < p.N; q += nt) { const float4 v = x[q]; s_old[q] = v; s_new[q] = v; s_in[q] = 0; }
    const int32_t *sub = atoms + mv.subset_offset;
    const int ns = mv.subset_len;
    if (t == 0) {
        mc_proposal(mv, philox4x32_10(make_uint4((uint32_t)slot, 0xE0000000u, (uint32_t)k, iteration), key), s_T);
        s_ok = 1;
    }
    __syncthreads();
    for (int q = t; q < ns; q += nt) s_in[sub[q]] = 1;
    const double L[3] = {p.Lx, p.Ly, p.Lz};
    const BoxF bf = box_f(p.Lx, p.Ly, p.Lz);
    // the stored proposal: f32, wrapped into the box as k_propagate wraps (a periodic system)
    auto store = [&](const double *v, float w) {
        float x = (float)v[0], y = (float)v[1], z = (float)v[2];
        if (lj) wrap_into(bf, x, y, z);
        return make_float4(x, y, z, w);
    };
    if (mv.kind == RX_MC_DISPLACEMENT) {
        for (int q = t; q < ns; q += nt) {
            const int i = sub[q];
            const float4 o = s_old[i];
            const double v[3] = {(double)o.x + s_T[0], (double)o.y + s_T[1], (double)o.z + s_T[2]};
            s_new[i] = store(v, o.w);
        }
    } else {
        // periodic: offsets from the first atom by minimum image (the subset made whole); otherwise the positions themselves
        const float4 f0 = s_old[sub[0]];
        const double base[3] = {lj ? (double)f0.x : 0.0, lj ? (double)f0.y : 0.0, lj ? (double)f0.z : 0.0};
        auto offset = [&](int i, double *o) {
            const float4 f = s_old[i];
            o[0] = (double)f.x - base[0]; o[1] = (double)f.y - base[1]; o[2] = (double)f.z - base[2];
            if (lj) for (int a = 0; a < 3; a++) o[a] = min_image_d(o[a], L[a]);
        };
        double m[3] = {0.0, 0.0, 0.0};
        for (int q = t; q < ns; q += nt) {
            double o[3];
            offset(sub[q], o);
            for (int a = 0; a < 3; a++) m[a] += o[a];
        }
        for (int a = 0; a < 3; a++) {
            const double s = block_reduce_sum(m[a], s_red);
            if (t == 0) s_T[9 + a] = s / ns;
        }
        __syncthreads();
        const double mean[3] = {s_T[9], s_T[10], s_T[11]};
        const double c[3] = {base[0] + mean[0], base[1] + mean[1], base[2] + mean[2]};
        for (int q = t; q < ns; q += nt) {
            const int i = sub[q];
            double o[3], d[3], v[3];
            offset(i, o);
            if (lj) {   // the rotated offset from the first atom must stay inside half a box edge
                mc_rotate(s_T, o, v);
                for (int a = 0; a < 3; a++) if (!(fabs(v[a]) < 0.5 * L[a])) s_ok = 0;
            }
            for (int a = 0; a < 3; a++) d[a] = o[a] - mean[a];
            mc_rotate(s_T, d, v);
            for (int a = 0; a < 3; a++) v[a] += c[a];
            s_new[i] = store(v, s_old[i].w);
        }
    }
    __syncthreads();
    const bool ok = s_ok != 0;
    double dU = 0.0;
    if (ok && !lj) {
        for (int q = t; q < ns; q += nt) {
            const float4 o = s_old[sub[q]], n = s_new[sub[q]];
            double eo = 0.0, en = 0.0;
            const double od[3] = {o.x - st.ho_x0[0], o.y - st.ho_x0[1], o.z - st.ho_x0[2]};
            const double nd[3] = {n.x - st.ho_x0[0], n.y - st.ho_x0[1], n.z - st.ho_x0[2]};
            for (int a = 0; a < 3; a++) { eo += od[a] * od[a]; en += nd[a] * nd[a]; }
            dU += 0.5 * st.ho_K * en - 0.5 * st.ho_K * eo;
        }
    } else if (ok) {
        // every pair with an atom i of the subset once: j outside the subset, or j in it with j > i
        for (int q = 0; q < ns; q++) {
            const int i = sub[q];
            const double4 ai = atom_d[i];
            const float4 oi = s_old[i], ni = s_new[i];
            for (int j = t; j < p.N; j += nt) {
                if (j == i || (s_in[j] && j < i)) continue;
                const double4 aj = atom_d[j];
                const float4 oj = s_old[j], nj = s_new[j];
                dU += mc_pair_energy<REG>(p, st, ai, aj, (double)ni.x - nj.x, (double)ni.y - nj.y, (double)ni.z - nj.z) -
                      mc_pair_energy<REG>(p, st, ai, aj, (double)oi.x - oj.x, (double)oi.y - oj.y, (double)oi.z - oj.z);
            }
        }
    }
    dU = block_reduce_sum(dU, s_red);
    __syncthreads();
    if (t == 0) {
        du[r * RX_MAX_MC_MOVES + slot] = ok ? dU : __longlong_as_double(0x7ff8000000000000ll);
        s_ok = mc_accept(ok, dU, st.beta, slot, k, iteration, key, n_acc + l * RX_MAX_MC_MOVES + slot,
                         n_prop + l * RX_MAX_MC_MOVES + slot) ? 1 : 0;
    }
    __syncthreads();
    if (s_ok)
        for (int q = t; q < ns; q += nt) { const float4 v = s_new[sub[q]]; x[sub[q]] = make_float4(v.x, v.y, v.z, 0.f); }
}

// A molecule: one warp per replica, lane q moves atom sub[q] (a subset has at most 32 atoms); the centre of a rotation is the
// plain mean of the subset (no periodic images).  pos: double[kloc][n][3].
template <bool GB, bool ALCH>
__global__ void __launch_bounds__(32) k_mc_move_mol(MolDev m, const StateDev *__restrict__ states, const int *__restrict__ perm,
                                                   const rx_mc_move *__restrict__ moves, const int32_t *__restrict__ atoms,
                                                   double *__restrict__ pos, int k0, int slot, uint2 key, uint32_t iteration,
                                                   unsigned long long *__restrict__ n_acc, unsigned long long *__restrict__ n_prop,
                                                   double *__restrict__ du, MolGB g) {
    __shared__ double X[MOL_MAX_ATOMS][3], XN[MOL_MAX_ATOMS][3];
    extern __shared__ unsigned long long mol_tab[];
    const int r = blockIdx.x, k = k0 + r, a = threadIdx.x, n = m.n;
    const int l = perm[k];
    const rx_mc_move mv = moves[l * RX_MAX_MC_MOVES + slot];
    if (mv.kind < 0) {
        if (a == 0) du[r * RX_MAX_MC_MOVES + slot] = __longlong_as_double(0x7ff8000000000000ll);
        return;
    }
    unsigned char *tb = (unsigned char *)mol_tab;
    mol_stage(tb, m.terms64, m.bytes64);
    double (*S)[3] = (double (*)[3])(tb + mol_slots_at(m, false));
    const MolGBArrays gs((double *)(tb + mol_gb_at(m, false)), n);
    if (a < n) for (int c = 0; c < 3; c++) X[a][c] = XN[a][c] = pos[((size_t)r * n + a) * 3 + c];
    __syncthreads();
    const StateDev st = states[l];
    const double U0 = __shfl_sync(0xffffffffu, mol_energy<GB, ALCH>(m, g, tb, X, S, gs, &st), 0);
    double T[9];
    mc_proposal(mv, philox4x32_10(make_uint4((uint32_t)slot, 0xE0000000u, (uint32_t)k, iteration), key), T);
    const int ns = mv.subset_len;
    const bool mine = a < ns;
    const int i = mine ? atoms[mv.subset_offset + a] : 0;
    if (mv.kind == RX_MC_DISPLACEMENT) {
        if (mine) for (int c = 0; c < 3; c++) XN[i][c] = X[i][c] + T[c];
    } else {
        double c[3], d[3], v[3];
        for (int q = 0; q < 3; q++) c[q] = __shfl_sync(0xffffffffu, mol_warp_sum(mine ? X[i][q] : 0.0), 0) / ns;
        if (mine) {
            for (int q = 0; q < 3; q++) d[q] = X[i][q] - c[q];
            mc_rotate(T, d, v);
            for (int q = 0; q < 3; q++) XN[i][q] = v[q] + c[q];
        }
    }
    __syncthreads();
    const double U1 = __shfl_sync(0xffffffffu, mol_energy<GB, ALCH>(m, g, tb, XN, S, gs, &st), 0);
    int yes = 0;
    if (a == 0) du[r * RX_MAX_MC_MOVES + slot] = U1 - U0;
    if (a == 0) yes = mc_accept(true, U1 - U0, states[l].beta, slot, k, iteration, key, n_acc + l * RX_MAX_MC_MOVES + slot,
                                n_prop + l * RX_MAX_MC_MOVES + slot) ? 1 : 0;
    yes = __shfl_sync(0xffffffffu, yes, 0);
    if (yes && mine) for (int c = 0; c < 3; c++) pos[((size_t)r * n + i) * 3 + c] = XN[i][c];
}

int rxi_mc_moves(rx_engine *h, uint64_t seed, uint64_t iteration, int *launches) {
    if (h->mc_slots == 0 || h->kloc == 0) return RX_OK;
    const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32) ^ (uint32_t)(iteration >> 32));
    const uint32_t it32 = (uint32_t)iteration;
    if (h->cfg.system_kind == RX_SYSTEM_MOLECULE) {
        const MolDev *md = &h->mol->dev;
        const MolGB *gb = mol_gb_of(h);
        auto kern = with_flag(gb != nullptr, [&](auto g) { return with_flag(mol_alch(h), [&](auto al) { return k_mc_move_mol<g, al>; }); });
        const int dyn = mol_dyn_bytes(*md, gb, false);
        const int rco = smem_opt_in(h, (const void *)kern, dyn);
        if (rco) return rco;
        for (int s = 0; s < h->mc_slots; s++) {
            kern<<<h->kloc, 32, dyn, h->stream>>>(*md, h->d_states, h->d_perm, h->d_mc_moves, h->d_mc_atoms, (double *)h->d_pos.get(), h->k0,
                                                  s, key, it32, h->d_mc_acc, h->d_mc_prop, h->d_mc_du, gb ? *gb : MolGB{});
            RX_CHECK_CUDA(h, cudaGetLastError());
        }
    } else {
        const EnParams p = en_params(h, h->cfg.n_states);
        const size_t smem = mc_smem_bytes(h->cfg.n_atoms);
        auto kern = h->two_regions ? (h->npt ? k_mc_move<true, true> : k_mc_move<false, true>)
                                   : (h->npt ? k_mc_move<true, false> : k_mc_move<false, false>);
        const int rco = smem_opt_in(h, (const void *)kern, (int)smem);
        if (rco) return rco;
        for (int s = 0; s < h->mc_slots; s++) {
            kern<<<h->kloc, 256, smem, h->stream>>>(p, h->d_atom_d, h->d_states, h->d_perm, h->d_mc_moves, h->d_mc_atoms, h->d_pos,
                                                    h->k0, s, key, it32, h->d_box, h->d_mc_acc, h->d_mc_prop, h->d_mc_du);
            RX_CHECK_CUDA(h, cudaGetLastError());
        }
    }
    *launches += h->mc_slots;
    return RX_OK;
}
